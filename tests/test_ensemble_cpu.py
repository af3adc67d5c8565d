"""CPU: several CLIP towers guiding one step (`clip_model_name=[...]`, GuidedStepB200 with sequences of towers).  The two-tower step's op
list on the interpreter against the fp32 ensemble oracle (tests/ensemble_oracle.py), the one-tower op list unchanged, the CPU-generator
draw order of the windows, the entry's per-tower targets and refusals, checkpoint paths as tower names, CUTOUTS_BWD flags checks."""
import ctypes
import os

import pytest
import torch as th

from clip_guided_diffusion_b200 import _lib
from clip_guided_diffusion_b200 import cgd
from clip_guided_diffusion_b200 import guidance as pg
from clip_guided_diffusion_b200 import rn as prn
from clip_guided_diffusion_b200 import vit as pv
from clip_guided_diffusion_b200 import weights as pw
from clip_guided_diffusion_b200.plan import Plan
from tests.ensemble_oracle import build_ensemble, interp_runner, run_ensemble_step
from tests.step_parity import build_tiny


# ---------------------------------------------------------------------------------------------------------------- one tower = today
def _ops(eng):
    return [(op.code, op.flags, list(op.i), list(op.f), [None if p is None else (p[0].off, p[0].dt, p[1]) for p in op.p]) for op in eng.plan.ops]


def test_one_element_list_engine_is_the_single_tower_engine(monkeypatch):
    ctx = build_tiny("cpu", B=2, cutn=3, image=32, cutn_variants=(2,))
    a = ctx["eng"]
    b = pg.GuidedStepB200(a.unet.cfg, ctx["ounet"].state_dict(), [a.towers[0].cfg], [ctx["oclip"].state_dict()], batch=2, num_cutouts=3,
                          device="cpu", cutn_variants=(2,), **ctx["kw"])
    assert a.T == b.T == 1 and b.loss_towers is None
    assert _ops(a) == _ops(b) and a.plan.marks == b.plan.marks and a.plan._size == b.plan._size
    assert bytes(a.plan.lower(0)) == bytes(b.plan.lower(0))  # the C structs the native plan is created from
    monkeypatch.setattr(Plan, "num_launches", lambda self, first=0, count=None: count)  # no native plan on the CPU: count ops
    for mode in ("ancestral", "ddim"):
        assert a.launches_per_step(mode) == b.launches_per_step(mode)


def test_two_tower_engine_layout():
    ctx = build_ensemble("cpu", B=1, cutn=2)
    eng = ctx["eng"]
    assert eng.T == 2 and [tw.tag for tw in eng.towers] == ["", "#1"]
    bwd = [op for op in eng.plan.ops if op.code == _lib.OP["CUTOUTS_BWD"]]
    assert [op.flags for op in bwd] == [0, 2]  # tower 0 stores, tower 1 adds, in that launch order
    assert bwd[0].p[2] == bwd[1].p[2] == (eng.g_clip, 0)
    for m in ("cut_fwd", "sph", "cut_bwd", "cut_end", "vit_fwd", "vit_bwd", "vit_end"):
        assert eng.plan.marks[m] < eng.plan.marks[m + "#1"] or m.startswith("vit")
        assert m + "#1" in eng.plan.marks
    assert eng.plan.marks["cut_end#1"] <= eng.plan.marks["guide"]
    with pytest.raises(ValueError, match="sequence"):
        eng.set_targets(ctx["targets"][0], ctx["weights"])
    with pytest.raises(ValueError):
        eng.set_targets(ctx["targets"][:1], ctx["weights"])
    with pytest.raises(ValueError, match="width"):
        eng.set_targets([ctx["targets"][1], ctx["targets"][0]], ctx["weights"])
    with pytest.raises(ValueError, match="window lists"):
        eng.stage_step(ctx["pdiff"].scalar_table(3, 3, 0.0), [[(0, 0, 32)] * 2], 3.0, None)


# ---------------------------------------------------------------------------------------------------------------- step vs oracle
@pytest.mark.parametrize("mode,kw", [("ancestral", dict(B=2, P=1)), ("ddim", dict(B=2, P=1)), ("ddim", dict(B=1, P=3, cutn=2)),
                                     ("ancestral", dict(B=2, sat_scale=30.0, use_magnitude=True)),
                                     ("ddim", dict(B=2, cutn=2, init_scale=1000.0)),
                                     ("ancestral", dict(B=1, cutn=8, cutn_variants=(2, 4), run_cutn=4))])
def test_two_tower_step_matches_the_ensemble_oracle(mode, kw):
    ctx = build_ensemble("cpu", **kw)
    res = run_ensemble_step(ctx, mode, runner=interp_runner(ctx["eng"]))
    assert res["cos_g"] > 0.999, res
    assert res["rel_g"] < 5e-2 and res["rel_x0"] < 2e-2 and res["rel_sample"] < 2e-2, res
    assert res["clip_loss_rel"] < 2e-2 and res["clip_sum_rel"] < 2e-2 and res["tv_loss_rel"] < 1e-3 and res["range_loss_rel"] < 1e-2, res
    per = ctx["eng"].losses()["clip_per_tower"]
    assert per.shape == (2, ctx["B"]) and bool((per > 0).all())


# ---------------------------------------------------------------------------------------------------------------- CPU generator
class _Eng:
    cutn, T = 4, 2
    vits = {4: None}


class _Diff:
    num_timesteps = 25


def test_windows_are_drawn_per_tower_in_tower_order():
    mks = [pg.MakeCutouts(32, 4), pg.MakeCutouts(224, 4)]
    cf = pg.CondFnB200(_Eng(), _Diff(), mks)
    th.manual_seed(5)
    got = cf.next_coords(256, 240)
    after = th.get_rng_state()
    th.manual_seed(5)
    want = [mks[0]._generate_coords(256, 240, 4), mks[1]._generate_coords(256, 240, 4)]
    assert got == want and th.equal(th.get_rng_state(), after)
    assert min(s for _, _, s in got[1]) >= 224 and max(s for _, _, s in got[1]) <= 240  # tower 1's own min_size = min(H, W, 224)
    th.manual_seed(6)
    sizes0 = [s for _, _, s in cf.next_coords(256, 240)[0]]
    assert min(sizes0) >= 32 and len(set(sizes0)) > 1
    # cached_cutouts: every tower's windows cached in tower order (cgd/cgd.py:113), then no draws at all
    th.manual_seed(7)
    for mk in mks:
        mk.cache_coordinates(240, 256)
    th.manual_seed(7)
    assert [mks[0].cached_coords, mks[1].cached_coords] == [m._generate_coords(240, 256, 4) for m in [pg.MakeCutouts(32, 4), pg.MakeCutouts(224, 4)]]
    cf = pg.CondFnB200(_Eng(), _Diff(), mks, cached_cutouts=True)
    state = th.get_rng_state()
    assert cf.next_coords(256, 240) == [mks[0].cached_coords, mks[1].cached_coords]
    assert th.equal(th.get_rng_state(), state)
    with pytest.raises(ValueError, match="MakeCutouts"):
        pg.CondFnB200(_Eng(), _Diff(), [pg.MakeCutouts(32, 4)])
    with pytest.raises(ValueError, match="same num_cutouts"):
        pg.CondFnB200(_Eng(), _Diff(), [pg.MakeCutouts(32, 4), pg.MakeCutouts(224, 3)])


def test_progressive_counts_apply_to_every_tower():
    class Eng(_Eng):
        cutn = 16
        vits = {4: None, 8: None, 16: None}
    cf = pg.CondFnB200(Eng(), _Diff(), [pg.MakeCutouts(32, 16), pg.MakeCutouts(64, 16)], progressive_cutout=True)
    for ct in (24, 12, 2):
        cf.current_timestep = ct
        got = cf.next_coords(64, 64)
        assert len(got) == 2 and len(got[0]) == len(got[1]) == cf.current_cutn()


def test_fused_steps_consume_the_generator_like_the_towers_make_cutouts():
    """DDIM, reduce_clip: guided steps draw tower 0's windows then tower 1's, then the noise; skipped steps draw only the noise"""
    ctx = build_ensemble("cpu", B=1, cutn=2)
    eng = ctx["eng"]
    it = interp_runner(eng)
    eng.plan.run_range = lambda a, b, stream=None: it(a, b)
    mks = [pg.MakeCutouts(cfg.input_resolution, 2) for cfg, _, _ in ctx["towers"]]
    cf = pg.CondFnB200(eng, ctx["pdiff"], mks, reduce_clip=True)
    x = th.randn(1, 3, 32, 32, generator=th.Generator().manual_seed(1))
    y = th.zeros(1, dtype=th.long)
    guided = []
    th.manual_seed(11)
    for ct in (24, 23):  # progress 4 %: guided; 8 %: skipped by reduce_clip's rule (cgd/cgd.py:157-164)
        cf.current_timestep = ct
        guided.append(not cf.skips_guidance())
        eng.fused_step(ctx["pdiff"], "ddim", ct, x, y, cf)
    assert guided == [True, False]
    after = th.get_rng_state()
    th.manual_seed(11)
    w = [m._generate_coords(32, 32, 2) for m in mks]  # the guided step: tower 0's windows, tower 1's, then the DDIM noise
    th.randn(1, 3, 32, 32)
    th.randn(1, 3, 32, 32)  # the skipped step: the noise only
    assert th.equal(th.get_rng_state(), after)
    assert [tuple(r) for r in eng.v(eng.towers[1].coords, (2, 3)).tolist()] == w[1]
    assert [tuple(r) for r in eng.v(eng.towers[0].coords, (2, 3)).tolist()] == w[0]


# ---------------------------------------------------------------------------------------------------------------- the entry
class _Stop(Exception):
    pass


class _RecordingEngine:
    """stands in for GuidedStepB200: records what the entry builds and stops the run at set_targets"""
    seen = {}

    def __init__(self, unet_cfg, unet_sd, vit_cfg, vit_sd, **kw):
        _RecordingEngine.seen = dict(vit_cfg=vit_cfg, vit_sd=vit_sd, **kw)

    def set_targets(self, target_embeds, weights):
        _RecordingEngine.seen.update(target_embeds=target_embeds, weights=weights)
        raise _Stop


def _sds():
    vcfg = pv.ViTConfig(32, 16, 64, 1, 32)
    rcfg = prn.RNConfig(layers=(1, 1, 1, 1), output_dim=48, input_resolution=64, width=64)
    return [(vcfg, pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 3)), (rcfg, pw.seeded_rn_state_dict(rcfg, seed=4))]


@pytest.fixture
def entry(monkeypatch, tmp_path):
    monkeypatch.setattr(cgd, "_require_cuda", lambda device: None)
    monkeypatch.setattr(cgd, "GuidedStepB200", _RecordingEngine)
    monkeypatch.chdir(tmp_path)
    events = []
    monkeypatch.setattr(cgd, "_text_encoder_choice", lambda *a: "vocab")

    def enc_device(prompts, clip_sd, vocab, device):
        D = clip_sd["visual.attnpool.c_proj.weight"].shape[0] if "visual.attnpool.c_proj.weight" in clip_sd else clip_sd["visual.proj"].shape[1]
        events.append(("text-device", D, tuple(prompts)))
        return th.full((len(prompts), D), float(D)), th.tensor([cgd.parse_prompt(p)[1] for p in prompts])

    def enc_clip(prompts, name, device):
        events.append(("text-clip", name, tuple(prompts)))
        return th.ones(len(prompts), 32), th.tensor([cgd.parse_prompt(p)[1] for p in prompts])
    monkeypatch.setattr(cgd, "_encode_text_device", enc_device)
    monkeypatch.setattr(cgd, "_encode_text", enc_clip)

    class FakeImageEncoder:
        def __init__(self, cfg, clip_sd, cutn, device):
            self.D, self.cutn = cfg.output_dim, cutn
            events.append(("image-encoder", self.D))

        def encode(self, path, w, size):
            events.append(("image", self.D, os.path.basename(path)))
            return th.zeros(self.cutn, self.D), [w / self.cutn] * self.cutn

        def __del__(self):
            events.append(("image-released", self.D))
    monkeypatch.setattr(cgd, "ImagePromptEncoder", FakeImageEncoder)
    kw = dict(image_size=64, num_cutouts=2, progress=False, device="cpu", unet_state_dict={}, prefix_path=tmp_path / "out")
    return events, kw


def _run(**kw):
    with pytest.raises(_Stop):
        next(cgd.clip_guided_diffusion(**kw))
    return _RecordingEngine.seen


def test_entry_encodes_targets_per_tower(entry, tmp_path):
    events, kw = entry
    (vcfg, vsd), (rcfg, rsd) = _sds()
    seen = _run(prompts=["a cat:2", "a dog"], clip_model_name=["ViT-B/32", "RN50"], clip_state_dict=[vsd, rsd], **kw)
    assert seen["vit_cfg"] == [vcfg, rcfg] and seen["vit_sd"] == [vsd, rsd] and seen["max_prompts"] == 2
    assert events == [("text-device", 32, ("a cat:2", "a dog")), ("text-device", 48, ("a cat:2", "a dog"))]
    assert [tuple(t.shape) for t in seen["target_embeds"]] == [(2, 32), (2, 48)] and th.allclose(seen["weights"], th.tensor([2 / 3, 1 / 3]))
    # the `clip` package path: _encode_text gets each tower's name
    events.clear()
    cgd._text_encoder_choice, keep = (lambda *a: None), cgd._text_encoder_choice
    try:
        _run(prompts=["a cat"], clip_model_name=["ViT-B/32", "RN50"], clip_state_dict=[vsd, rsd], **kw)
    finally:
        cgd._text_encoder_choice = keep
    assert events == [("text-clip", "ViT-B/32", ("a cat",)), ("text-clip", "RN50", ("a cat",))]
    # image prompts tower-major: tower 0's encoder takes every image, is released, then tower 1's
    events.clear()
    for n in ("a.png", "b.png"):
        (tmp_path / n).write_bytes(b"")
    seen = _run(image_prompts=[str(tmp_path / "a.png") + ":3", str(tmp_path / "b.png")], clip_model_name=["ViT-B/32", "RN50"],
                clip_state_dict=[vsd, rsd], **kw)
    assert events == [("image-encoder", 32), ("image", 32, "a.png"), ("image", 32, "b.png"), ("image-released", 32),
                      ("image-encoder", 48), ("image", 48, "a.png"), ("image", 48, "b.png"), ("image-released", 48)]
    assert [tuple(t.shape) for t in seen["target_embeds"]] == [(4, 32), (4, 48)]
    assert th.allclose(seen["weights"], th.tensor([1.5, 1.5, 0.5, 0.5]) / 4)
    # target_embeds= as one tensor per tower; weights= shared
    events.clear()
    tg = [th.randn(3, 32), th.randn(3, 48)]
    seen = _run(target_embeds=tg, weights=[1.0, 1.0, 2.0], clip_model_name=["ViT-B/32", "RN50"], clip_state_dict=[vsd, rsd], **kw)
    assert events == [] and all(a is b for a, b in zip(seen["target_embeds"], tg)) and th.allclose(seen["weights"], th.tensor([.25, .25, .5]))
    # one tower: the engine gets the plain config / state_dict / tensor as before
    seen = _run(target_embeds=tg[0], clip_model_name="ViT-B/32", clip_state_dict=vsd, **kw)
    assert seen["vit_cfg"] == vcfg and seen["vit_sd"] is vsd and seen["target_embeds"] is tg[0]


def test_entry_refusals_come_before_any_file_is_opened(entry, monkeypatch):
    events, kw = entry
    (_, vsd), (_, rsd) = _sds()

    def opened(*a, **k):
        raise AssertionError("a checkpoint or image was opened")
    for name in ("_load_clip_sd", "_load_clip_file", "check_local", "_load_unet_sd"):
        monkeypatch.setattr(cgd, name, opened)
    two = dict(clip_model_name=["ViT-B/32", "ViT-B/16"], prompts=["x"], image_prompts=["a.png"])
    with pytest.raises(NotImplementedError, match="use_augs"):
        next(cgd.clip_guided_diffusion(use_augs=True, **two, **kw))
    with pytest.raises(NotImplementedError, match="lanczos3"):
        next(cgd.clip_guided_diffusion(cutout_resize="lanczos3", **two, **kw))
    with pytest.raises(ValueError, match="clip_state_dict"):
        next(cgd.clip_guided_diffusion(clip_state_dict=[vsd], **two, **kw))
    with pytest.raises(ValueError, match="clip_state_dict"):
        next(cgd.clip_guided_diffusion(clip_state_dict=vsd, **two, **kw))
    with pytest.raises(ValueError, match="non-empty"):
        next(cgd.clip_guided_diffusion(clip_model_name=[], **kw))
    with pytest.raises(ValueError, match="sequence"):
        next(cgd.clip_guided_diffusion(clip_model_name=["ViT-B/32", "RN50"], target_embeds=th.randn(1, 32), **kw))
    with pytest.raises(ValueError, match="one \\[P, D_m\\] tensor per CLIP tower"):
        next(cgd.clip_guided_diffusion(clip_model_name=["ViT-B/32", "RN50"], target_embeds=[th.randn(1, 32)], **kw))
    with pytest.raises(ValueError, match="one \\[P, D_m\\] tensor per CLIP tower"):
        next(cgd.clip_guided_diffusion(clip_model_name=["ViT-B/32", "RN50"], target_embeds=[th.randn(1, 32), th.randn(2, 48)], **kw))
    assert events == []


def _scripted_clip(sd):
    """a TorchScript archive whose state_dict is `sd` (what OpenAI's CLIP .pt files are)"""
    root = th.nn.Module()
    for key, v in sd.items():
        mod = root
        *path, leaf = key.split(".")
        for part in path:
            if not hasattr(mod, part):
                mod.add_module(part, th.nn.Module())
            mod = getattr(mod, part)
        mod.register_buffer(leaf, v.clone())

    class Wrap(th.nn.Module):
        def __init__(self):
            super().__init__()
            self.visual = root.visual

        def forward(self, x):
            return x
    return th.jit.script(Wrap())


def test_checkpoint_paths_as_tower_names(entry, tmp_path):
    events, kw = entry
    (vcfg, vsd), (rcfg, rsd) = _sds()
    _scripted_clip(vsd).save(str(tmp_path / "vit_custom.pt"))
    th.save(rsd, tmp_path / "rn_plain.bin")  # an existing file counts as a path whatever its suffix
    sd, cfg = cgd._clip_tower(str(tmp_path / "vit_custom.pt"), None, str(tmp_path))
    assert cfg == vcfg and set(sd) == set(vsd) and all(th.equal(sd[k], vsd[k]) for k in vsd)
    sd, cfg = cgd._clip_tower(str(tmp_path / "rn_plain.bin"), None, str(tmp_path))
    assert cfg == rcfg and set(sd) == set(rsd)
    seen = _run(prompts=["a cat"], clip_model_name=[str(tmp_path / "vit_custom.pt"), str(tmp_path / "rn_plain.bin")], **kw)
    assert seen["vit_cfg"] == [vcfg, rcfg]
    assert events == [("text-device", 32, ("a cat",)), ("text-device", 48, ("a cat",))]
    events.clear()
    cgd._text_encoder_choice, keep = (lambda *a: None), cgd._text_encoder_choice
    try:
        _run(prompts=["a cat"], clip_model_name=str(tmp_path / "vit_custom.pt"), **kw)
    finally:
        cgd._text_encoder_choice = keep
    assert events == [("text-clip", str(tmp_path / "vit_custom.pt"), ("a cat",))]  # like the reference's clip.load(path)
    missing = str(tmp_path / "nowhere" / "vitb32_dalleblog_noise.pt")
    with pytest.raises(FileNotFoundError, match="vitb32_dalleblog_noise.pt"):
        cgd._clip_tower(missing, None, str(tmp_path))
    with pytest.raises(FileNotFoundError, match="nowhere"):
        next(cgd.clip_guided_diffusion(clip_model_name=[str(tmp_path / "vit_custom.pt"), missing], **kw))


# ---------------------------------------------------------------------------------------------------------------- CUTOUTS_BWD flags
def test_cutouts_bwd_flags_are_checked_before_any_cuda_call():
    lib = _lib.load()

    def run(flags, **over):
        op = _lib.CgdOp()
        op.code, op.flags = _lib.OP["CUTOUTS_BWD"], flags
        dims = dict(B=1, H=64, W=64, cutn=4, cs=32, P=16, kpad=768)
        dims.update(over)
        for j, v in enumerate(dims.values()):
            op.i[j] = v
        op.f[3] = op.f[4] = op.f[5] = op.f[6] = 1.0
        for j in range(3):
            op.p[j] = 256 * (j + 1)  # never dereferenced: the checks come first
        return lib.cgd_run_op(ctypes.byref(op), None), _lib.load().cgd_last_error().decode()
    for flags in (1, 3, 4, 6, -1):
        rc, msg = run(flags)
        assert rc < 0 and "flags" in msg, (flags, rc, msg)
    for bad in (dict(cutn=0), dict(cs=30), dict(kpad=10), dict(cs=2048, P=16)):
        rc, msg = run(2, **bad)
        assert rc < 0 and "cutouts" in msg, (bad, rc, msg)
