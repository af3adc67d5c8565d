"""CPU: the OpenCLIP towers (``"open_clip:<arch>"``, vit.OPEN_CLIP_CONFIGS) interpreted op by op (tests/open_clip_oracle.py).

- Reduced-depth towers of every geometry (real widths, heads, patch sizes and activations; 2 layers): the fp32 oracle against the
  independent ``transformers`` CLIP towers to fp32 round-off (skipped without ``transformers``), and separately the package's plan on the
  interpreter against the oracle (forward and input gradient, ViT-B-32 also at 1 and 2 images; the text towers forward).
- ViT-H's 80-wide heads packed to 128: zero rows / columns exactly where expected, the softmax scale 1 / sqrt(80).
- Name resolution, the checkpoint lookup, the shape checks and the text-encoder rules, each refusal before any file is opened.
- The plans of the OpenAI towers are unchanged (scripts/plan_fingerprint.py prints the table committed in tests/golden/).
- Every launch of the new plans has an owner (tests/open_clip_plan_table.py or an existing table)."""
from __future__ import annotations

import dataclasses
import math
import os
import subprocess
import sys
import types

import pytest
import torch as th

from clip_guided_diffusion_b200 import cgd
from clip_guided_diffusion_b200 import plan as pplan
from clip_guided_diffusion_b200 import text as ptx
from clip_guided_diffusion_b200 import vit as pv
from clip_guided_diffusion_b200 import weights as pw
from tests.open_clip_oracle import OpenClipInterp, encode_text, hf_text_model, hf_vision_model, vision_oracle
from tests.plan_interp import Interp
from tests.step_parity import cos, rel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARCHS = list(pv.OPEN_CLIP_CONFIGS)


def reduced(arch, layers=2):
    """(vision config, text config) of `arch` at `layers` layers"""
    v, t = pv.OPEN_CLIP_CONFIGS[arch]
    return dataclasses.replace(v, layers=layers), dataclasses.replace(t, layers=layers)


def seeded_sd(vcfg, tcfg=None, seed=1235):
    sd = pw.seeded_state_dict(pw.vit_param_shapes(vcfg), seed)
    if tcfg is not None:
        sd.update(pw.seeded_state_dict(pw.text_param_shapes(tcfg), seed + 1))
    return sd


def _fwd_grad(fn, x, seed):
    x = x.clone().requires_grad_()
    y = fn(x)
    (g,) = th.autograd.grad((y * seed).sum(), x)
    return y.detach(), g


# ---------------------------------------------------------------------- towers against transformers and the oracle
def _vision_case(arch, n=3):
    """(reduced config, weights, images, seed, oracle embeddings, oracle input gradient)"""
    cfg, _ = reduced(arch)
    sd = seeded_sd(cfg)
    g = th.Generator().manual_seed(3)
    x = th.randn(n, 3, cfg.input_resolution, cfg.input_resolution, generator=g)
    seed = th.randn(n, cfg.output_dim, generator=g)
    y0, g0 = _fwd_grad(vision_oracle(cfg, sd).encode_image, x, seed)
    return cfg, sd, x, seed, y0, g0


@pytest.mark.parametrize("arch", ARCHS)
def test_vision_oracle_matches_transformers(arch):
    pytest.importorskip("transformers")
    cfg, sd, x, seed, y0, g0 = _vision_case(arch)
    y1, g1 = _fwd_grad(lambda t: hf_vision_model(cfg, sd)(pixel_values=t).image_embeds, x, seed)
    ey, eg = float((y0 - y1).abs().max() / y1.abs().max()), float((g0 - g1).abs().max() / g1.abs().max())
    assert ey < 2e-5 and eg < 2e-5, (arch, ey, eg)


@pytest.mark.parametrize("arch,n", [(a, 3) for a in ARCHS] + [("ViT-B-32", 1), ("ViT-B-32", 2)])
def test_vision_plan_matches_the_oracle(arch, n):
    """the package's tower on the interpreter against the oracle, forward and input gradient; ViT-B-32 at 1 and 2 images too, where the
    c_proj dgrad spans one pixel tile and the planner forces the GELU' epilogue's BN >= 64 / no split-K"""
    cfg, sd, x, seed, y0, g0 = _vision_case(arch, n)
    R = cfg.input_resolution
    net = pv.ViTB200(cfg, sd, n_images=n, device="cpu")
    it = OpenClipInterp(net.plan)
    G2, kp, P = cfg.grid ** 2, cfg.kpad, cfg.patch_size
    net.plan.view(net.patches, (n, G2, kp)).copy_(Interp._patchify(x, P, kp))
    it.run_range("vit_fwd", "vit_bwd")
    emb = net.plan.view(net.embeds, (n, cfg.output_dim)).clone()
    assert rel(emb, y0) < 2e-2 and cos(emb, y0) > 0.999, (arch, rel(emb, y0), cos(emb, y0))
    net.plan.view(net.d_embeds, (n, cfg.output_dim)).copy_(seed)
    it.run_range("vit_bwd", "vit_end")
    gp = Interp._unpatchify(net.plan.view(net.d_patches, (n, G2, kp)).float(), P, R)
    assert rel(gp, g0) < 4e-2 and cos(gp, g0) > 0.999, (arch, rel(gp, g0), cos(gp, g0))
    codes = {(pplan.OP["QGELU_FWD"], 1 if cfg.act == "gelu" else 0), (pplan.OP["CONV"], 8 if cfg.act == "gelu" else 4)}
    assert codes <= {(op.code, op.flags) for op in net.plan.ops}, arch
    for op in net.plan.ops:
        if op.code == pplan.OP["CONV"] and op.flags & 8:
            assert op.i[16] >= 64 and op.i[17] == 1 and op.i[23] == 0, list(op.i)


def test_exact_gelu_backward_needs_the_wgmma_kernels():
    cfg, _ = reduced("ViT-B-32", layers=1)
    sd = seeded_sd(cfg)
    with pytest.raises(NotImplementedError, match="conv_impl=1"):
        pv.ViTB200(cfg, sd, n_images=3, device="cpu", conv_impl=1)
    pv.ViTB200(cfg, sd, n_images=3, device="cpu", conv_impl=1, build_backward=False)  # the forward alone builds
    mp = pytest.MonkeyPatch()
    mp.setenv("CGD_QGELU_EPI", "0")  # the QuickGELU A/B switch: the exact GELU has no other backward and ignores it
    try:
        net = pv.ViTB200(cfg, sd, n_images=3, device="cpu")
    finally:
        mp.undo()
    assert any(op.code == pplan.OP["CONV"] and op.flags & 8 for op in net.plan.ops)


TEXT_ARCHS = ["ViT-B-32", "ViT-B-32-quickgelu", "ViT-L-14", "ViT-H-14"]


def _text_case(arch):
    _, tcfg = reduced(arch)
    sd = pw.seeded_state_dict(pw.text_param_shapes(tcfg), 7)
    g = th.Generator().manual_seed(4)
    ids = th.randint(1, 400, (3, tcfg.context_length), generator=g)
    ids[:, 9:] = 0
    ids[th.arange(3), th.tensor([5, 8, 3])] = tcfg.vocab_size - 1  # the end-of-text token: the largest id of each sequence
    return tcfg, sd, ids, encode_text(sd, ids, tcfg.act)


@pytest.mark.parametrize("arch", TEXT_ARCHS)
def test_text_oracle_matches_transformers(arch):
    pytest.importorskip("transformers")
    tcfg, sd, ids, ref = _text_case(arch)
    with th.no_grad():
        hf = hf_text_model(sd, tcfg)(input_ids=ids).text_embeds
    assert float((ref - hf).abs().max() / hf.abs().max()) < 2e-5, arch


@pytest.mark.parametrize("arch", TEXT_ARCHS)
def test_text_plan_matches_the_oracle(arch):
    tcfg, sd, ids, ref = _text_case(arch)
    assert ptx.text_config_from_state_dict(sd, act=tcfg.act) == tcfg
    tower = ptx.TextB200(tcfg, sd, 3, device="cpu")
    rows = th.arange(3) * tcfg.context_length + ids.argmax(dim=-1)
    tower.plan.view(tower.ids).copy_(ids.reshape(-1).to(th.int32))
    tower.plan.view(tower.eot_rows).copy_(rows.to(th.int32))
    OpenClipInterp(tower.plan).run()
    emb = tower.plan.view(tower.embeds, (3, tcfg.output_dim))
    assert rel(emb, ref) < 2e-2 and cos(emb, ref) > 0.999, (arch, rel(emb, ref))
    assert (pplan.OP["QGELU_FWD"], 1 if tcfg.act == "gelu" else 0) in {(op.code, op.flags) for op in tower.plan.ops}


# ---------------------------------------------------------------------- ViT-H's padded heads
def test_vit_h_heads_are_zero_padded_to_128():
    cfg, _ = reduced("ViT-H-14", layers=1)
    assert (cfg.heads, cfg.head_width, cfg.head_pad) == (16, 80, 128)
    sd = seeded_sd(cfg)
    net = pv.ViTB200(cfg, sd, n_images=1, device="cpu", build_backward=True)
    pre = "transformer.resblocks.0"
    w_in = net.plan.view(net._wcache[pre + ".in_proj"].fwd).view(-1, cfg.width).float()
    b_in = net.plan.view(net._wcache[pre + ".in_proj"].bias).float()
    w_out = net.plan.view(net._wcache[pre + ".out_proj"].fwd).view(-1, 16 * 128).float()
    assert w_in.shape[0] == 3 * 16 * 128 and w_out.shape == (1280, 16 * 128)
    src_w = sd[f"visual.{pre}.attn.in_proj_weight"].view(3, 16, 80, 1280)
    src_b = sd[f"visual.{pre}.attn.in_proj_bias"].view(3, 16, 80)
    wi, bi = w_in.view(3, 16, 128, 1280), b_in.view(3, 16, 128)
    assert th.equal(wi[:, :, :80], src_w.half().float()) and not wi[:, :, 80:].any()
    assert th.equal(bi[:, :, :80], src_b) and not bi[:, :, 80:].any()
    wo = w_out.view(1280, 16, 128)
    assert th.equal(wo[:, :, :80], sd[f"visual.{pre}.attn.out_proj.weight"].view(1280, 16, 80).half().float()) and not wo[:, :, 80:].any()
    # the dgrad orientation of out_proj: its padded rows are zero too, so d a's padded columns are exactly zero
    wb = net.plan.view(net._wcache[pre + ".out_proj"].bwd).view(16 * 128, 1280).float()
    assert not wb.view(16, 128, 1280)[:, 80:].any()
    attn = [op for op in net.plan.ops if op.code in (pplan.OP["ATTN_FWD"], pplan.OP["ATTN_BWD"])]
    assert len(attn) == 2 and all(op.i[1] == 16 and op.i[3] == 128 and op.f[0] == 1.0 / math.sqrt(80) for op in attn)


def test_openai_vit_packing_and_attention_are_unchanged():
    cfg = pv.VIT_CONFIGS["ViT-B/32"]
    assert (cfg.head_width, cfg.head_pad, cfg.act, cfg.heads) == (64, 64, "quick_gelu", 12)
    assert pv.ViTConfig(224, 32, 768, 12, 512) == cfg and ptx.TextConfig().act == "quick_gelu"


# ---------------------------------------------------------------------- names, files and refusals
@pytest.fixture
def no_files(monkeypatch):
    """every way a checkpoint could be opened raises: a refusal must come first"""
    def opened(*a, **k):
        raise AssertionError(f"a file was opened: {a[:1]}")
    for name in ("_load_open_clip_sd", "_load_clip_sd", "_load_clip_file", "_load_unet_sd"):
        monkeypatch.setattr(cgd, name, opened)
    monkeypatch.setattr(cgd.th, "load", opened)
    monkeypatch.setattr(cgd, "_require_cuda", lambda device: None)


def test_names_resolve_to_the_registry():
    assert cgd.open_clip_arch("open_clip:ViT-H-14") == "ViT-H-14" and cgd.open_clip_arch("ViT-B/32") is None
    assert cgd.open_clip_arch("ViT-B-32.pt") is None
    with pytest.raises(ValueError, match="ViT-g-14"):
        cgd.open_clip_arch("open_clip:ViT-g-14")
    cfg, tcfg = reduced("ViT-B-32")
    sd = seeded_sd(pv.OPEN_CLIP_CONFIGS["ViT-B-32"].vision)
    got_sd, got = cgd._clip_tower("open_clip:ViT-B-32", sd, None)
    assert got_sd is sd and got == pv.OPEN_CLIP_CONFIGS["ViT-B-32"].vision and got.act == "gelu"
    # the same weights under the OpenAI name run QuickGELU: the name, not the keys, picks the semantics
    assert cgd._clip_tower("ViT-B/32", sd, None)[1].act == "quick_gelu"


def test_checkpoint_lookup_order(tmp_path, monkeypatch):
    monkeypatch.setattr(cgd, "CACHE_PATH", str(tmp_path / "cache"))
    places = cgd.open_clip_checkpoint_paths("ViT-B-32", str(tmp_path / "ckpt"))
    assert places == [str(tmp_path / d / "open_clip" / f"ViT-B-32{s}") for d in ("ckpt", "cache") for s in (".safetensors", ".bin", ".pt")]
    with pytest.raises(FileNotFoundError) as e:
        cgd._load_open_clip_sd("ViT-B-32", str(tmp_path / "ckpt"))
    assert all(p in str(e.value) for p in places)
    sd = seeded_sd(pv.OPEN_CLIP_CONFIGS["ViT-B-32"].vision)
    os.makedirs(tmp_path / "cache" / "open_clip")
    th.save(sd, tmp_path / "cache" / "open_clip" / "ViT-B-32.bin")
    from safetensors.torch import save_file
    os.makedirs(tmp_path / "ckpt" / "open_clip")
    marked = dict(sd, **{"visual.ln_pre.bias": th.full_like(sd["visual.ln_pre.bias"], 3.0)})
    save_file({k: v.contiguous() for k, v in marked.items()}, str(tmp_path / "ckpt" / "open_clip" / "ViT-B-32.safetensors"))
    got, cfg = cgd._clip_tower("open_clip:ViT-B-32", None, str(tmp_path / "ckpt"))
    assert float(got["visual.ln_pre.bias"][0]) == 3.0 and cfg.act == "gelu"
    os.remove(tmp_path / "ckpt" / "open_clip" / "ViT-B-32.safetensors")
    got, _ = cgd._clip_tower("open_clip:ViT-B-32", None, str(tmp_path / "ckpt"))
    assert th.equal(got["visual.ln_pre.bias"], sd["visual.ln_pre.bias"])


@pytest.mark.parametrize("key,shape", [
    ("visual.conv1.weight", (768, 3, 16, 16)), ("visual.positional_embedding", (197, 768)),
    ("visual.transformer.resblocks.3.attn.in_proj_weight", (3 * 768, 768)), ("visual.transformer.resblocks.0.mlp.c_fc.weight", (2048, 1280)),
    ("visual.transformer.resblocks.5.mlp.c_proj.weight", (1280, 2048)), ("visual.proj", (1280, 768)),
    ("text_projection", (1024, 768)), ("transformer.resblocks.2.mlp.c_fc.weight", (4096, 1280)), ("token_embedding.weight", (49408, 768)),
])
def test_shape_mismatch_names_the_key(key, shape):
    v, t = pv.OPEN_CLIP_CONFIGS["ViT-H-14"]
    shapes = {**pw.vit_param_shapes(v), **pw.text_param_shapes(t), key: shape}
    sd = {k: types.SimpleNamespace(shape=s) for k, s in shapes.items()}  # shapes only: the check reads nothing else
    with pytest.raises(ValueError, match=key.replace(".", r"\.")):
        pv.check_open_clip_state_dict("ViT-H-14", sd, text=True)


def test_layer_count_and_missing_keys_are_refused():
    v, t = pv.OPEN_CLIP_CONFIGS["ViT-L-14"]
    sd = {k: types.SimpleNamespace(shape=s) for k, s in {**pw.vit_param_shapes(v), **pw.text_param_shapes(t)}.items()}
    pv.check_open_clip_state_dict("ViT-L-14", sd, text=True)
    short = {k: s for k, s in sd.items() if not k.startswith("visual.transformer.resblocks.23.")}
    with pytest.raises(ValueError, match="23 layers"):
        pv.check_open_clip_state_dict("ViT-L-14", short)
    with pytest.raises(ValueError, match="'visual.proj'"):
        pv.check_open_clip_state_dict("ViT-L-14", {k: s for k, s in sd.items() if k != "visual.proj"})
    # the ViT-B/32 OpenAI layout is not ViT-L-14's
    b32 = {k: types.SimpleNamespace(shape=s) for k, s in pw.vit_param_shapes(pv.VIT_CONFIGS["ViT-B/32"]).items()}
    with pytest.raises(ValueError, match="visual.conv1.weight"):
        pv.check_open_clip_state_dict("ViT-L-14", b32)


def _run(**kw):
    args = dict(prompts=["a lighthouse"], clip_model_name="open_clip:ViT-B-32", image_size=64, checkpoints_dir="/nonexistent",
                prefix_path="/nonexistent/out")
    args.update(kw)
    return next(cgd.clip_guided_diffusion(**args))


def test_text_encoder_clip_is_refused_for_open_clip_before_any_file(no_files):
    with pytest.raises(ValueError, match="text_encoder='clip'"):
        _run(text_encoder="clip")
    with pytest.raises(ValueError, match="text_encoder='clip'"):
        _run(text_encoder="clip", clip_model_name=["ViT-B/32", "open_clip:ViT-H-14"])
    with pytest.raises(ValueError, match="not supported"):
        _run(clip_model_name=["ViT-B/32", "open_clip:ViT-bigG-14"])


def test_unknown_arch_is_refused_before_any_file(no_files):
    from clip_guided_diffusion_b200 import clip_model
    monkey = pytest.MonkeyPatch()
    monkey.setattr(clip_model, "_require_cuda", lambda d: None)
    try:
        with pytest.raises(ValueError, match="not supported"):
            clip_model.load_clip("open_clip:ViT-g-14", "cpu")
        with pytest.raises(ValueError, match="not supported"):
            cgd.encode_image_prompt("x.png", 1.0, 64, 4, "open_clip:RN50", "cpu")
        with pytest.raises(ValueError, match="not supported"):
            cgd.encode_text_prompt("a cat", 1.0, "open_clip:ViT-B-32-xyz", "cpu")
    finally:
        monkey.undo()


def test_text_encoder_rules_pick_the_device_tower(monkeypatch, tmp_path):
    """open_clip towers encode on the device tower whatever text_encoder says ("auto" with the clip package importable too); an OpenAI
    tower of the same ensemble keeps the clip package; the engine is never built (stopped right after the prompts)"""
    vocab = tmp_path / "bpe_simple_vocab_16e6.txt.gz"
    vocab.write_bytes(b"")
    calls = []

    class Stop(Exception):
        pass

    monkeypatch.setattr(cgd, "_require_cuda", lambda device: None)
    monkeypatch.setattr(cgd, "_clip_importable", lambda: True)
    monkeypatch.setattr(cgd, "_clip_tower", lambda n, sd, d: ({"name": n}, pv.OPEN_CLIP_CONFIGS["ViT-H-14"].vision if "open_clip" in n
                                                                  else pv.VIT_CONFIGS["ViT-B/32"]))
    monkeypatch.setattr(cgd, "_encode_text_device", lambda p, sd, v, dev, act="quick_gelu": calls.append(("device", sd["name"], v, act))
                        or (th.zeros(1, 4), th.ones(1)))
    monkeypatch.setattr(cgd, "_encode_text", lambda p, n, dev: calls.append(("clip", n)) or (th.zeros(1, 4), th.ones(1)))
    monkeypatch.setattr(cgd, "config_for", lambda *a, **k: (_ for _ in ()).throw(Stop()))
    with pytest.raises(Stop):
        _run(clip_model_name=["ViT-B/32", "open_clip:ViT-H-14"], bpe_path=str(vocab), prefix_path=str(tmp_path / "out"), unet_state_dict={},
             device="cpu")
    assert calls == [("clip", "ViT-B/32"), ("device", "open_clip:ViT-H-14", str(vocab), "gelu")]
    calls.clear()
    with pytest.raises(FileNotFoundError, match="bpe"):
        _run(clip_model_name="open_clip:ViT-B-32", prefix_path=str(tmp_path / "out"), checkpoints_dir=str(tmp_path / "none"))
    assert not calls


# ---------------------------------------------------------------------- plan fingerprints of the OpenAI towers
def test_plan_fingerprints_are_unchanged():
    """scripts/plan_fingerprint.py prints the table it printed before the OpenCLIP towers existed (tests/golden/plan_fingerprint.txt)"""
    with open(os.path.join(ROOT, "tests", "golden", "plan_fingerprint.txt")) as f:
        want = f.read()
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "plan_fingerprint.py")], capture_output=True, text=True, cwd=ROOT,
                         check=True).stdout
    assert out == want


# ---------------------------------------------------------------------- launch ownership of the new plans
def test_every_launch_of_the_open_clip_plans_has_an_owner():
    from scripts.open_clip_signatures import collect, expected, owners
    from tests.open_clip_plan_table import OPEN_CLIP_CONV_PLAN, OPEN_CLIP_OP_PLAN, OPEN_CLIP_OTHER_PLAN
    conv, other, table, _ = collect()
    own_conv, own_other, own_table = owners()
    missing = [("CONV", s) for s in conv - own_conv - set(OPEN_CLIP_CONV_PLAN)] + \
        [("other", s) for s in other - own_other - set(OPEN_CLIP_OTHER_PLAN)] + [("table", s) for s in table - own_table - set(OPEN_CLIP_OP_PLAN)]
    assert not missing, "launches no GPU case runs (regenerate tests/open_clip_plan_table.py with scripts/open_clip_signatures.py):\n" + \
        "\n".join(map(repr, missing))
    with open(os.path.join(ROOT, "tests", "open_clip_plan_table.py")) as f:
        assert f.read() == expected(), "stale rows: run scripts/open_clip_signatures.py"
    flags = {s[10] for s in OPEN_CLIP_CONV_PLAN}
    assert 8 in flags, "no CONV flags 8 row: the collector went blind to the exact-GELU epilogue"
