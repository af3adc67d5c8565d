"""CPU: image prompts (``image_prompts=``, cgd/clip_util.py:90-101 as intended; quirk B5) -- the oracle encoder against what the
reference's own ResizeRight and MakeCutouts produced (tests/golden/image_prompt_golden.npz), the host tables of any tap count, the
entry's orchestration on the plan interpreter (prompt order, weights, P, the CPU generator), and the argument checks of RESIZE_AXIS."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch as th

from clip_guided_diffusion_b200 import cgd
from clip_guided_diffusion_b200 import guidance as pg
from clip_guided_diffusion_b200 import image_prompt as pip
from clip_guided_diffusion_b200 import resize_right as rr
from clip_guided_diffusion_b200 import unet as pu
from clip_guided_diffusion_b200 import vit as pv
from clip_guided_diffusion_b200 import weights as pw
from oracle import resize_right as orr
from oracle.clip_vit import CLIPVisualOnly, ViTConfig as OViTConfig
from tests import image_prompt_oracle as oip
from tests.plan_interp import Interp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "image_prompt_golden.npz"))
CASES = ("landscape", "portrait", "heavy", "small")


def _case(name):
    H, W, image_size, cut_size, cutn, seed = (int(v) for v in GOLD[name + "_cfg"])
    x = th.from_numpy(GOLD[name + "_image"]).permute(2, 0, 1).unsqueeze(0).float().div(255)
    return x, image_size, cut_size, cutn, seed


@pytest.mark.parametrize("name", CASES)
def test_oracle_encoder_reproduces_the_reference_pieces(name):
    """resized image (1e-5 of max), windows and generator state (exact), pooled cutouts -- against the reference's ResizeRight.resize
    and cgd.modules.MakeCutouts under manual_seed; the product's resized shape rule agrees with torchvision's"""
    x, image_size, cut_size, cutn, seed = _case(name)
    ref = th.from_numpy(GOLD[name + "_resized"])
    assert pip.resized_shape(x.shape[2], x.shape[3], image_size) == tuple(ref.shape[2:]) == oip.resized_shape(x.shape[2], x.shape[3], image_size)
    th.manual_seed(seed)
    emb, w, ex = oip.encode_image_prompt(x, 0.5, image_size, cutn, lambda t: t.flatten(1)[:, :8], cut_size)
    assert ex["image"].shape == ref.shape
    assert float((ex["image"] - ref).abs().max()) <= 1e-5 * float(ref.abs().max())
    assert [list(c) for c in ex["coords"]] == GOLD[name + "_coords"].tolist()
    assert th.equal(th.get_rng_state(), th.from_numpy(GOLD[name + "_rng"]))
    cuts = th.from_numpy(GOLD[name + "_cutouts"])
    assert float((ex["cutouts"] - cuts).abs().max()) <= 1e-5 * float(cuts.abs().max())
    assert w == [0.5 / cutn] * cutn and emb.shape == (cutn, 8)
    if name == "portrait":  # quirk B3: x offsets drawn over the height, windows clipped at the right border
        assert any(ox + s > ref.shape[3] for ox, _, s in ex["coords"])
    if name == "small":  # smaller than image_size: the identity
        assert th.equal(ex["image"], x)


def _dense(left, w, T, S):
    """tables -> the [O, S] matrix they apply (taps outside [0, S) read zeros)"""
    O = left.shape[0]
    M = th.zeros(O, S, dtype=th.float64)
    for o in range(O):
        for i in range(T):
            j = int(left[o]) + i
            if 0 <= j < S:
                M[o, j] += float(w[o, i])
    return M


@pytest.mark.parametrize("S,O", [(240, 85), (180, 64), (2000, 64), (4000, 64), (1024, 256), (100, 64)])
def test_uncapped_tables_match_the_oracle_resampler(S, O):
    """tables(S, O, t_max=None) for any tap count: [O, T] weights whose matrix is the oracle's resize of the identity"""
    left, w, T = rr.tables(S, O, t_max=None)
    assert w.shape == (O, T) and left.dtype == th.int32 and T == int(np.ceil(6 * S / O - 1e-6))
    ref = orr._resize_dim(th.eye(S), 0, O).double()
    assert float((_dense(left, w, T, S) - ref).abs().max()) < 1e-6


def test_cutout_tables_are_unchanged():
    """the ResizeRight cutout mode's tables keep their T_MAX = 16 layout, values (sha256 of the parent's tables) and error"""
    known = {(237, 224): (7, "c51c208a8c19ba78"), (64, 56): (7, "9982258d1ae734db"), (32, 32): (1, "9e7840fdd605423b"),
             (16, 56): (6, "552eaba670f8aa05"), (256, 224): (7, "92945b67fe8aac6d"), (80, 32): (15, "2475aae1e127e730")}
    for (S, O), (T, digest) in known.items():
        left, w, t = rr.tables(S, O)
        assert t == T and w.shape == (O, rr.T_MAX) == (O, 16)
        assert hashlib.sha256(left.numpy().tobytes() + w.numpy().tobytes()).hexdigest()[:16] == digest
        l2, w2, t2 = rr.tables(S, O, t_max=None)
        assert t2 == T and th.equal(l2, left) and th.equal(w2, w[:, :w2.shape[1]])
    with pytest.raises(ValueError, match=r"resize 90 -> 32: 17 taps exceed the device tables \(16\); scale factors below 0.4 are unsupported"):
        rr.tables(90, 32)


# ---------------------------------------------------------------- the entry on the interpreter
VCFG = pv.ViTConfig(32, 16, 64, 1, 32)  # a one-layer CLIP tower (as tests/test_entry_cpu.py)


class _RecordingEngine(pg.GuidedStepB200):
    seen = []

    def __init__(self, *a, **k):
        k["device"] = "cpu"
        self.seen.append({"P": k["max_prompts"], "rng": th.get_rng_state()})
        super().__init__(*a, **k)
        it = Interp(self.plan)
        self.plan.run_range = lambda a, b, stream=None: it.run_range(a, b)
        self.plan.run = lambda first=0, count=None, stream=None: it.run(first, len(self.plan.ops) - first if count is None else count)

    def set_targets(self, target_embeds, weights):
        self.seen[-1].update(targets=target_embeds.clone(), weights=weights.clone())
        super().set_targets(target_embeds, weights)


def _oracle_tower(vsd):
    m = CLIPVisualOnly(OViTConfig(32, 16, 64, 1, 32)).eval()
    m.load_state_dict(vsd)
    return m.encode_image


class _OracleEncoder:
    """stand-in for cgd.ImagePromptEncoder (the device encoder): the fp32 oracle with the same tower weights"""
    built = 0

    def __init__(self, tower_cfg, clip_sd, num_cutouts, device="cuda"):
        type(self).built += 1
        self.cfg, self.cutn, self.tower = tower_cfg, num_cutouts, _oracle_tower(clip_sd)

    def encode(self, image, weight, diffusion_size):
        emb, w, _ = oip.encode_image_prompt(oip.load_image(image), weight, diffusion_size, self.cutn, self.tower, self.cfg.input_resolution)
        return emb, w


@pytest.fixture
def entry(tmp_path, monkeypatch):
    monkeypatch.setattr(cgd, "_require_cuda", lambda device: None)
    monkeypatch.setattr(cgd, "GuidedStepB200", _RecordingEngine)
    monkeypatch.setattr(cgd, "ImagePromptEncoder", _OracleEncoder)
    monkeypatch.chdir(tmp_path)
    _RecordingEngine.seen.clear()
    _OracleEncoder.built = 0
    ucfg = pu.config_for(64, True)
    usd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234)
    vsd = pw.seeded_state_dict(pw.vit_param_shapes(VCFG), 1235)
    a = oip.write_png(tmp_path / "a.png", 80, 120, seed=1)   # landscape, downscaled to 64 x 96
    b = oip.write_png(tmp_path / "b.png", 50, 40, seed=2)    # portrait, smaller than image_size: identity
    return dict(usd=usd, vsd=vsd, paths=(str(tmp_path / "a.png"), str(tmp_path / "b.png")), images=(a, b), tmp=tmp_path)


def _run(e, **kw):
    args = dict(image_size=64, num_cutouts=4, batch_size=1, timestep_respacing="25", skip_timesteps=24, save_frequency=1,
                prefix_path=e["tmp"] / "out", progress=False, seed=3, device="cpu", unet_state_dict=e["usd"], clip_state_dict=e["vsd"])
    args.update(kw)
    return list(cgd.clip_guided_diffusion(**args))


def _expected(e, paths_weights, seed=3, cutn=4, text=None):
    """the reference's sequence: manual_seed, text prompts, each image prompt's cutouts (oracle), weights / |sum|"""
    th.manual_seed(seed)
    tower = _oracle_tower(e["vsd"])
    embeds, weights = ([text[0]], list(text[1])) if text else ([], [])
    for path, w in paths_weights:
        emb, ws, _ = oip.encode_image_prompt(oip.load_image(path), w, 64, cutn, tower, VCFG.input_resolution)
        embeds.append(emb)
        weights += ws
    wt = th.tensor(weights)
    return th.cat(embeds), wt / wt.sum().abs(), th.get_rng_state()


def test_entry_with_image_prompts_only(entry, monkeypatch):
    """no text prompt: the `clip` package is never needed; P = cutn * images; order and weights of the reference; the CPU generator
    is where the reference's set-up leaves it when the engine is built (so the loop's windows match)"""
    def no_text(*a, **k):
        raise AssertionError("an image-only run must not load the text tower")
    monkeypatch.setattr(cgd, "_encode_text", no_text)
    pa, pb = entry["paths"]
    got = _run(entry, prompts=[], image_prompts=[f"{pa}:2", f"{pb}:-0.5"])
    assert len(got) == 1 and os.path.exists(got[0][1])
    tgt, wts, rng = _expected(entry, [(pa, 2.0), (pb, -0.5)])
    seen = _RecordingEngine.seen[-1]
    assert seen["P"] == 8 and _OracleEncoder.built == 1
    assert th.allclose(seen["targets"], tgt, rtol=0, atol=1e-6)
    assert th.allclose(seen["weights"], wts, rtol=0, atol=1e-7)
    assert th.allclose(wts, th.tensor([2.0 / 4] * 4 + [-0.5 / 4] * 4) / 1.5)
    assert th.equal(seen["rng"], rng)


def test_entry_with_text_and_image_prompts(entry, monkeypatch):
    """text embeddings first, then each image prompt's cutn embeddings; weights [text..., w / cutn * cutn] normalised together"""
    text = th.randn(2, 32, generator=th.Generator().manual_seed(9))
    monkeypatch.setattr(cgd, "_encode_text", lambda prompts, name, device: (text[:len(prompts)].clone(), th.tensor([1.0, 3.0][:len(prompts)])))
    pa, _ = entry["paths"]
    _run(entry, prompts=["a", "b"], image_prompts=[pa + ":4"], num_cutouts=2)
    tgt, wts, rng = _expected(entry, [(pa, 4.0)], cutn=2, text=(text, [1.0, 3.0]))
    seen = _RecordingEngine.seen[-1]
    assert seen["P"] == 4 and th.equal(seen["targets"][:2], text)
    assert th.allclose(seen["targets"], tgt, rtol=0, atol=1e-6)
    assert th.allclose(seen["weights"], th.tensor([1.0, 3.0, 2.0, 2.0]) / 8.0, rtol=0, atol=1e-7)
    assert th.equal(seen["rng"], rng)


def test_entry_refuses_urls_and_target_embeds_with_image_prompts(entry):
    with pytest.raises(ValueError, match="URLs are not fetched"):
        _run(entry, image_prompts=["https://example.com/x.png:0.5"])
    with pytest.raises(ValueError, match="URLs are not fetched"):
        pip.load_image("http://example.com/x.png")
    with pytest.raises(NotImplementedError, match="encode_image_prompt"):  # before any file is opened
        _run(entry, image_prompts=["does-not-exist.png"], target_embeds=th.zeros(1, 32), weights=[1.0])
    assert _OracleEncoder.built == 0 and not _RecordingEngine.seen


RESIZE_CHILD = r"""
import ctypes, sys
sys.path.insert(0, sys.argv[1])
from clip_guided_diffusion_b200 import _lib
lib = _lib.load()
good = 1 << 40
base = dict(i=[3, 300, 400, 1, 64, 38], p=[good, good + 4096, good + 8192, good + 12288])
n, zero = 0, []
for axis in (0, 1):
    cases = [("i", j, v) for j in range(6) for v in (0, -1, (1 << 31), 1 << 40, -(1 << 40)) if (j, v) != (3, 0)]  # axis 0 is valid
    cases += [("i", 3, v) for v in (2, 7)]
    cases += [("p", j, 0) for j in range(4)] + [("ok", 0, 0)]
    for w, j, v in cases:
        op = _lib.CgdOp()
        op.code = _lib.OP["RESIZE_AXIS"]
        vals = list(base["i"]); vals[3] = axis
        if w == "i":
            vals[j] = v
        for k, x in enumerate(vals):
            op.i[k] = x
        for k, x in enumerate(base["p"]):
            op.p[k] = 0 if (w == "p" and k == j) else x
        rc = lib.cgd_run_op(ctypes.byref(op), None)
        n += 1
        msg = lib.cgd_last_error().decode()
        print("CASE", w, j, v, rc, msg, flush=True)
        if rc == 0:
            zero.append((w, j, v))
print("DONE", n, zero, flush=True)
"""


@pytest.mark.skipif(th.cuda.is_available(), reason="needs a box WITHOUT a GPU: only the argument checks may run")
def test_resize_axis_rejects_malformed_operands_without_a_device():
    """null pointers, dims <= 0 or >= 2^31, T <= 0, an axis outside {0, 1}: a negative return before any CUDA call; a well-formed op
    reaches the launch, which fails for lack of a device (positive cudaError_t) -- never 0, never a crash or hang"""
    r = subprocess.run([sys.executable, "-c", RESIZE_CHILD, ROOT], capture_output=True, text=True, timeout=120)
    lines = r.stdout.splitlines()
    assert r.returncode == 0 and lines and lines[-1].startswith("DONE"), r.stderr[-400:]
    assert lines[-1] == f"DONE {2 * (29 + 2 + 4 + 1)} []", lines[-1]
    for l in lines[:-1]:
        _, w, j, v, rc, *msg = l.split(" ")
        if w == "ok":
            assert int(rc) > 0, l  # no device: the launch itself fails
        else:
            assert int(rc) == -1 and "resize_axis" in " ".join(msg), l
