"""CPU: CLIP visual towers under torch.autograd (clip_model.py, load_clip), interpreted op by op (tests/clip_autograd_interp.py).

encode_image's forward and input gradient against the oracle towers' autograd (a tiny ViT and a tiny ModifiedResNet, full and padded
calls), CLIP_SEED's rule against a float64 restatement, the guards, load_clip's name / path / state_dict resolution, the oracle's cond_fn
on load_clip's model driving the package's *_with_grad steps, malformed new ops and the launch coverage of load_clip's plans."""
from __future__ import annotations

import json
import math
import subprocess
import sys
import textwrap
import types

import pytest
import torch as th

from clip_guided_diffusion_b200 import clip_model as cm
from clip_guided_diffusion_b200 import clip_util
from clip_guided_diffusion_b200 import gaussian_diffusion as pgd
from clip_guided_diffusion_b200 import rn as prn
from clip_guided_diffusion_b200 import vit as pv
from clip_guided_diffusion_b200 import weights as pw
from oracle import clip_rn as orn
from oracle import diffusion as od
from oracle.clip_vit import CLIPVisualOnly, ViTConfig as OViTConfig
from oracle.unet import seeded_init_
from tests.clip_autograd_interp import ClipInterp, clip_seed_scale, interpreted
from tests.step_parity import cos, rel
from tests.test_autograd_cpu import _check, _cond, _oracle_step, inputs, tiny

ROOT = __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__)))


def tiny_tower(kind):
    """(package config, state_dict, fp32 oracle with .encode_image) of a tiny ViT (32 px, patch 16) or a tiny ModifiedResNet (64 px)"""
    if kind == "vit":
        oracle = seeded_init_(CLIPVisualOnly(OViTConfig(32, 16, 128, 2, 64)), seed=5).eval()
        return pv.ViTConfig(32, 16, 128, 2, 64), oracle.state_dict(), oracle
    cfg = prn.RNConfig(layers=(1, 2, 1, 1), output_dim=128, input_resolution=64, width=64)
    sd = pw.seeded_rn_state_dict(cfg, seed=3)
    oracle = orn.CLIPVisualRN(orn.RNConfig(layers=(1, 2, 1, 1), output_dim=128, input_resolution=64, width=64)).eval()
    oracle.load_state_dict(sd, strict=False)
    return cfg, sd, oracle


def tiny_model(kind, max_images=4):
    cfg, sd, oracle = tiny_tower(kind)
    for prm in oracle.parameters():
        prm.requires_grad_(False)
    return interpreted(cm.ClipModelB200(cfg, sd, max_images, device="cpu")), oracle, cfg


def images(n, R, seed=0):
    return th.randn(n, 3, R, R, generator=th.Generator().manual_seed(seed))


# ---------------------------------------------------------------------- tiny towers vs the oracle
@pytest.mark.parametrize("n", [4, 3], ids=["full", "padded"])
@pytest.mark.parametrize("kind", ["vit", "rn"])
def test_encode_image_matches_oracle_autograd(kind, n):
    model, oracle, cfg = tiny_model(kind)
    R = cfg.input_resolution
    x = images(n, R)
    w = th.randn(n, cfg.output_dim, generator=th.Generator().manual_seed(7))
    xe = x.clone().requires_grad_()
    emb = model.encode_image(xe)
    assert emb.dtype == th.float32 and emb.shape == (n, cfg.output_dim) and emb.grad_fn is not None
    (ge,) = th.autograd.grad((w * emb).sum(), xe)
    xo = x.clone().requires_grad_()
    ref = oracle.encode_image(xo).float()
    (go,) = th.autograd.grad((w * ref).sum(), xo)
    assert rel(emb.detach(), ref.detach()) < 2e-2, rel(emb.detach(), ref.detach())
    assert cos(ge, go) > 0.995 and rel(ge, go) < 5e-2, (cos(ge, go), rel(ge, go))


@pytest.mark.parametrize("kind", ["vit", "rn"])
def test_padded_rows_equal_unpadded_call(kind):
    """a call with 3 images on a 4-image tower gives the rows and gradients of a 3-image tower, up to the order of the interpreter's
    GEMM sums (they block by row count) and the fp16 roundings that follow"""
    padded, _, cfg = tiny_model(kind, max_images=4)
    exact, _, _ = tiny_model(kind, max_images=3)
    x = images(3, cfg.input_resolution, seed=2)
    w = th.randn(3, cfg.output_dim, generator=th.Generator().manual_seed(8))
    out = []
    for m in (padded, exact):
        xe = x.clone().requires_grad_()
        e = m.encode_image(xe)
        out.append((e.detach(), th.autograd.grad((w * e).sum(), xe)[0]))
    assert rel(out[0][0], out[1][0]) < 2e-3 and rel(out[0][1], out[1][1]) < 5e-3, (rel(out[0][0], out[1][0]), rel(out[0][1], out[1][1]))


# ---------------------------------------------------------------------- CLIP_SEED's rule
def seed_scale_f64(d: th.Tensor, band: float) -> list:
    """float64 restatement: m = max |d| over non-NaN entries, inf counted as 3e38; 2^clamp(floor(log2(band / m)), -60, 60); 1 if m == 0"""
    out = []
    for row in d.double().tolist():
        vals = [min(abs(v), 3.0e38) for v in row if not math.isnan(v)]
        m = max(vals, default=0.0)
        out.append(1.0 if m == 0 else 2.0 ** min(max(math.floor(math.log2(band / m)), -60), 60))
    return out


def seed_rows(D=96):
    g = th.Generator().manual_seed(3)
    d = th.randn(8, D, generator=g)
    d[0] = 0                        # all-zero row: scale 1
    d[1, 5] = float("nan")          # NaN dropped from the maximum
    d[2, 7] = float("inf")          # inf saturates: the scale clamps low
    d[3] *= 1e-30                   # clamped at +60
    d[4] *= 1e30                    # clamped at -60
    d[5] *= 3e-9
    d[6] *= 7e7
    return d


def test_clip_seed_rule_matches_float64():
    d = seed_rows()
    for band in (1.0, 1024.0, 32768.0):
        assert clip_seed_scale(d, band).double().tolist() == seed_scale_f64(d, band)
    s = seed_scale_f64(d, 1024.0)
    assert s[0] == 1.0 and s[3] == 2.0 ** 60 and s[4] == 2.0 ** -60


def test_clip_seed_op_interpreted():
    """the op through the interpreter: scaled rows, the scale in dyn, rows n.. zero with scale 1"""
    model, _, cfg = tiny_model("vit", max_images=4)
    it = ClipInterp(model.plan)
    d = seed_rows(cfg.output_dim)[3:7]
    model.plan.view(model.d_in, (4, cfg.output_dim)).copy_(d)
    op = model.plan.ops[model.plan.marks["clip_seed"]]
    op.i[0] = 3
    it.run_range("clip_seed", "clip_unpatchify")
    s = th.tensor(seed_scale_f64(d[:3], cm.CLIP_SEED_BAND) + [1.0])
    assert th.equal(model.plan.view(model.dyn).double(), s)
    got = model.plan.view(model.tower.d_embeds, (4, cfg.output_dim))
    assert th.equal(got[:3], d[:3] * s[:3, None].float()) and th.equal(got[3], th.zeros(cfg.output_dim))


# ---------------------------------------------------------------------- guards
def test_guards():
    model, _, cfg = tiny_model("vit", max_images=4)
    R = cfg.input_resolution
    with pytest.raises(ValueError, match="32, 32"):
        model.encode_image(th.zeros(2, 3, 64, 64))
    with pytest.raises(ValueError, match="32, 32"):
        model.encode_image(th.zeros(2, 4, R, R))
    with pytest.raises(ValueError, match="5 images.*1..4"):
        model.encode_image(th.zeros(5, 3, R, R))
    with pytest.raises(ValueError, match="fp32, fp16 or bf16"):
        model.encode_image(th.zeros(2, 3, R, R, dtype=th.float64))
    x = images(2, R).requires_grad_()
    e = model.encode_image(x)
    model.encode_image(x.detach())  # any later forward overwrites the activations
    with pytest.raises(RuntimeError, match="later encode_image call"):
        th.autograd.grad(e.sum(), x)
    e1, e2 = model.encode_image(x), model.encode_image(x)
    with pytest.raises(RuntimeError, match="Two encode_image calls under one backward"):
        th.autograd.grad((e1 + e2).sum(), x)
    e = model.encode_image(x)
    with pytest.raises(RuntimeError, match="double backward"):
        th.autograd.grad(e.sum(), x, create_graph=True)
    with th.no_grad():
        a = model.encode_image(x)
    b = model.encode_image(x.detach())
    assert a.grad_fn is None and b.grad_fn is None and th.equal(a, b)
    assert a.data_ptr() != model.plan.view(model.tower.embeds).data_ptr()


@pytest.mark.parametrize("dtype", [th.float32, th.float16, th.bfloat16])
def test_gradient_dtype_follows_input_and_repeats(dtype):
    model, _, cfg = tiny_model("vit", max_images=4)
    x = images(3, cfg.input_resolution, seed=4).to(dtype).requires_grad_()
    e = model.encode_image(x)
    assert e.dtype == th.float32
    (g1,) = th.autograd.grad(e.sum(), x, retain_graph=True)
    (g2,) = th.autograd.grad(e.sum(), x)
    assert g1.dtype == dtype and th.equal(g1, g2)
    # the fp32 staging copy is exact: the same images in fp32 give the same embeddings
    assert th.equal(e.detach(), model.encode_image(x.detach().float()))


def test_model_chain_and_visual():
    model, _, cfg = tiny_model("rn")
    assert model.eval().requires_grad_(False).to("cpu") is model
    assert model.visual.input_resolution == 64 and model.visual.output_dim == cfg.output_dim
    assert [p.data_ptr() for p in model.parameters()] == [model.plan.arena.data_ptr()]
    with pytest.raises(RuntimeError, match="load_clip once per device"):
        model.to("cuda")


# ---------------------------------------------------------------------- load_clip
def test_load_clip_resolution(tmp_path, monkeypatch):
    with pytest.raises(RuntimeError, match="CUDA"):
        clip_util.load_clip("ViT-B/32", "cpu")
    monkeypatch.setattr(cm, "_require_cuda", lambda device: None)  # the CPU build of the same plan, interpreted nowhere: shapes only
    cfg, sd, _ = tiny_tower("vit")
    m, size = clip_util.load_clip("ignored", "cpu", clip_state_dict=sd, max_images=2)
    assert size == 32 == m.visual.input_resolution and m.cfg == cfg and m.max_images == 2
    path = tmp_path / "tiny-rn.pt"
    rcfg, rsd, _ = tiny_tower("rn")
    th.save(rsd, path)
    m, size = clip_util.load_clip(str(path), "cpu")
    assert size == 64 and m.cfg == rcfg and m.max_images == 16
    # a tower name: the published architecture, the checkpoint under checkpoints_dir/clip/
    vcfg = pv.VIT_CONFIGS["ViT-B/32"]
    (tmp_path / "clip").mkdir()
    th.save({k: v.half() for k, v in pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 11).items()}, tmp_path / "clip" / "ViT-B-32.pt")
    m, size = clip_util.load_clip("ViT-B/32", "cpu", max_images=1, checkpoints_dir=str(tmp_path))
    assert size == 224 and m.cfg == vcfg
    with pytest.raises(FileNotFoundError, match="ViT-H-14.pt not found"):
        clip_util.load_clip("ViT-H/14", "cpu", checkpoints_dir=str(tmp_path))
    with pytest.raises(ValueError, match="max_images"):
        clip_util.load_clip("ignored", "cpu", clip_state_dict=sd, max_images=0)


# ---------------------------------------------------------------------- end to end: the oracle's cond_fn on load_clip's model
@pytest.mark.parametrize("mode", ["ancestral", "ddim"])
def test_package_steps_with_oracle_cond_fn_on_load_clip_model(mode):
    """the package's p_sample_with_grad / ddim_sample_with_grad, engine.model for the UNet and the interpreted CLIP model for the
    oracle's cond_fn (3 cutouts x batch 2 = 6 images on an 8-image tower), against the all-oracle step"""
    eng, ounet, oclip = tiny()
    model = interpreted(cm.ClipModelB200(pv.ViTConfig(32, 16, 128, 2, 64), oclip.state_dict(), max_images=8, device="cpu"))
    odiff = od.create_gaussian_diffusion(1000, "linear", "25")
    pdiff = pgd.create_gaussian_diffusion(1000, "linear", "25")
    x, _, y, _ = inputs(2, seed=4)
    coords = [(0, 0, 32), (3, 5, 24), (12, 1, 17)]
    o = _oracle_step(ounet, odiff, oclip, mode, x, 14, y, coords, False)
    cond_fn, seen = _cond(odiff, model, coords, 14)
    th.manual_seed(123)
    fn = pdiff.p_sample_with_grad if mode == "ancestral" else pdiff.ddim_sample_with_grad
    e = fn(eng.model, x, th.full((2,), 14, dtype=th.long), clip_denoised=False, cond_fn=cond_fn, model_kwargs={"y": y})
    assert model.forward_generation == 1
    _check(dict(e, g=seen["g"]), o)


# ---------------------------------------------------------------------- malformed new ops
CHILD = textwrap.dedent('''
    import ctypes, json, sys
    sys.path.insert(0, sys.argv[1])
    from clip_guided_diffusion_b200 import _lib
    from tests.plan_interp import CODE
    from tests.test_clip_autograd_cpu import tiny_model
    lib = _lib.load()
    vals = [0, -1, 1, 3, 7, (1 << 31) - 1, 1 << 40, -(1 << 40)]
    n, zero = 0, []
    for kind in ("vit", "rn"):
        plan = tiny_model(kind)[0].plan
        arr = plan.lower(1 << 40)
        for k in range(plan.marks["clip_patchify"], plan.marks["clip_end"]):
            base = arr[k]
            muts = [("i", j, v) for j in range(24) for v in vals if base.i[j] != v]
            muts += [("f", 0, v) for v in (0.0, -1024.0, 3.0, 1e30, float("nan"), float("inf"))]
            muts += [("p", j, v) for j in range(12) for v in (0, 3) if base.p[j]] + [("flags", 0, v) for v in (-1, 1 << 30, 255)]
            for w, j, v in muts:
                o = type(base)()
                ctypes.memmove(ctypes.byref(o), ctypes.byref(base), ctypes.sizeof(base))
                if w == "i":
                    o.i[j] = v
                elif w == "f":
                    o.f[j] = v
                elif w == "p":
                    o.p[j] = 0 if v == 0 else o.p[j] + v
                else:
                    o.flags = v
                print("TRY", CODE[o.code], w, j, v, flush=True)
                n += 1
                if lib.cgd_run_op(ctypes.byref(o), None) == 0:
                    zero.append((CODE[o.code], w, j, v))
    print("DONE", n, json.dumps(zero), flush=True)
''')


@pytest.mark.skipif(th.cuda.is_available(), reason="needs a box WITHOUT a GPU: only the argument checks may run")
def test_malformed_clip_autograd_ops_return_error_codes():
    try:
        r = subprocess.run([sys.executable, "-c", CHILD, ROOT], capture_output=True, text=True, timeout=300)
    except subprocess.TimeoutExpired as e:
        pytest.fail(f"cgd_run_op hung on {[l for l in (e.stdout or b'').decode().splitlines() if l.startswith('TRY')][-1:]}")
    lines = r.stdout.splitlines()
    assert r.returncode == 0 and lines and lines[-1].startswith("DONE"), f"crashed (rc {r.returncode}): {r.stderr[-400:]}"
    _, n, zero = lines[-1].split(" ", 2)
    assert int(n) > 1000 and json.loads(zero) == [], json.loads(zero)[:5]


# ---------------------------------------------------------------------- launch coverage of load_clip's plans
# the sizes the GPU tests and scripts/autograd_step_cost.py build: every published tower at 16 images, four of them at 64
COVERAGE = [(name, 16) for name in (*pv.VIT_CONFIGS, *prn.RN_CONFIGS)] + [(name, 64) for name in ("ViT-B/32", "ViT-B/16", "ViT-L/14", "RN50")]


def published_model(name, max_images, device="cpu", seed=1234):
    cfg = pv.VIT_CONFIGS.get(name) or prn.RN_CONFIGS[name]
    sd = pw.seeded_state_dict(pw.vit_param_shapes(cfg), seed) if name in pv.VIT_CONFIGS else pw.seeded_rn_state_dict(cfg, seed=3)
    return cm.ClipModelB200(cfg, sd, max_images, device), cfg, sd


@pytest.mark.parametrize("name,max_images", COVERAGE, ids=[f"{n}-{m}" for n, m in COVERAGE])
def test_load_clip_plans_make_only_tested_launches(name, max_images):
    from tests import test_gpu_clip_autograd as KA
    from tests import test_gpu_conv_kernels as KC
    from tests import test_gpu_unet_kernels as KU
    from tests.test_conv_coverage_cpu import plan_conv_signatures
    from tests.test_unet_kernel_coverage_cpu import plan_signatures
    th.manual_seed(0)
    plan = published_model(name, max_images)[0].plan
    conv = plan_conv_signatures(plan)
    other = plan_signatures(types.SimpleNamespace(plan=plan))
    assert len(conv) > 3 and any(s[0] == "ATTN_BWD" for s in other)
    missing = sorted((s for s in conv if s not in KC.covered_signatures() | KA.covered_conv_signatures()), key=repr) + \
        sorted((s for s in other if s not in KU.covered_signatures() | KA.covered_other_signatures()), key=repr)
    assert not missing, missing[:8]
