"""CPU: LPIPS(net='vgg') under torch.autograd (lpips.py, LPIPS), interpreted op by op (tests/lpips_autograd_interp.py).

Value and both input gradients against oracle.lpips.LPIPSVgg's autograd (equal batches, either side broadcast, one side requiring grad,
normalize=True), LPIPS_SEED's rule against float64, the guards, one plan per shape, the oracle's cond_fn with LPIPS on the package's
*_with_grad steps, and malformed new ops."""
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
from clip_guided_diffusion_b200 import gaussian_diffusion as pgd
from clip_guided_diffusion_b200 import lpips as pl
from clip_guided_diffusion_b200 import vit as pv
from oracle import diffusion as od
from oracle import guidance as og
from oracle import lpips as ol
from tests.clip_autograd_interp import interpreted as clip_interpreted
from tests.lpips_autograd_interp import LpipsInterp, interpreted, lpips_seed_scale, pair_seed
from tests.step_parity import cos, rel
from tests.test_autograd_cpu import _check, inputs, tiny

ROOT = __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__)))
SD = ol.seeded_state_dict()


def model():
    return interpreted(pl.LPIPS(lpips_state_dict=SD, device="cpu"))


def images(n, H, W, seed):
    return th.rand(n, 3, H, W, generator=th.Generator().manual_seed(seed)) * 2 - 1


def _grads(fn, a, b, need=(True, True)):
    ae, be = a.clone().requires_grad_(need[0]), b.clone().requires_grad_(need[1])
    v = fn(ae, be)
    w = th.arange(1, v.shape[0] + 1, dtype=th.float32).view(-1, 1, 1, 1)  # a different upstream weight per image
    gs = th.autograd.grad((w * v).sum(), [t for t, n in zip((ae, be), need) if n])
    it = iter(gs)
    return v.detach(), [next(it) if n else None for n in need]


# ---------------------------------------------------------------------- value and gradients against the oracle
CASES = [(2, 2, 32, 48), (2, 1, 32, 48), (1, 2, 16, 16), (2, 2, 16, 16)]


@pytest.mark.parametrize("n0,n1,H,W", CASES, ids=[f"{a}x{b}-{h}x{w}" for a, b, h, w in CASES])
def test_value_and_gradients_match_oracle(n0, n1, H, W):
    m, o = model(), ol.LPIPSVgg(SD)
    a, b = images(n0, H, W, 1), images(n1, H, W, 2)
    v, (ga, gb) = _grads(m, a, b)
    vo, (oa, ob) = _grads(o, a, b)
    assert v.dtype == th.float32 and v.shape == (max(n0, n1), 1, 1, 1) and ga.shape == a.shape and gb.shape == b.shape
    assert rel(v, vo) < 1e-2, rel(v, vo)
    for g, go in ((ga, oa), (gb, ob)):
        assert cos(g, go) > 0.995 and rel(g, go) < 0.1, (cos(g, go), rel(g, go))


def test_only_in0_requires_grad_skips_in1_backward():
    m, o = model(), ol.LPIPSVgg(SD)
    a, b = images(2, 32, 48, 3), images(1, 32, 48, 4)
    v, (ga, gb) = _grads(m, a, b, need=(True, False))
    _, (oa, _) = _grads(o, a, b, need=(True, False))
    assert gb is None and cos(ga, oa) > 0.995 and rel(ga, oa) < 0.1
    pp = m.plans[(32, 48, 2, 1)]
    assert pp.ran == ["lp_fwd0", "lp_seed", "lp_seed0", "lp_bwd0"]  # no lp_bwd1, and the seeds of in0 alone
    _, (_, gb) = _grads(m, a, b, need=(False, True))
    assert pp.ran[-3:] == ["lp_seed", "lp_seed1", "lp_bwd1"]


def test_normalize_maps_unit_range():
    m, o = model(), ol.LPIPSVgg(SD)
    a, b = (images(2, 16, 32, 5) + 1) / 2, (images(2, 16, 32, 6) + 1) / 2
    v, (ga, gb) = _grads(lambda x, y: m(x, y, normalize=True), a, b)
    vo, (oa, ob) = _grads(lambda x, y: o(2 * x - 1, 2 * y - 1), a, b)
    assert rel(v, vo) < 1e-2 and cos(ga, oa) > 0.995 and cos(gb, ob) > 0.995


def test_no_grad_records_nothing_and_dtypes_follow_inputs():
    m = model()
    a, b = images(2, 16, 16, 7), images(2, 16, 16, 8)
    with th.no_grad():
        v1 = m(a.requires_grad_(), b)
    v2 = m(a.detach(), b)
    assert v1.grad_fn is None and v2.grad_fn is None and th.equal(v1, v2)
    for dt in (th.float16, th.bfloat16):
        x = a.detach().to(dt).requires_grad_()
        v = m(x, b)
        (g1,) = th.autograd.grad(v.sum(), x, retain_graph=True)
        (g2,) = th.autograd.grad(v.sum(), x)
        assert v.dtype == th.float32 and g1.dtype == dt and th.equal(g1, g2)


# ---------------------------------------------------------------------- LPIPS_SEED's rule and the saturated seed
def seed_f64(d: list, n0: int, n1: int, band: float) -> list:
    def s(ms):
        vals = [min(abs(v), 3.0e38) for v in ms if not math.isnan(v)]
        m = max(vals, default=0.0)
        return 1.0 if m == 0 else 2.0 ** min(max(math.floor(math.log2(band / m)), -60), 60)
    B = len(d)
    return [s([d[r]]) if n == B else s(d) for n in (n0, n1) for r in range(n)]


def test_lpips_seed_rule_matches_float64():
    d = th.tensor([0.0, float("nan"), float("inf"), 1e-30, 1e30, 3e-9, -7e7, 0.37])
    for band in (1.0, 2.0 ** 20, 2.0 ** 30):
        for n0, n1 in ((8, 8), (8, 1), (1, 8)):
            assert lpips_seed_scale(d, n0, n1, band).double().tolist() == seed_f64(d.tolist(), n0, n1, band)
    s = seed_f64(d.tolist(), 8, 8, 2.0 ** 20)
    assert s[0] == 1.0 and s[3] == 2.0 ** 60 and s[4] == 2.0 ** -60 and s[2] == 2.0 ** -60


def test_zero_feature_pixel_seed_saturates_finite():
    g = th.Generator().manual_seed(9)
    f0, f1 = th.rand(2, 4, 64, generator=g), th.rand(2, 4, 64, generator=g)
    f0[0, 1] = 0  # every channel of one pixel is zero after ReLU
    w = th.rand(64, generator=g)
    s = pair_seed(f0, f1, w, th.tensor([2.0 ** 20 / 16, 1.0]))
    assert th.isfinite(s).all() and s[0, 1].abs().max() == 60000
    s = pair_seed(f0, f1, w, th.tensor([float("nan"), 1.0]))
    assert th.isnan(s[0]).all() and th.isfinite(s[1]).all()


# ---------------------------------------------------------------------- guards
def test_guards():
    m = model()
    a = images(2, 16, 16, 10)
    odd = images(2, 24, 16, 0)
    for in0, in1, msg in ((odd, odd, "multiples of 16"), (a, images(3, 16, 16, 0), "one of them 1"), (a, a[:, :2], r"\[N, 3, H, W\]"),
                          (a.double(), a, "fp32, fp16 or bf16"), (a, images(2, 32, 16, 0), "must agree")):
        with pytest.raises(ValueError, match=msg):
            m(in0, in1)
    with pytest.raises(ValueError, match="net='vgg'"):
        pl.LPIPS("alex", lpips_state_dict=SD, device="cpu")
    with pytest.raises(ValueError, match="retPerLayer"):
        m(a, a, retPerLayer=True)
    x = a.clone().requires_grad_()
    v = m(x, a)
    m(x.detach(), a)  # a later forward on the same plan overwrites the activations
    with pytest.raises(RuntimeError, match="later LPIPS call"):
        th.autograd.grad(v.sum(), x)
    v = m(x, a)
    with pytest.raises(RuntimeError, match="double backward"):
        th.autograd.grad(v.sum(), x, create_graph=True)
    assert m.eval().requires_grad_(False).to("cpu") is m
    with pytest.raises(RuntimeError, match="one per device"):
        m.to("cuda")


def test_device_check():
    m = model()
    m.device = th.device("meta")
    with pytest.raises(ValueError, match="the model on meta"):
        m(images(1, 16, 16, 0), images(1, 16, 16, 1))


def test_one_plan_per_shape():
    m = model()
    a = images(2, 16, 16, 11)
    m(a, a[:1])
    p = m.plans[(16, 16, 2, 1)]
    m(a, a[1:])
    assert m.plans[(16, 16, 2, 1)] is p and len(m.plans) == 1
    m(images(1, 32, 16, 0), images(1, 32, 16, 1))
    assert set(m.plans) == {(16, 16, 2, 1), (32, 16, 1, 1)}


# ---------------------------------------------------------------------- the oracle's cond_fn with LPIPS, all three networks on the plans
@pytest.mark.parametrize("mode", ["ancestral", "ddim"])
def test_package_steps_with_oracle_cond_fn_lpips(mode):
    eng, ounet, oclip = tiny()
    clip = clip_interpreted(cm.ClipModelB200(pv.ViTConfig(32, 16, 128, 2, 64), oclip.state_dict(), max_images=8, device="cpu"))
    lp = model()
    odiff = od.create_gaussian_diffusion(1000, "linear", "25")
    pdiff = pgd.create_gaussian_diffusion(1000, "linear", "25")
    x, _, y, _ = inputs(2, seed=4)
    init = images(1, 32, 32, 12)
    coords = [(0, 0, 32), (3, 5, 24), (12, 1, 17)]
    tgt = th.randn(1, 64, generator=th.Generator().manual_seed(99))
    res = []
    for unet, fn_of, cmodel, lmodel in ((eng.model, pdiff, clip, lp), (ounet, odiff, oclip, ol.LPIPSVgg(SD))):
        cf = og.OracleCondFn(odiff, cmodel, tgt, th.ones(1), cut_size=32, num_cutouts=3, lpips_model=lmodel, init_tensor=init, init_scale=1000.0)
        cf.current_timestep = 14
        seen = {}

        def cond_fn(xx, t, out, y=None, cf=cf, seen=seen):
            seen["g"] = cf(xx, t, out, y=y, coords=coords).detach().clone()
            return seen["g"]
        th.manual_seed(123)
        fn = fn_of.p_sample_with_grad if mode == "ancestral" else fn_of.ddim_sample_with_grad
        out = fn(unet, x, th.full((2,), 14, dtype=th.long), clip_denoised=False, cond_fn=cond_fn, model_kwargs={"y": y})
        res.append((dict(out, g=seen["g"]), cf.last_terms["init"]))
    (e, ie), (o, io) = res
    assert abs(ie - io) < 1e-2 * abs(io), (ie, io)
    assert lp.plans[(32, 32, 2, 1)].generation == 1
    _check(e, o)


# ---------------------------------------------------------------------- malformed new ops
CHILD = textwrap.dedent('''
    import ctypes, json, sys
    sys.path.insert(0, sys.argv[1])
    from clip_guided_diffusion_b200 import _lib
    from clip_guided_diffusion_b200 import lpips as pl
    from oracle.lpips import seeded_state_dict
    from tests.plan_interp import CODE
    lib = _lib.load()
    vals = [0, -1, 1, 3, 7, (1 << 31) - 1, 1 << 40, -(1 << 40)]
    n, zero = 0, []
    for key in ((16, 32, 2, 1), (32, 16, 1, 3)):
        plan = pl.LpipsPairPlan({k: v.float() for k, v in seeded_state_dict().items()}, *key, device="cpu").plan
        arr = plan.lower(1 << 40)
        for k in range(plan.marks["lp_tap"], plan.marks["lp_end"]):
            base = arr[k]
            if CODE[base.code] not in ("LPIPS_PAIR_FWD", "LPIPS_LOSS", "LPIPS_SEED", "LPIPS_PAIR_BWD", "PM_TO_NCHW"):
                continue
            muts = [("i", j, v) for j in range(24) for v in vals if base.i[j] != v]
            muts += [("f", j, v) for j in range(5) for v in (0.0, -1024.0, 3.0, 1e30, float("nan"), float("inf"))]
            muts += [("p", j, v) for j in range(12) for v in (0, 3) if base.p[j]] + [("flags", 0, v) for v in (-1, 1 << 30, 255, 0, 4)]
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
def test_malformed_lpips_autograd_ops_return_error_codes():
    try:
        r = subprocess.run([sys.executable, "-c", CHILD, ROOT], capture_output=True, text=True, timeout=600)
    except subprocess.TimeoutExpired as e:
        pytest.fail(f"cgd_run_op hung on {[l for l in (e.stdout or b'').decode().splitlines() if l.startswith('TRY')][-1:]}")
    lines = r.stdout.splitlines()
    assert r.returncode == 0 and lines and lines[-1].startswith("DONE"), f"crashed (rc {r.returncode}): {r.stderr[-400:]}"
    _, n, zero = lines[-1].split(" ", 2)
    assert int(n) > 1000 and json.loads(zero) == [], json.loads(zero)[:5]


# ---------------------------------------------------------------------- launch coverage of LPIPS's plans
# the shapes (H, W, N0, N1) the GPU tests, scripts/autograd_step_cost.py and scripts/lpips_seed_band.py build
COVERAGE = [(s, s, n0, n1) for s in (256, 512) for n0, n1 in ((1, 1), (4, 4), (4, 1), (2, 1))] + [(64, 64, 2, 1)]


def coverage_plan(key):
    """the op list of one shape's plan (not finalized: no arena)"""
    th.manual_seed(0)
    return pl.LpipsPairPlan({k: v.float() for k, v in SD.items()}, *key).plan


@pytest.mark.parametrize("key", COVERAGE, ids=[f"{h}x{w}-{a}x{b}" for h, w, a, b in COVERAGE])
def test_lpips_plans_make_only_tested_launches(key):
    from tests import test_gpu_conv_kernels as KC
    from tests import test_gpu_lpips_autograd as KL
    from tests import test_gpu_unet_kernels as KU
    from tests.test_conv_coverage_cpu import plan_conv_signatures
    from tests.test_unet_kernel_coverage_cpu import plan_signatures
    plan = coverage_plan(key)
    conv = plan_conv_signatures(plan)
    other = plan_signatures(types.SimpleNamespace(plan=plan))
    assert len(conv) >= 13 and any(s[0] == "PM_TO_NCHW" and s[5] & 8 for s in other)
    missing = sorted((s for s in conv if s not in KC.covered_signatures() | KL.covered_conv_signatures()), key=repr) + \
        sorted((s for s in other if s not in KU.covered_signatures() | KL.covered_other_signatures()), key=repr)
    assert not missing, missing[:8]


def test_lpips_plan_table_is_current():
    r = subprocess.run([sys.executable, f"{ROOT}/scripts/lpips_autograd_signatures.py", "--check"], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-800:]
