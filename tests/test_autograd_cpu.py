"""CPU: the engine's UNet under torch.autograd (GuidedStepB200(..., input_grad=True)), interpreted op by op (tests/autograd_interp.py).

`model()`'s input gradient against the oracle UNet's autograd, PMV_BWD against float64 autograd of the oracle's p_mean_variance, the
oracle's and the package's *_with_grad steps driven by a plain PyTorch cond_fn, the guards (stale forward, double backward, no-grad
views, unchanged default plans), malformed new ops and the launch coverage of the new path."""
from __future__ import annotations

import json
import subprocess
import sys
import textwrap

import pytest
import torch as th

from clip_guided_diffusion_b200 import gaussian_diffusion as pgd
from clip_guided_diffusion_b200 import guidance as pg
from clip_guided_diffusion_b200 import unet as pu
from clip_guided_diffusion_b200 import vit as pv
from clip_guided_diffusion_b200 import weights as pw
from clip_guided_diffusion_b200._lib import OP
from oracle import diffusion as od
from oracle import guidance as og
from oracle.clip_vit import CLIPVisualOnly, ViTConfig as OViTConfig
from oracle.unet import UNetModel, seeded_init_, tiny_config
from tests.autograd_interp import interpreted
from tests.step_parity import cos, prod_unet_cfg, rel

ROOT = __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__)))
IMAGE = 32


def tiny(B=2, tower=False, input_grad=True, image=IMAGE):
    """a tiny input_grad engine (interpreted) and the oracle networks of the same weights"""
    ocfg = tiny_config(image_size=image, model_channels=64, channel_mult=(1, 2), num_res_blocks=1, attention_resolutions=(image // 2,),
                       class_cond=True)
    ounet = seeded_init_(UNetModel(ocfg)).eval()
    oclip = seeded_init_(CLIPVisualOnly(OViTConfig(32, 16, 128, 2, 64)), seed=5).eval()
    for prm in list(ounet.parameters()) + list(oclip.parameters()):
        prm.requires_grad_(False)
    vit = (pv.ViTConfig(32, 16, 128, 2, 64), oclip.state_dict()) if tower else (None, None)
    eng = pg.GuidedStepB200(prod_unet_cfg(ocfg), ounet.state_dict(), *vit, batch=B, num_cutouts=3, device="cpu", use_graph=False,
                            input_grad=input_grad)
    return interpreted(eng), ounet, oclip


def inputs(B, seed=0, image=IMAGE):
    g = th.Generator().manual_seed(seed)
    return th.randn(B, 3, image, image, generator=g), th.full((B,), 420.0), th.randint(0, 10, (B,), generator=g), \
        th.randn(B, 6, image, image, generator=g)


# ---------------------------------------------------------------------- (a) model() input gradient
@pytest.mark.parametrize("tower", [False, True], ids=["unet_only", "with_clip_tower"])
def test_model_input_gradient_matches_oracle_autograd(tower):
    eng, ounet, _ = tiny(tower=tower)
    x, t, y, w = inputs(2)
    xe = x.clone().requires_grad_()
    (ge,) = th.autograd.grad((w * eng.model(xe, t, y)).sum(), xe)
    xo = x.clone().requires_grad_()
    (go,) = th.autograd.grad((w * ounet(xo, t, y=y)).sum(), xo)
    assert cos(ge, go) > 0.999 and rel(ge, go) < 2e-2, (cos(ge, go), rel(ge, go))


def test_backward_twice_with_retain_graph_is_identical():
    """the UNet backward re-enters only forward activations and its own buffers: retain_graph=True may run it again"""
    eng, _, _ = tiny()
    x, t, y, w = inputs(2, seed=1)
    xe = x.clone().requires_grad_()
    out = eng.model(xe, t, y)
    (g1,) = th.autograd.grad((w * out).sum(), xe, retain_graph=True)
    (g2,) = th.autograd.grad((w * out).sum(), xe)
    assert th.equal(g1, g2)


# ---------------------------------------------------------------------- (b) PMV_BWD
def _pmv_case(which, seed=2):
    """PMV_BWD of one plan, interpreted, against float64 autograd of oracle.diffusion's p_mean_variance algebra"""
    eng, _, _ = tiny(B=2)
    diff = pgd.create_gaussian_diffusion(1000, "linear", "25")
    odiff = od.create_gaussian_diffusion(1000, "linear", "25")
    ti = 9
    B, shp = 2, (2, 3, IMAGE, IMAGE)
    g = th.Generator().manual_seed(seed)
    x, mo = th.randn(shp, generator=g), th.randn(B, 6, IMAGE, IMAGE, generator=g)
    ups = [th.randn(shp, generator=g) if k in which else None for k in range(4)]
    eng.v(eng.sc).copy_(th.from_numpy(diff.scalar_table(ti, ti)))
    eng.v(eng.unet.out, (B, 6, IMAGE, IMAGE)).copy_(mo)
    eng.img(eng.unet.x_in).copy_(x)
    eng.plan.run_range("pmv", "cond")  # the forward's variance buffer PMV_BWD reads
    grads = eng.v(eng.ag_pmv_grads, (4,) + shp)
    for k in range(4):
        grads[k].copy_(ups[k] if ups[k] is not None else th.zeros(shp))
    eng.plan.run_range("ag_pmv_bwd", "ag_seed")
    xd, md = x.double().requires_grad_(), mo.double().requires_grad_()
    out = odiff.p_mean_variance(lambda xx, tt, **k: md, xd, th.full((B,), ti), clip_denoised=False)
    loss = sum((out[k] * ups[j].double()).sum() for j, k in enumerate(pg.PMV_KEYS) if ups[j] is not None)
    dx, dmo = th.autograd.grad(loss, (xd, md), allow_unused=True)
    dx = th.zeros_like(xd) if dx is None else dx
    return eng.v(eng.ag_d_out, (B, 6, IMAGE, IMAGE)).double(), eng.img(eng.ag_dx_direct).double(), dmo, dx


@pytest.mark.parametrize("which", [(0,), (1,), (2,), (3,), (0, 1, 2, 3)], ids=["pred_xstart", "mean", "variance", "log_variance", "all"])
def test_pmv_bwd_is_the_transpose_of_p_mean_variance(which):
    d_out, dx_direct, want_dout, want_dx = _pmv_case(which)
    assert rel(d_out, want_dout) < 1e-5, rel(d_out, want_dout)
    # the model output does not see x: d loss / dx of the oracle's algebra is exactly the direct term
    assert rel(dx_direct, want_dx) < 1e-5 if want_dx.abs().max() > 0 else dx_direct.abs().max() == 0


# ---------------------------------------------------------------------- (c), (d) sampling steps with a plain PyTorch cond_fn
def _cond(odiff, oclip, coords, ti, use_magnitude=False):
    cf = og.OracleCondFn(odiff, oclip, th.randn(1, 64, generator=th.Generator().manual_seed(99)), th.ones(1), cut_size=32, num_cutouts=3,
                         clip_guidance_scale=1000.0, tv_scale=150.0, range_scale=50.0, sat_scale=0.0, use_magnitude=use_magnitude)
    cf.current_timestep = ti
    seen = {"cf": cf}

    def cond_fn(x, t, out, y=None):  # a plain callable: what a user's PyTorch guidance looks like to the loops
        g = cf(x, t, out, y=y, coords=coords)
        seen["g"] = g.detach().clone()
        return g
    return cond_fn, seen


def _oracle_step(model, odiff, oclip, mode, x, ti, y, coords, clip_denoised):
    cond_fn, seen = _cond(odiff, oclip, coords, ti)
    th.manual_seed(123)
    fn = odiff.p_sample_with_grad if mode == "ancestral" else odiff.ddim_sample_with_grad
    out = fn(model, x, th.full((x.shape[0],), ti, dtype=th.long), clip_denoised=clip_denoised, cond_fn=cond_fn, model_kwargs={"y": y})
    return dict(out, g=seen["g"])


def _check(e, o):
    assert cos(e["g"], o["g"]) > 0.995 and rel(e["pred_xstart"], o["pred_xstart"]) < 2e-2 and rel(e["sample"], o["sample"]) < 2e-2, \
        (cos(e["g"], o["g"]), rel(e["pred_xstart"], o["pred_xstart"]), rel(e["sample"], o["sample"]))


@pytest.mark.parametrize("mode", ["ancestral", "ddim"])
@pytest.mark.parametrize("clip_denoised", [False, True])
def test_oracle_steps_with_engine_model(mode, clip_denoised):
    """(c) the oracle's own *_with_grad step (clip_denoised, its own p_mean_variance) with model = engine.model"""
    eng, ounet, oclip = tiny()
    odiff = od.create_gaussian_diffusion(1000, "linear", "25")
    x, _, y, _ = inputs(2, seed=3)
    # late in the chain, where most of pred_xstart lies inside [-1, 1]: with clip_denoised the gradient flows through the unclipped
    # pixels only, and a random-weight UNet early in the chain leaves almost none
    x, ti = 0.5 * x, 4
    coords = [(0, 0, 32), (4, 2, 20), (10, 8, 16)]
    e = _oracle_step(eng.model, odiff, oclip, mode, x, ti, y, coords, clip_denoised)
    o = _oracle_step(ounet, odiff, oclip, mode, x, ti, y, coords, clip_denoised)
    _check(e, o)


@pytest.mark.parametrize("mode", ["ancestral", "ddim"])
def test_package_steps_with_plain_cond_fn(mode):
    """(d) the package's p_sample_with_grad / ddim_sample_with_grad (p_mean_variance and update on the engine's kernels) with the same
    plain cond_fn, against the oracle step"""
    eng, ounet, oclip = tiny()
    odiff = od.create_gaussian_diffusion(1000, "linear", "25")
    pdiff = pgd.create_gaussian_diffusion(1000, "linear", "25")
    x, _, y, _ = inputs(2, seed=4)
    coords = [(0, 0, 32), (3, 5, 24), (12, 1, 17)]
    o = _oracle_step(ounet, odiff, oclip, mode, x, 14, y, coords, False)
    cond_fn, seen = _cond(odiff, oclip, coords, 14)
    th.manual_seed(123)
    fn = pdiff.p_sample_with_grad if mode == "ancestral" else pdiff.ddim_sample_with_grad
    e = fn(eng.model, x, th.full((2,), 14, dtype=th.long), clip_denoised=False, cond_fn=cond_fn, model_kwargs={"y": y})
    assert e["sample"].grad_fn is None and e["pred_xstart"].grad_fn is None
    _check(dict(e, g=seen["g"]), o)


def test_package_loop_with_plain_cond_fn():
    """the package's loop hands a plain cond_fn x with requires_grad inside enable_grad, step after step"""
    eng, ounet, oclip = tiny(B=1)
    odiff = od.create_gaussian_diffusion(1000, "linear", "25")
    pdiff = pgd.create_gaussian_diffusion(1000, "linear", "25")
    coords = [(0, 0, 32), (3, 5, 24), (12, 1, 17)]
    finals = []
    for diff, model in ((pdiff, eng.model), (odiff, ounet)):
        inner, seen = _cond(odiff, oclip, coords, 24, use_magnitude=True)  # the RMS clamp keeps a random-weight chain bounded
        calls = []

        def cond_fn(x, t, out, y=None, inner=inner, seen=seen, calls=calls):
            calls.append(bool(x.requires_grad and th.is_grad_enabled()))
            g = inner(x, t, out, y=y)
            seen["cf"].current_timestep -= 1  # the driver loop's step_done (cgd/cgd.py:267)
            return g
        th.manual_seed(5)
        out = None
        for k, out in enumerate(diff.ddim_sample_loop_progressive(model, (1, 3, IMAGE, IMAGE), clip_denoised=False, cond_fn=cond_fn,
                                                                  model_kwargs={"y": th.zeros(1, dtype=th.long)}, cond_fn_with_grad=True)):
            if k == 3:
                break
        assert calls == [True] * 4
        finals.append(out["sample"].detach())
    assert rel(finals[0], finals[1]) < 2e-2, rel(finals[0], finals[1])


# ---------------------------------------------------------------------- (e) guards
def test_backward_after_another_forward_raises():
    eng, _, _ = tiny()
    x, t, y, w = inputs(2)
    xe = x.clone().requires_grad_()
    out = eng.model(xe, t, y)
    eng.model(x, t, y)  # a no-grad forward overwrites the activations
    with pytest.raises(RuntimeError, match="another UNet forward"):
        th.autograd.grad((w * out).sum(), xe)
    out = eng.model(xe, t, y)
    with pytest.raises(RuntimeError, match="double backward"):
        th.autograd.grad((w * out).sum(), xe, create_graph=True)
    with pytest.raises(ValueError, match="shape"):
        eng.model(th.zeros(1, 3, IMAGE, IMAGE, requires_grad=True), t[:1], y[:1])
    plain, _, _ = tiny(input_grad=False)
    with pytest.raises(RuntimeError, match="input_grad=True"):
        plain.model(xe, t, y)


def test_update_after_another_forward_raises():
    eng, _, _ = tiny()
    pdiff = pgd.create_gaussian_diffusion(1000, "linear", "25")
    x, t, y, _ = inputs(2)

    def greedy(xx, tt, out, y=None):  # runs the engine's model itself: x and the p_mean_variance buffers are gone
        eng.model(xx.detach(), th.full((2,), 1.0), y)
        return th.zeros_like(xx)
    with pytest.raises(RuntimeError, match="update after another UNet forward"):
        pdiff.ddim_sample_with_grad(eng.model, x, th.full((2,), 5, dtype=th.long), clip_denoised=False, cond_fn=greedy, model_kwargs={"y": y})


def test_no_grad_model_is_a_view_with_unchanged_values():
    eng, _, _ = tiny()
    plain, _, _ = tiny(input_grad=False)
    x, t, y, _ = inputs(2)
    with th.no_grad():
        a = eng.model(x.clone().requires_grad_(), t, y)
    b = plain.model(x, t, y)
    assert a.grad_fn is None and a.data_ptr() == eng.unet.out_view.data_ptr() and th.equal(a, b)


def test_default_plans_unchanged():
    """an input_grad engine's ops before engine_end lower to the default engine's structs, byte for byte, and its range marks agree"""
    eng, _, _ = tiny(tower=True)
    ref, _, _ = tiny(tower=True, input_grad=False)
    n = ref.plan.marks["engine_end"]
    assert n == eng.plan.marks["engine_end"] and {k: v for k, v in eng.plan.marks.items() if not k.startswith("ag_")} == ref.plan.marks
    a, b = eng.plan.lower(1 << 40), ref.plan.lower(1 << 40)
    assert len(b) == n and all(bytes(a[k]) == bytes(b[k]) for k in range(n))
    assert [eng.plan.ops[k].code for k in range(n, len(eng.plan.ops))] == [OP[c] for c in ("PMV_BWD", "GRAD_SEED", "GRAD_UNSCALE", "GRAD_UNSCALE")]


def test_plan_fingerprint_unchanged():
    """scripts/plan_fingerprint.py (default engines of every published configuration) prints what it printed before input_grad existed"""
    want = open(f"{ROOT}/tests/golden/plan_fingerprint.txt").read()
    r = subprocess.run([sys.executable, f"{ROOT}/scripts/plan_fingerprint.py"], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-800:]
    assert r.stdout == want


# ---------------------------------------------------------------------- (f) malformed new ops
CHILD = textwrap.dedent('''
    import ctypes, json, sys
    sys.path.insert(0, sys.argv[1])
    from clip_guided_diffusion_b200 import _lib
    from tests.plan_interp import CODE
    from tests.test_autograd_cpu import tiny
    lib = _lib.load()
    plan = tiny()[0].plan
    arr = plan.lower(1 << 40)
    vals = [0, -1, 1, 3, 7, (1 << 31) - 1, 1 << 40, -(1 << 40)]
    n, zero = 0, []
    for k in range(plan.marks["ag_pmv_bwd"], plan.marks["ag_end"]):
        base = arr[k]
        muts = [("i", j, v) for j in range(24) for v in vals if base.i[j] != v]
        muts += [("p", j, v) for j in range(12) for v in (0, 3) if base.p[j]] + [("flags", 0, v) for v in (-1, 1 << 30, 255)]
        for w, j, v in muts:
            o = type(base)()
            ctypes.memmove(ctypes.byref(o), ctypes.byref(base), ctypes.sizeof(base))
            if w == "i":
                o.i[j] = v
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
def test_malformed_autograd_ops_return_error_codes():
    try:
        r = subprocess.run([sys.executable, "-c", CHILD, ROOT], capture_output=True, text=True, timeout=180)
    except subprocess.TimeoutExpired as e:
        pytest.fail(f"cgd_run_op hung on {[l for l in (e.stdout or b'').decode().splitlines() if l.startswith('TRY')][-1:]}")
    lines = r.stdout.splitlines()
    assert r.returncode == 0 and lines and lines[-1].startswith("DONE"), f"crashed (rc {r.returncode}): {r.stderr[-400:]}"
    _, n, zero = lines[-1].split(" ", 2)
    assert int(n) > 600 and json.loads(zero) == [], json.loads(zero)[:5]


# ---------------------------------------------------------------------- (g) launch coverage of the new path
@pytest.mark.parametrize("size", [64, 128, 256, 512])
def test_input_grad_engines_make_only_tested_launches(size):
    from tests import test_gpu_conv_kernels as KC
    from tests import test_gpu_unet_kernels as KU
    from tests.test_conv_coverage_cpu import plan_conv_signatures
    from tests.test_unet_kernel_coverage_cpu import plan_signatures
    th.manual_seed(0)
    ucfg = pu.config_for(size, class_cond=True)
    eng = pg.GuidedStepB200(ucfg, pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234), batch=1, device="cpu", input_grad=True)
    conv = plan_conv_signatures(eng.plan)
    other = plan_signatures(eng)
    assert any(s[0] == "GN_BWD" for s in other) and len(conv) > 10
    missing = sorted((s for s in conv if s not in KC.covered_signatures()), key=repr) + \
        sorted((s for s in other if s not in KU.covered_signatures()), key=repr)
    assert not missing, missing[:8]
