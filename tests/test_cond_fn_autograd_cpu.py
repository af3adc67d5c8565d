"""CPU: MakeCutouts, CLIP_NORMALIZE and the losses under torch.autograd (guidance.py, clip_util.py, losses.py), with the new ops and flags
interpreted on the CPU (tests/cond_fn_autograd_interp.py in place of ``_lib.run_op``).

Value and gradient against the oracle's float64 autograd (pool and use_augs cutouts on clipped windows, tv / range, spherical at the
reference's shapes and a generic broadcast), the five cond_fn goldens of the reference's own closure, the reference's unmodified closure on
the package's modules (when the reference tree is present), and malformed new ops."""
from __future__ import annotations

import ast
import importlib.util
import json
import os
import subprocess
import sys
import textwrap
import types

import pytest
import torch as th

from clip_guided_diffusion_b200 import _lib, augs, clip_util
from clip_guided_diffusion_b200 import losses as pl
from clip_guided_diffusion_b200.guidance import MakeCutouts
from oracle import guidance as og
from tests.cond_fn_autograd_interp import reference_style_cond_fn, run_op
from tests.test_cond_fn_reference import CASES, GOLD, StubClip, stub_pred_xstart

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"


@pytest.fixture(autouse=True)
def interpreted(monkeypatch):
    monkeypatch.setattr(_lib, "run_op", run_op)


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp(min=1e-30))


def _value_grad(fn, *xs, w=None):
    xs = [x.clone().requires_grad_() for x in xs]
    v = fn(*xs)
    w = th.randn(v.shape, generator=th.Generator().manual_seed(7)).to(v.dtype) if w is None else w
    return v.detach(), th.autograd.grad((v * w).sum(), xs)


# ---------------------------------------------------------------------- cutouts
def test_pool_cutouts_value_and_gradient_on_clipped_windows():
    x = th.rand(2, 3, 48, 40, generator=th.Generator().manual_seed(1))
    mk = MakeCutouts(16, 6, 0.5)
    th.manual_seed(3)
    mk.cache_coordinates(48, 40)  # sic (H, W) as (side_x, side_y): windows clipped at the right border
    coords = mk.cached_coords
    assert any(ox + s > 40 for ox, _, s in coords)
    v, (g,) = _value_grad(lambda t: mk(t, use_cache=True), x)
    ref = og.MakeCutouts(16, 6)
    vo, (go,) = _value_grad(lambda t: ref(t, coords=coords), x.double())
    assert v.dtype == th.float32 and v.shape == (12, 3, 16, 16) and g.shape == x.shape
    assert rel(v, vo) < 1e-5 and rel(g, go) < 1e-5, (rel(v, vo), rel(g, go))
    with th.no_grad():
        assert th.equal(mk(x.requires_grad_(), use_cache=True), v)


def test_use_augs_cutouts_value_and_gradient():
    x = th.rand(2, 3, 48, 40, generator=th.Generator().manual_seed(2))
    mk = MakeCutouts(16, 4, use_augs=True)
    th.manual_seed(11)
    v, (g,) = _value_grad(lambda t: mk(t), x)
    th.manual_seed(11)  # the same draws again, in the same order: windows, then the parameters and noise of every cutout
    coords = mk._generate_coords(48, 40, 4)
    noise = th.zeros(4, 4, 2, 3, 40, 40)
    prm = augs.draw_aug_params(coords, 2, 48, 40, noise_out=noise)
    vo, (go,) = _value_grad(lambda t: og.MakeCutouts(16, 4)(t, coords=coords, aug_params=prm, aug_noise=noise.double()), x.double())
    assert v.shape == (8, 3, 16, 16) and rel(v, vo) < 2e-3, rel(v, vo)  # the kernel stores the augmented cutouts in fp16
    assert rel(g, go) < 1e-5, rel(g, go)


def test_two_cutout_calls_under_one_backward_and_no_double_backward():
    x = th.rand(1, 3, 32, 32, generator=th.Generator().manual_seed(3)).requires_grad_()
    mk = MakeCutouts(8, 3)
    th.manual_seed(0)
    a, b = mk(x), mk(x * 2)
    (g,) = th.autograd.grad(a.sum() + b.sum(), x)
    th.manual_seed(0)
    ref = og.MakeCutouts(8, 3)
    (go,) = th.autograd.grad(ref(x).sum() + ref(x * 2).sum(), x)
    assert rel(g, go) < 1e-5
    with pytest.raises(RuntimeError, match="differentiate twice|does not require grad"):
        (gg,) = th.autograd.grad(mk(x).sum(), x, create_graph=True)
        th.autograd.grad(gg.sum(), x)


# ---------------------------------------------------------------------- tv / range
@pytest.mark.parametrize("B", [1, 2, 3, 4])
def test_tv_and_range_value_and_gradient(B):
    x = th.randn(B, 3, 24, 20, generator=th.Generator().manual_seed(B)) * 1.4
    for fn, ref in ((pl.tv_loss, og.tv_loss), (pl.range_loss, og.range_loss)):
        v, (g,) = _value_grad(fn, x)
        vo, (go,) = _value_grad(ref, x.double())
        assert v.shape == (B,) and v.dtype == th.float32 and rel(v, vo) < 1e-5 and rel(g, go) < 1e-5, fn.__name__


def test_losses_keep_the_input_dtype_and_reject_bad_input():
    x = th.randn(2, 3, 8, 8, dtype=th.float16).requires_grad_()
    v = pl.tv_loss(x)
    (g,) = th.autograd.grad(v.sum(), x)
    assert v.dtype == th.float32 and g.dtype == th.float16
    with pytest.raises(ValueError, match=r"\[B, C, H, W\]"):
        pl.range_loss(th.zeros(3, 8, 8))
    with pytest.raises(ValueError, match="floating-point"):
        pl.tv_loss(th.zeros(1, 3, 8, 8, dtype=th.int32))
    with th.no_grad():
        assert pl.range_loss(x).grad_fn is None


# ---------------------------------------------------------------------- spherical
SPH = [((1, 5, 2, 32), (1, 1, 32)), ((1, 5, 1, 32), (1, 3, 32)), ((1, 4, 1, 24), (1, 17, 24)), ((1, 4, 3, 16), (1, 3, 16)),
       ((4, 1, 5, 16), (3, 1, 16)), ((16,), (6, 16))]


@pytest.mark.parametrize("xs,ys", SPH, ids=[f"{a}-{b}" for a, b in SPH])
def test_spherical_value_and_gradients(xs, ys):
    g = th.Generator().manual_seed(len(xs) * 100 + ys[-2])
    x, y = th.randn(xs, generator=g), th.randn(ys, generator=g)
    v, (gx, gy) = _value_grad(pl.spherical_dist_loss, x, y)
    vo, (ox, oy) = _value_grad(og.spherical_dist_loss, x.double(), y.double())
    assert v.shape == vo.shape == th.broadcast_shapes(xs[:-1], ys[:-1])
    assert rel(v, vo) < 1e-5 and rel(gx, ox) < 1e-5 and rel(gy, oy) < 1e-5, (rel(v, vo), rel(gx, ox), rel(gy, oy))


def test_spherical_only_x_requires_grad_and_bad_shapes_raise():
    x, y = th.randn(1, 3, 2, 8).requires_grad_(), th.randn(1, 1, 8)
    (gx,) = th.autograd.grad(pl.spherical_dist_loss(x, y).sum(), x)
    (ox,) = th.autograd.grad(og.spherical_dist_loss(x, y).sum(), x)
    assert rel(gx, ox) < 1e-5
    with pytest.raises(RuntimeError, match="shape|size"):
        pl.spherical_dist_loss(th.randn(1, 4, 2, 8), th.randn(1, 3, 8))  # batch 2 against 3 prompts: torch cannot broadcast either
    with pytest.raises(RuntimeError):
        og.spherical_dist_loss(th.randn(1, 4, 2, 8), th.randn(1, 3, 8))
    with pytest.raises(ValueError, match="same D"):
        pl.spherical_dist_loss(th.randn(2, 8), th.randn(2, 6))


def test_clip_normalize_is_the_reference_normalize():
    x = th.rand(4, 3, 8, 8).requires_grad_()
    (g,) = th.autograd.grad(clip_util.CLIP_NORMALIZE(x).sum(), x)
    assert th.allclose(clip_util.CLIP_NORMALIZE(x), og.clip_normalize(x))
    assert th.allclose(g[0, :, 0, 0], 1 / th.tensor(og.CLIP_STD))


# ---------------------------------------------------------------------- the reference's closure
def package_ns(c, name, **kw):
    return types.SimpleNamespace(
        diffusion=types.SimpleNamespace(sqrt_one_minus_alphas_cumprod={c["t"]: GOLD[name + "_fac"][0]}), current_timestep=c["t"],
        make_cutouts=MakeCutouts(32, c["cutn"], cutout_size_power=c["pow"]), clip_util=clip_util, losses=pl, clip_model=StubClip(32, 16),
        target_embeds=th.from_numpy(GOLD[name + "_target"]), weights=th.from_numpy(GOLD[name + "_weights"]), num_cutouts=c["cutn"],
        clip_guidance_scale=1000, tv_scale=150, range_scale=50, sat_scale=c["sat"], use_magnitude=c["mag"], **kw)


@pytest.mark.parametrize("name", list(CASES))
def test_package_modules_reproduce_the_reference_closure_golden(name):
    c = CASES[name]
    cond_fn = reference_style_cond_fn(package_ns(c, name))
    th.manual_seed(c["seed"])
    x = th.from_numpy(GOLD[name + "_x"]).clone().requires_grad_()
    got = cond_fn(x, th.full((c["B"],), c["t"]), {"pred_xstart": stub_pred_xstart(x)})
    want = th.from_numpy(GOLD[name + "_grad"])
    assert rel(got, want) < 1e-5, (name, rel(got, want))


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "cgd")), reason="the reference tree is not present")
@pytest.mark.parametrize("name", list(CASES))
def test_reference_closure_on_package_modules(name):
    """cond_fn cut out of cgd/cgd.py with ast, unmodified: once on the reference's losses / MakeCutouts / CLIP_NORMALIZE, once on the
    package's"""
    import torchvision.transforms as tvt
    tree = ast.parse(open(os.path.join(REF, "cgd", "cgd.py")).read())
    outer = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "clip_guided_diffusion")
    code = compile(ast.Module([next(n for n in ast.walk(outer) if isinstance(n, ast.FunctionDef) and n.name == "cond_fn")], []), "cgd.py", "exec")
    norm = next(n for n in ast.parse(open(os.path.join(REF, "cgd", "clip_util.py")).read()).body
                if isinstance(n, ast.Assign) and getattr(n.targets[0], "id", "") == "CLIP_NORMALIZE")
    ref_mods = dict(losses=_load(os.path.join(REF, "cgd", "losses.py"), "ref_losses"),
                    clip_util=types.SimpleNamespace(CLIP_NORMALIZE=eval(compile(ast.Expression(norm.value), "clip_util.py", "eval"), {"tvt": tvt})),
                    mk=_load(os.path.join(REF, "cgd", "modules.py"), "ref_modules").MakeCutouts)
    c = CASES[name]
    grads = []
    for mods in (ref_mods, dict(losses=pl, clip_util=clip_util, mk=MakeCutouts)):
        ns = dict(th=th, losses=mods["losses"], clip_util=mods["clip_util"], tqdm=types.SimpleNamespace(write=lambda *a, **k: None), wandb_project=None,
                  progress=False, lpips_vgg=None, init_tensor=None, init_scale=0, reduce_clip=False, progressive_cutout=False, cached_cutouts=False,
                  timestep_respacing="25", diffusion=types.SimpleNamespace(num_timesteps=c["T"], sqrt_one_minus_alphas_cumprod={c["t"]: GOLD[name + "_fac"][0]}),
                  current_timestep=c["t"], num_cutouts=c["cutn"], make_cutouts=mods["mk"](32, c["cutn"], cutout_size_power=c["pow"]),
                  clip_model=StubClip(32, 16), target_embeds=th.from_numpy(GOLD[name + "_target"]), weights=th.from_numpy(GOLD[name + "_weights"]),
                  clip_guidance_scale=1000, tv_scale=150, range_scale=50, sat_scale=c["sat"], use_saturation=c["sat"] != 0, use_magnitude=c["mag"])
        exec(code, ns)
        th.manual_seed(c["seed"])
        x = th.from_numpy(GOLD[name + "_x"]).clone().requires_grad_()
        grads.append(ns["cond_fn"](x, th.full((c["B"],), c["t"]), {"pred_xstart": stub_pred_xstart(x)}))
    assert rel(grads[1], grads[0]) < 1e-5, rel(grads[1], grads[0])


# ---------------------------------------------------------------------- malformed new ops
CHILD = textwrap.dedent('''
    import ctypes, json, sys
    sys.path.insert(0, sys.argv[1])
    from clip_guided_diffusion_b200 import _lib
    lib = _lib.load()
    A = 1 << 20  # never dereferenced on a machine without a GPU
    bases = [("CUTOUTS_BWD", 4, [2, 64, 48, 3, 16, 16, 768], [0, 0, 0, .5, .5, .5, 1], [A, A + 64, A + 128]),
             ("CUTOUTS_BWD", 6, [2, 64, 48, 200, 16, 16, 768], [0, 0, 0, .5, .5, .5, 1], [A, A + 64, A + 128]),
             ("CUTOUTS_AUG_BWD", 4, [2, 64, 48, 3, 16, 16, 768], [0, 0, 0, 1, 1, 1, 2], [A, A + 64, A + 128, A + 256]),
             ("IMG_LOSS_FWD", 1, [2, 3, 64, 48, 16], [], [A, A + 64, A + 128]), ("IMG_LOSS_BWD", 2, [2, 3, 64, 48], [], [A, A + 64, A + 128]),
             ("SPH_DIST_FWD", 0, [6, 512, 3, 2], [], [A, A + 64, A + 128, A + 256]),
             ("SPH_DIST_BWD", 3, [6, 512, 3, 2], [], [A, A + 64, A + 128, A + 256, A + 512, A + 1024, A + 2048, A + 2112, A + 2176, A + 2240])]
    vals = [0, -1, 1, 3, 7, (1 << 31) - 1, 1 << 40, -(1 << 40)]
    n, zero = 0, []
    for code, flags, i, f, p in bases:
        muts = [("i", j, v) for j in range(len(i) + 1) for v in vals]
        muts += [("p", j, v) for j in range(len(p)) for v in (0, 3)] + [("flags", 0, v) for v in (-1, 1 << 30, 255, 8, 1, 5)]
        for w, j, v in muts:
            o = _lib.CgdOp()
            o.code, o.flags = _lib.OP[code], flags
            for k, x in enumerate(i): o.i[k] = x
            for k, x in enumerate(f): o.f[k] = x
            for k, x in enumerate(p): o.p[k] = x
            if w == "i": o.i[j] = v
            elif w == "p": o.p[j] = 0 if v == 0 else o.p[j] + v
            else: o.flags = v
            print("TRY", code, w, j, v, flush=True)
            n += 1
            if lib.cgd_run_op(ctypes.byref(o), None) == 0:
                zero.append((code, w, j, v))
    print("DONE", n, json.dumps(zero), flush=True)
''')


@pytest.mark.skipif(th.cuda.is_available(), reason="needs a box WITHOUT a GPU: only the argument checks may run")
def test_malformed_new_ops_return_error_codes():
    try:
        r = subprocess.run([sys.executable, "-c", CHILD, ROOT], capture_output=True, text=True, timeout=600)
    except subprocess.TimeoutExpired as e:
        pytest.fail(f"cgd_run_op hung on {[l for l in (e.stdout or b'').decode().splitlines() if l.startswith('TRY')][-1:]}")
    lines = r.stdout.splitlines()
    assert r.returncode == 0 and lines and lines[-1].startswith("DONE"), f"crashed (rc {r.returncode}): {r.stderr[-400:]}"
    _, n, zero = lines[-1].split(" ", 2)
    assert int(n) > 400 and json.loads(zero) == [], json.loads(zero)[:5]


def test_flag_4_layout_is_checked_before_any_cuda_call():
    import ctypes
    lib = _lib.load()
    for code in ("CUTOUTS_BWD", "CUTOUTS_AUG_BWD"):
        op = _lib.CgdOp()
        op.code, op.flags = _lib.OP[code], 4
        for j, v in enumerate([1, 64, 64, 4, 32, 16, 768]):  # ViT patch rows, not fp32 cutouts
            op.i[j] = v
        for j in range(4):
            op.p[j] = 256 * (j + 1)
        assert lib.cgd_run_op(ctypes.byref(op), None) < 0 and b"flags 4" in lib.cgd_last_error(), code


def test_run_op_refuses_cpu_operands(monkeypatch):
    monkeypatch.undo()
    with pytest.raises(_lib.CgdError, match="GPU only"):
        pl.tv_loss(th.zeros(1, 3, 8, 8))
    with pytest.raises(_lib.CgdError, match="GPU only"):
        MakeCutouts(8, 2)(th.zeros(1, 3, 16, 16))
