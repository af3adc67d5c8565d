"""GPU: LPIPS(net='vgg') under torch.autograd (lpips.py, LPIPS).

- LPIPS_PAIR_FWD + LPIPS_LOSS against float64 at the tap geometries of 64^2, 256^2 and 512^2 (B = 1, 2, 8, both broadcast directions),
  LPIPS_SEED and PM_TO_NCHW flags 8 bit for bit, LPIPS_PAIR_BWD to one fp16 ulp of float64 (all-zero feature pixels, NaN d_loss);
- value and both input gradients against the fp32 oracle at 256^2 and 512^2, B = 1 and 4;
- scale invariance bit for bit, retain_graph repeats, two forwards give the same loss bits;
- one cfg2-size guided step with an init image: the oracle's cond_fn on load_clip's model, LPIPS and engine.model against the oracle and
  against the fused CondFnB200 step built with the same LPIPS weights;
- every CONV / glue launch of LPIPS's plans that the shipped-plan tables do not list, through the bit-exact harnesses of
  tests/test_gpu_conv_kernels.py and tests/test_gpu_unet_kernels.py (tests/lpips_autograd_plan_table.py)."""
from __future__ import annotations

import math

import pytest
import torch as th

from tests.lpips_autograd_plan_table import LPIPS_CONV_PLAN, LPIPS_OTHER_PLAN

pytestmark = pytest.mark.gpu

CHANNELS = (64, 128, 256, 512, 512)
U32 = 2.0 ** -24


def covered_conv_signatures() -> set:
    return set(LPIPS_CONV_PLAN)


def covered_other_signatures() -> set:
    return set(LPIPS_OTHER_PLAN)


def _geoms(size):
    return [((size >> k) ** 2, c) for k, c in enumerate(CHANNELS)]


BATCH = [(b, n0, n1) for b in (1, 2, 8) for n0, n1 in ((b, b), (b, 1), (1, b)) if (n0, n1) != (1, 1) or b == 1]
BATCH = sorted(set(BATCH))


def _features(n, hw, c, g, zero_pixel=True):
    f = th.relu(th.randn(n, hw, c, device="cuda", generator=g)).half()
    if zero_pixel:
        f[:, min(3, hw - 1)] = 0  # a pixel whose channels are all zero after ReLU
    return f


def _cos(a, b):
    return float(th.nn.functional.cosine_similarity(a.flatten().double(), b.flatten().double(), dim=0))


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


# ---------------------------------------------------------------------- the four kernels and PM_TO_NCHW flags 8
@pytest.mark.parametrize("B,n0,n1", BATCH, ids=[f"B{b}-{x}x{y}" for b, x, y in BATCH])
@pytest.mark.parametrize("size", [64, 256, 512])
def test_pair_fwd_loss_vs_float64(size, B, n0, n1):
    from clip_guided_diffusion_b200._lib import run_op
    from clip_guided_diffusion_b200.lpips import _fwd_blocks
    g = th.Generator(device="cuda").manual_seed(size + 10 * B + n0)
    parts, nblk, inv, want, mag = [], [], [], th.zeros(B, dtype=th.float64, device="cuda"), th.zeros(B, dtype=th.float64, device="cuda")
    for hw, c in _geoms(size):
        f0, f1 = _features(n0, hw, c, g), _features(n1, hw, c, g)
        w = th.rand(c, device="cuda", generator=g) * 0.2
        nb = _fwd_blocks(hw)
        part = th.full((B, nb), float("nan"), device="cuda")
        run_op("LPIPS_PAIR_FWD", i=[B, hw, c, n0, n1, nb], p=[f0, f1, w, part])
        x0 = f0.double() / (f0.double().pow(2).sum(-1, keepdim=True).sqrt() + 1e-10)
        x1 = f1.double() / (f1.double().pow(2).sum(-1, keepdim=True).sqrt() + 1e-10)
        term = ((x0 - x1) ** 2 * w.double()).expand(B, hw, c)
        want += term.sum((1, 2)) / hw
        mag += term.abs().sum((1, 2)) / hw * (c + hw / (8 * nb) + nb + 16)  # worst-case length of each fp32 summation chain
        parts.append(part)
        nblk.append(nb)
        inv.append(1.0 / hw)
    loss = [th.full((B,), float("nan"), device="cuda") for _ in range(2)]
    for out in loss:
        run_op("LPIPS_LOSS", i=[B, *nblk], f=inv, p=[*parts, out])
    assert th.equal(loss[0], loss[1])
    err = (loss[0].double() - want).abs()
    assert bool((err <= 4 * U32 * mag).all()), (err / want).max().item()


def _seed_f64(d, n0, n1, band):
    def s(ms):
        vals = [min(abs(v), 3.0e38) for v in ms if not math.isnan(v)]
        m = max(vals, default=0.0)
        return 1.0 if m == 0 else 2.0 ** min(max(math.floor(math.log2(band / m)), -60), 60)
    B = len(d)
    return [s([d[r]]) if n == B else s(d) for n in (n0, n1) for r in range(n)]


@pytest.mark.parametrize("B,n0,n1", BATCH, ids=[f"B{b}-{x}x{y}" for b, x, y in BATCH])
def test_seed_bitwise(B, n0, n1):
    from clip_guided_diffusion_b200._lib import run_op
    from clip_guided_diffusion_b200.lpips import LPIPS_SEED_BAND
    g = th.Generator(device="cuda").manual_seed(B + n0)
    d = th.randn(B, device="cuda", generator=g) * th.exp2(th.randint(-100, 100, (B,), device="cuda", generator=g).float())
    specials = [0.0, float("nan"), float("inf"), 1e-30, 1e30, -3e-9, 7e7, 0.5]
    if B == 8:
        d = th.tensor(specials, device="cuda")
    for band in (1.0, LPIPS_SEED_BAND, 2.0 ** 30):
        dyn = th.full((n0 + n1,), float("nan"), device="cuda")
        run_op("LPIPS_SEED", i=[B, n0, n1], f=[band], p=[d, dyn])
        assert dyn.double().tolist() == _seed_f64(d.tolist(), n0, n1, band)


def pm_to_nchw_divide(N, C, HW, ld, flags, scale, *mul):
    """PM_TO_NCHW with flags 8 (image n divided by div[n], powers of two from 2^-60 to 2^60): bitwise the kernel's fp32 product
    (x scale, x mul_c with flags 4) divided exactly; the source's guard channels are NaN"""
    from clip_guided_diffusion_b200._lib import run_op
    g = th.Generator(device="cuda").manual_seed(HW + N + flags)
    src = th.full((N, HW, ld), float("nan"), device="cuda", dtype=th.float16)
    src[:, :, :C] = (th.randn(N, HW, C, device="cuda", generator=g) * 100).half()
    div = th.exp2(th.randint(-60, 61, (N,), device="cuda", generator=g).float())
    dst = th.full((N, C, HW), float("nan"), device="cuda")
    run_op("PM_TO_NCHW", flags=flags, i=[N, C, HW, ld], f=[scale, *mul], p=[src, dst, div])
    v = src[:, :, :C].float() * scale
    if flags & 4:
        v = v * th.tensor(mul[:C], device="cuda")
    assert th.equal(dst, (v / div.view(N, 1, 1)).permute(0, 2, 1))


@pytest.mark.parametrize("size", [64, 256, 512])
def test_pm_to_nchw_divide_bitwise(size):
    from clip_guided_diffusion_b200.lpips import SCALE
    pm_to_nchw_divide(4, 3, size * size, 64, 4 | 8, 1.0, *(1.0 / s for s in SCALE))
    pm_to_nchw_divide(2, 3, size * size, 64, 8, 0.5)


def _ulp16(x):
    a = x.abs().clamp(min=2.0 ** -14)
    return th.exp2(th.floor(th.log2(a)) - 10)


@pytest.mark.parametrize("B,n0,n1", BATCH, ids=[f"B{b}-{x}x{y}" for b, x, y in BATCH])
@pytest.mark.parametrize("size", [64, 256, 512])
def test_pair_bwd_one_ulp(size, B, n0, n1):
    from clip_guided_diffusion_b200._lib import run_op
    from clip_guided_diffusion_b200.lpips import LPIPS_SEED_BAND
    from tests.lpips_autograd_interp import pair_seed
    g = th.Generator(device="cuda").manual_seed(size * 3 + B + n1)
    eps = float(th.tensor(1e-10, dtype=th.float32))
    d = th.rand(B, device="cuda", generator=g) + 0.5
    if B > 1:
        d[1] = float("nan")
    dyn = th.full((n0 + n1,), float("nan"), device="cuda")
    run_op("LPIPS_SEED", i=[B, n0, n1], f=[LPIPS_SEED_BAND], p=[d, dyn])
    for k, (hw, c) in enumerate(_geoms(size)):
        f0, f1 = _features(n0, hw, c, g), _features(n1, hw, c, g, zero_pixel=False)
        w = th.rand(c, device="cuda", generator=g) * 0.2
        df0 = th.full((n0, hw, c), float("nan"), device="cuda", dtype=th.float16)
        df1 = th.full((n1, hw, c), float("nan"), device="cuda", dtype=th.float16)
        run_op("LPIPS_PAIR_BWD", flags=3, i=[B, hw, c, n0, n1], p=[f0, f1, w, d, dyn, df0, df1])
        for s, (fs, fo, got, ns) in enumerate(((f0, f1, df0, n0), (f1, f0, df1, n1))):
            srow = dyn[s * n0:s * n0 + ns].double()
            a = d.double() * (srow if ns == B else srow.expand(B)) / hw
            ref = pair_seed(fs.double(), fo.double(), w.double(), a, eps=eps)
            fin = th.isfinite(ref)
            # a non-finite d_loss gives non-finite seeds on the rows it reaches, never finite ones
            assert bool((~th.isfinite(got[~fin].float())).all())
            if not bool(fin.any()):
                continue
            # one fp16 ulp, plus fp32's own error where g / n and f (g . f) / (n^2 r) cancel: 2^-18 of the largest |seed| of the same
            # pixel (1/256 of an fp16 ulp there), so a saturated pixel loosens nothing but itself
            pix = th.where(th.isfinite(ref), ref.abs(), th.zeros_like(ref)).amax(-1, keepdim=True).expand_as(ref)
            gf, rf = got.float().double()[fin], ref[fin]
            tol = _ulp16(rf) + 2.0 ** -18 * pix[fin]
            assert bool(((gf - rf).abs() <= tol).all()), (size, k, s, float(((gf - rf).abs() / tol).max()))
            if s == 0 and n0 == B:
                assert bool(th.isfinite(got[0].float()).all()) and bool((got[0].float().abs().amax(-1)[min(3, hw - 1)] == 60000))
            if B > 1 and ns == B:
                assert bool(th.isnan(got[1].float()).all()) and bool(th.isfinite(got[0].float()).all())


# ---------------------------------------------------------------------- the model against the fp32 oracle
def _models():
    from clip_guided_diffusion_b200 import lpips as pl
    from oracle import lpips as ol
    sd = ol.seeded_state_dict()
    return pl.LPIPS(lpips_state_dict=sd).to("cuda"), ol.LPIPSVgg({k: v.cuda() for k, v in sd.items()}).cuda(), sd


def _natural(n, size, seed):
    g = th.Generator(device="cuda").manual_seed(seed)
    low = th.randn(n, 3, size // 16, size // 16, device="cuda", generator=g)
    return th.tanh(th.nn.functional.interpolate(low, size=(size, size), mode="bicubic", align_corners=False))


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("size", [256, 512])
def test_value_and_gradients_vs_oracle(size, B):
    m, o, _ = _models()
    # uniform noise, as the fused path's test uses: on smooth inputs the fp32 reference itself is 9 % (rel) from float64, and every fp16
    # VGG (this one, the fused LpipsB200, eager autocast) lands near cos 0.992 (scripts/lpips_grad_accuracy.py, DESIGN.md section 2)
    g = th.Generator(device="cuda").manual_seed(size + B)
    a, b = th.rand(B, 3, size, size, device="cuda", generator=g) * 2 - 1, th.rand(B, 3, size, size, device="cuda", generator=g) * 2 - 1
    res = []
    for fn in (m, o):
        ae, be = a.clone().requires_grad_(), b.clone().requires_grad_()
        v = fn(ae, be)
        res.append((v.detach(), *th.autograd.grad(v.sum() * 1000.0, (ae, be))))
    (v, ga, gb), (vo, oa, ob) = res
    vals = (_rel(v, vo), _cos(ga, oa), _rel(ga, oa), _cos(gb, ob), _rel(gb, ob))
    print(f"\nLPIPS {size}^2 B={B}: rel(value) {vals[0]:.2e} cos/rel(d in0) {vals[1]:.5f} {vals[2]:.2e} cos/rel(d in1) {vals[3]:.5f} {vals[4]:.2e}")
    assert v.shape == (B, 1, 1, 1) and vals[0] < 3e-2 and vals[1] > 0.998 and vals[2] < 6e-2 and vals[3] > 0.998 and vals[4] < 6e-2, vals


def test_invariants_bitwise():
    m, _, _ = _models()
    a, b = _natural(4, 256, 3), _natural(1, 256, 4)
    x = a.clone().requires_grad_()
    d = th.rand(4, 1, 1, 1, device="cuda") + 0.1
    grads = {}
    for k in (-20, 0, 20):
        v = m(x, b)
        (grads[k],) = th.autograd.grad(v, x, grad_outputs=d * 2.0 ** k)
    assert grads[0].abs().max() > 0
    for k in (-20, 20):
        assert th.equal(grads[k], grads[0] * 2.0 ** k), k
    v = m(x, b)
    (g1,) = th.autograd.grad(v.sum(), x, retain_graph=True)
    (g2,) = th.autograd.grad(v.sum(), x)
    assert th.equal(g1, g2)
    assert th.equal(m(a, b), m(a, b))


# ---------------------------------------------------------------------- one cfg2-size step with an init image
@pytest.mark.parametrize("mode", ["ancestral", "ddim"])
def test_cfg2_step_with_init_image(mode):
    from clip_guided_diffusion_b200 import clip_util
    from clip_guided_diffusion_b200 import guidance as pg
    from clip_guided_diffusion_b200 import lpips as pl
    from clip_guided_diffusion_b200 import unet as pu
    from clip_guided_diffusion_b200 import vit as pv
    from clip_guided_diffusion_b200 import weights as pw
    from oracle import diffusion as od
    from oracle import guidance as og
    from oracle import lpips as ol
    from oracle.clip_vit import VIT_CONFIGS, CLIPVisualOnly
    from oracle.unet import UNetModel, config_for
    ucfg, vcfg = pu.config_for(256, True), pv.VIT_CONFIGS["ViT-B/32"]
    usd, vsd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234), pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 1235)
    lsd = ol.seeded_state_dict()
    eng = pg.GuidedStepB200(ucfg, usd, batch=1, device="cuda", input_grad=True)
    clip_model, clip_size = clip_util.load_clip("ViT-B/32", "cuda", clip_state_dict=vsd)
    lpips_vgg = pl.LPIPS(net="vgg", lpips_state_dict=lsd).to("cuda")
    ounet = UNetModel(config_for(256, True)).eval()
    ounet.load_state_dict(usd)
    oclip = CLIPVisualOnly(VIT_CONFIGS["ViT-B/32"]).eval()
    oclip.load_state_dict(vsd)
    ounet, oclip = ounet.cuda(), oclip.cuda()
    for prm in list(ounet.parameters()) + list(oclip.parameters()):
        prm.requires_grad_(False)
    odiff = od.create_gaussian_diffusion(1000, "linear", "ddim25" if mode == "ddim" else "25")
    th.manual_seed(0)
    tgt = th.randn(1, 512, device="cuda")
    coords = og.MakeCutouts(224, 16)._generate_coords(256, 256, 16)
    g = th.Generator().manual_seed(3)
    x, y = th.randn(1, 3, 256, 256, generator=g).cuda(), th.randint(0, 1000, (1,), generator=g).cuda()
    init = _natural(1, 256, 7)
    res = []
    for model, cm, lm in ((eng.model, clip_model, lpips_vgg), (ounet, oclip, ol.LPIPSVgg({k: v.cuda() for k, v in lsd.items()}).cuda())):
        cf = og.OracleCondFn(odiff, cm, tgt, th.ones(1, device="cuda"), cut_size=clip_size, num_cutouts=16, lpips_model=lm,
                             init_tensor=init, init_scale=1000.0)
        cf.current_timestep = 14
        seen = {}

        def cond_fn(xx, tt, out, y=None, cf=cf, seen=seen):
            seen["g"] = cf(xx, tt, out, y=y, coords=coords)
            return seen["g"]
        th.manual_seed(21)
        fn = odiff.p_sample_with_grad if mode == "ancestral" else odiff.ddim_sample_with_grad
        o = fn(model, x, th.full((1,), 14, dtype=th.long, device="cuda"), clip_denoised=False, cond_fn=cond_fn, model_kwargs={"y": y})
        res.append(dict(o, g=seen["g"].detach(), init=cf.last_terms["init"]))
    e, o = res
    vals = (_cos(e["g"], o["g"]), _rel(e["g"], o["g"]), _rel(e["pred_xstart"], o["pred_xstart"]), _rel(e["sample"], o["sample"]))
    print(f"\ncfg2-size {mode} step with init image, engine.model + load_clip + LPIPS vs oracle: cos(g) {vals[0]:.5f} rel(g) {vals[1]:.3e} "
          f"rel(pred_xstart) {vals[2]:.3e} rel(sample) {vals[3]:.3e} init term {e['init']:.4f} vs {o['init']:.4f}")
    assert lpips_vgg.plans[(256, 256, 1, 1)].generation == 1
    assert abs(e["init"] - o["init"]) < 3e-2 * abs(o["init"])
    assert vals[0] > 0.995 and vals[1] < 2e-2 and vals[2] < 2e-2 and vals[3] < 2e-2, vals
    # the fused CondFnB200 step of an engine built with the same LPIPS weights and init image, on the same cutout windows
    from clip_guided_diffusion_b200 import gaussian_diffusion as pgd
    del eng, ounet, oclip
    th.cuda.empty_cache()
    pdiff = pgd.create_gaussian_diffusion(1000, "linear", "ddim25" if mode == "ddim" else "25")
    feng = pg.GuidedStepB200(ucfg, usd, vcfg, vsd, batch=1, num_cutouts=16, device="cuda", lpips_sd=lsd, init_scale=1000.0)
    feng.set_targets(tgt, th.ones(1))
    feng.set_init_image(init)
    feng.stage_step(pdiff.scalar_table(14, 14, 0.0), coords, pdiff.model_timestep(14), y)
    feng.img(feng.unet.x_in).copy_(x)
    feng.img(feng.noise).zero_()
    feng.replay(mode, 16)
    th.cuda.synchronize()
    f = dict(g=feng.img(feng.g).float().clone(), pred_xstart=feng.img(feng.x0).float().clone(), sample=feng.img(feng.sample).float().clone())
    fused = (_cos(e["g"], f["g"]), _rel(e["g"], f["g"]), _rel(e["pred_xstart"], f["pred_xstart"]), _cos(f["g"], o["g"]), _rel(f["g"], o["g"]))
    print(f"cfg2-size {mode} step with init image, generic vs fused CondFnB200: cos(g) {fused[0]:.5f} rel(g) {fused[1]:.3e} "
          f"rel(pred_xstart) {fused[2]:.3e}; fused vs oracle: cos(g) {fused[3]:.5f} rel(g) {fused[4]:.3e}")
    if mode == "ddim":  # eta 0: no noise in the update
        print(f"cfg2-size ddim step, generic vs fused: rel(sample) {_rel(e['sample'], f['sample']):.3e}")
    assert fused[0] > 0.995 and fused[1] < 2e-2 and fused[2] < 2e-2, fused


# ---------------------------------------------------------------------- launches of LPIPS's plans outside the shipped-plan tables
def _conv_ids():
    from tests.test_gpu_conv_kernels import conv_id
    return [conv_id(s) for s in LPIPS_CONV_PLAN]


@pytest.mark.parametrize("case", LPIPS_CONV_PLAN, ids=_conv_ids())
def test_trunk_conv_launches(case):
    from tests import test_gpu_conv_kernels as KC
    KC.test_conv_exact("cuda", case)
    KC.test_conv_randn("cuda", case)


@pytest.mark.parametrize("sig", LPIPS_OTHER_PLAN, ids=[repr(s) for s in LPIPS_OTHER_PLAN])
def test_trunk_other_launches(sig):
    from tests import test_gpu_unet_kernels as KU
    kind, rest = sig[0], tuple(sig[1:])
    if kind == "PM_TO_NCHW" and rest[4] & 8:
        pm_to_nchw_divide(*rest)
    elif kind == "PM_TO_NCHW":
        KU.test_pm_to_nchw("cuda", rest)
    elif kind == "NCHW_TO_PM":
        KU.test_nchw_to_pm("cuda", rest)
    elif kind in ("POOL2", "UP2"):
        KU.test_pool2_up2("cuda", (kind, rest))
    elif kind in ("ADD", "COPY"):
        KU.test_add_copy("cuda", (kind, rest))
    else:
        pytest.fail(f"no GPU harness for {kind}")
