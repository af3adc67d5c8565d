"""GPU: MakeCutouts, CLIP_NORMALIZE and the losses under torch.autograd on the device kernels (CUTOUTS_BWD / CUTOUTS_AUG_BWD flags 4,
IMG_LOSS_FWD / _BWD, SPH_DIST_FWD / _BWD).

- each new op and flag at production shapes against float64 references: the cutout gather at every tower resolution x images 64^2 to
  512^2 x cutn 4 to 64 and one case above 128 cutouts (the element kernel), to a few fp32 ulps per summed term, repeating bitwise;
  tv / range at 64^2 to 512^2, B 1 to 4; spherical at D 512 / 640 / 768 / 1024 with up to 65 prompts;
- the five goldens of the reference's own closure (tests/golden/cond_fn_golden.npz) with the package's modules and StubClip on CUDA;
- invariants: 2^k upstream scaling, retain_graph repeats, no-grad calls, dtype and device errors;
- one cfg2-size step (ancestral and DDIM, init image with LPIPS) with every piece of the cond_fn on the package, against the fp32 oracle
  step and the fused CondFnB200 step on the same windows, and a use_augs step against the oracle with the same draws."""
from __future__ import annotations

import types

import pytest
import torch as th
import torch.nn.functional as F

from clip_guided_diffusion_b200 import _lib, augs, clip_util
from clip_guided_diffusion_b200 import losses as pl
from clip_guided_diffusion_b200.guidance import MakeCutouts
from oracle import guidance as og
from tests.cond_fn_autograd_interp import reference_style_cond_fn
from tests.test_cond_fn_reference import CASES, GOLD, StubClip, stub_pred_xstart

pytestmark = pytest.mark.gpu
EPS32 = 2.0 ** -24


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp(min=1e-30))


def _cos(a, b):
    return float(F.cosine_similarity(a.double().flatten(), b.double().flatten(), dim=0))


def _pool64(x, coords, cs, d):
    """float64 d / d x of sum(d * cutouts), and the same with |d| (the scale of the summed terms)"""
    out = []
    for w in (d, d.abs()):
        xe = th.zeros_like(x, dtype=th.float64, requires_grad=True)
        cuts = th.cat([F.adaptive_avg_pool2d(xe[:, :, oy:oy + s, ox:ox + s], cs) for ox, oy, s in coords])
        out.append(th.autograd.grad((cuts * w.double()).sum(), xe)[0])
    return out


# ---------------------------------------------------------------------- cutout backward, flag 4
CUT = [(cs, hw, n) for cs in (224, 288, 336, 384) for hw in ((64, 64), (128, 96), (256, 256), (512, 448)) for n in (4, 16, 64)] + \
      [(224, (256, 256), 160)]


@pytest.mark.parametrize("cs,hw,n", CUT, ids=[f"{c}-{h}x{w}-{n}" for c, (h, w), n in CUT])
def test_cutouts_bwd_fp32_upstream(cs, hw, n):
    H, W = hw
    B = 2 if n <= 16 else 1
    th.manual_seed(cs + H + n)
    coords = og.MakeCutouts(cs, n)._generate_coords(H, W, n)  # (H, W) as (side_x, side_y) like the reference: clipped windows
    cdev = th.tensor(coords, dtype=th.int32, device="cuda")
    d = th.randn(n * B, 3, cs, cs, device="cuda")
    dims = [B, H, W, n, cs, cs, 3 * cs * cs]
    dx = th.empty(B, 3, H, W, device="cuda")
    _lib.run_op("CUTOUTS_BWD", flags=4, i=dims, f=[0, 0, 0, 0.5, 0.5, 0.5, 1.0], p=[d, cdev, dx])
    ref, mag = _pool64(th.zeros(B, 3, H, W, device="cuda"), coords, cs, d)
    err = (dx.double() - ref).abs()
    terms = n * (cs // min(H, W) + 2) ** 2  # summed terms per pixel: cutouts x output bins that contain it
    assert (err <= 4 * EPS32 * terms * mag + 1e-30).all(), float((err / (mag * terms * EPS32 + 1e-30)).max())
    dx2 = th.empty_like(dx)
    _lib.run_op("CUTOUTS_BWD", flags=4, i=dims, f=[0, 0, 0, 0.5, 0.5, 0.5, 1.0], p=[d, cdev, dx2])
    assert th.equal(dx, dx2)  # a gather: the same bits every run
    acc = th.randn_like(dx)
    old = acc.clone()
    _lib.run_op("CUTOUTS_BWD", flags=6, i=dims, f=[0, 0, 0, 0.5, 0.5, 0.5, 1.0], p=[d, cdev, acc])
    assert th.equal(acc, old + dx)


@pytest.mark.parametrize("cs,hw", [(224, (256, 256)), (384, (512, 448))])
def test_cutouts_aug_bwd_fp32_upstream(cs, hw):
    """flags 4 reads the fp32 layout: against flags 0 fed the same values rounded to fp16 in the patch layout with P = cs"""
    H, W, n, B = *hw, 8, 2
    th.manual_seed(5)
    coords = og.MakeCutouts(cs, n)._generate_coords(H, W, n)
    cdev = th.tensor(coords, dtype=th.int32, device="cuda")
    prm = augs.draw_aug_params(coords, B, H, W).cuda()
    d = th.randn(n * B, 3, cs, cs, device="cuda").half().float()
    dims = [B, H, W, n, cs, cs, 3 * cs * cs]
    out = []
    for flags, dd in ((4, d), (0, d.half())):
        dx = th.zeros(B, 3, H, W, device="cuda")
        _lib.run_op("CUTOUTS_AUG_BWD", flags=flags, i=dims, f=[0, 0, 0, 1, 1, 1, 2.0], p=[dd, cdev, dx, prm])
        out.append(dx)
    assert out[0].abs().max() > 0 and _rel(out[0], out[1]) < 1e-5


# ---------------------------------------------------------------------- tv / range
@pytest.mark.parametrize("B", [1, 2, 4])
@pytest.mark.parametrize("size", [64, 256, 512])
def test_tv_range_vs_float64(size, B):
    x = th.randn(B, 3, size, size, device="cuda", generator=th.Generator(device="cuda").manual_seed(size + B)) * 1.3
    d = th.rand(B, device="cuda") + 0.5
    for fn, ref in ((pl.tv_loss, og.tv_loss), (pl.range_loss, og.range_loss)):
        xe, xo = x.clone().requires_grad_(), x.double().requires_grad_()
        v, vo = fn(xe), ref(xo)
        (g,), (go,) = th.autograd.grad(v, xe, d), th.autograd.grad(vo, xo, d.double())
        assert _rel(v, vo) < 2e-6 and _rel(g, go) < 2e-6, (fn.__name__, _rel(v, vo), _rel(g, go))
        assert th.equal(fn(x), v.detach())  # fixed fold order: the same bits every run


# ---------------------------------------------------------------------- spherical
SPH = [(D, n, P) for D in (512, 640, 768, 1024) for n, P in ((2, 1), (1, 3), (1, 65), (4, 4))]


@pytest.mark.parametrize("D,n,P", SPH, ids=[f"D{d}-n{n}-P{p}" for d, n, p in SPH])
def test_spherical_vs_float64(D, n, P):
    g = th.Generator(device="cuda").manual_seed(D + P)
    x, y = th.randn(1, 16, n, D, device="cuda", generator=g), th.randn(1, P, D, device="cuda", generator=g)
    w = th.rand(th.broadcast_shapes((1, 16, n), (1, P)), device="cuda", generator=g)
    res = []
    for fn, a, b in ((pl.spherical_dist_loss, x, y), (og.spherical_dist_loss, x.double(), y.double())):
        a, b = a.clone().requires_grad_(), b.clone().requires_grad_()
        v = fn(a, b)
        res.append((v.detach(), *th.autograd.grad(v, (a, b), w.to(v.dtype))))
    (v, gx, gy), (vo, ox, oy) = res
    assert _rel(v, vo) < 1e-5 and _rel(gx, ox) < 1e-5 and _rel(gy, oy) < 1e-5, (_rel(v, vo), _rel(gx, ox), _rel(gy, oy))
    assert th.equal(pl.spherical_dist_loss(x, y), v)


# ---------------------------------------------------------------------- the reference's closure on the device
@pytest.mark.parametrize("name", list(CASES))
def test_closure_goldens_on_device(name):
    c = CASES[name]
    clip = StubClip(32, 16)
    clip.w = clip.w.cuda()
    ns = types.SimpleNamespace(
        diffusion=types.SimpleNamespace(sqrt_one_minus_alphas_cumprod={c["t"]: GOLD[name + "_fac"][0]}), current_timestep=c["t"],
        make_cutouts=MakeCutouts(32, c["cutn"], cutout_size_power=c["pow"]), clip_util=clip_util, losses=pl, clip_model=clip,
        target_embeds=th.from_numpy(GOLD[name + "_target"]).cuda(), weights=th.from_numpy(GOLD[name + "_weights"]).cuda(),
        num_cutouts=c["cutn"], clip_guidance_scale=1000, tv_scale=150, range_scale=50, sat_scale=c["sat"], use_magnitude=c["mag"])
    th.manual_seed(c["seed"])
    x = th.from_numpy(GOLD[name + "_x"]).cuda().requires_grad_()
    got = reference_style_cond_fn(ns)(x, th.full((c["B"],), c["t"]), {"pred_xstart": stub_pred_xstart(x)})
    r = _rel(got.cpu(), th.from_numpy(GOLD[name + "_grad"]))
    print(f"\nclosure golden {name} on the device: rel-to-max {r:.2e}")
    assert r < 1e-4, r


# ---------------------------------------------------------------------- invariants
def test_invariants():
    x = th.rand(2, 3, 256, 256, device="cuda")
    mk = MakeCutouts(224, 16)
    th.manual_seed(4)
    mk.cache_coordinates(256, 256)
    d = th.randn(32, 3, 224, 224, device="cuda")
    xe = x.clone().requires_grad_()
    cuts = mk(xe, use_cache=True)
    grads = {k: th.autograd.grad(cuts, xe, d * 2.0 ** k, retain_graph=True)[0] for k in (-20, 0, 20)}
    assert grads[0].abs().max() > 0 and all(th.equal(grads[k], grads[0] * 2.0 ** k) for k in (-20, 20))
    assert th.equal(th.autograd.grad(cuts, xe, d)[0], grads[0])  # retain_graph: the same bits again
    for fn in (pl.tv_loss, pl.range_loss):
        v = fn(xe * 3 - 1)
        dl = th.rand(2, device="cuda") + 0.5
        gs = {k: th.autograd.grad(v, xe, dl * 2.0 ** k, retain_graph=True)[0] for k in (-20, 0, 20)}
        assert all(th.equal(gs[k], gs[0] * 2.0 ** k) for k in (-20, 20)), fn.__name__
    with th.no_grad():
        plain = mk(xe, use_cache=True)
        assert plain.grad_fn is None and pl.tv_loss(xe).grad_fn is None and pl.spherical_dist_loss(xe[:, 0], xe[:, 1]).grad_fn is None
    # a no-grad call returns what the stand-alone CUTOUTS_FWD flags 1 launch writes, bit for bit
    today = th.empty(32, 3, 224, 224, device="cuda")
    cdev = th.tensor(mk.cached_coords, dtype=th.int32, device="cuda")
    _lib.run_op("CUTOUTS_FWD", flags=1, i=[2, 256, 256, 16, 224, 224, 3 * 224 * 224], f=[0.5] * 6, p=[x, cdev, today])
    assert th.equal(plain, today) and th.equal(cuts.detach(), today)
    # dtypes follow the input; errors for other devices and dtypes
    xh = x.half().requires_grad_()
    (gh,) = th.autograd.grad(mk(xh, use_cache=True).sum() + pl.tv_loss(xh).sum(), xh)
    assert gh.dtype == th.float16
    with pytest.raises(_lib.CgdError, match="GPU only"):
        pl.range_loss(x.cpu())
    with pytest.raises(_lib.CgdError, match="GPU only"):
        mk(x.cpu(), use_cache=True)
    with pytest.raises(ValueError, match="floating-point"):
        mk(x.int(), use_cache=True)
    with pytest.raises(ValueError, match="x is on"):
        pl.spherical_dist_loss(th.randn(2, 8, device="cuda"), th.randn(2, 8))
    with pytest.raises(RuntimeError, match="differentiate twice|does not require grad"):
        (gg,) = th.autograd.grad(pl.tv_loss(xe).sum(), xe, create_graph=True)
        th.autograd.grad(gg.sum(), xe)


# ---------------------------------------------------------------------- cfg2-size steps
def _cfg2():
    from clip_guided_diffusion_b200 import guidance as pg
    from clip_guided_diffusion_b200 import unet as pu
    from clip_guided_diffusion_b200 import vit as pv
    from clip_guided_diffusion_b200 import weights as pw
    from oracle.clip_vit import VIT_CONFIGS, CLIPVisualOnly
    from oracle.unet import UNetModel, config_for
    ucfg, vcfg = pu.config_for(256, True), pv.VIT_CONFIGS["ViT-B/32"]
    usd, vsd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234), pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 1235)
    eng = pg.GuidedStepB200(ucfg, usd, batch=1, device="cuda", input_grad=True)
    clip_model, clip_size = clip_util.load_clip("ViT-B/32", "cuda", clip_state_dict=vsd)
    ounet = UNetModel(config_for(256, True)).eval()
    ounet.load_state_dict(usd)
    oclip = CLIPVisualOnly(VIT_CONFIGS["ViT-B/32"]).eval()
    oclip.load_state_dict(vsd)
    ounet, oclip = ounet.cuda(), oclip.cuda()
    for prm in list(ounet.parameters()) + list(oclip.parameters()):
        prm.requires_grad_(False)
    return types.SimpleNamespace(ucfg=ucfg, vcfg=vcfg, usd=usd, vsd=vsd, eng=eng, clip_model=clip_model, clip_size=clip_size, ounet=ounet, oclip=oclip)


def _step(odiff, mode, model, ns, x, y):
    cf = reference_style_cond_fn(ns)
    seen = {}

    def cond_fn(xx, tt, out, y=None):
        seen["g"] = cf(xx, tt, out, y=y)
        return seen["g"]
    th.manual_seed(21)
    fn = odiff.p_sample_with_grad if mode == "ancestral" else odiff.ddim_sample_with_grad
    o = fn(model, x, th.full((1,), 14, dtype=th.long, device="cuda"), clip_denoised=False, cond_fn=cond_fn, model_kwargs={"y": y})
    return dict(o, g=seen["g"].detach(), terms={k: float(v) for k, v in ns.terms.items()})


def _ns(odiff, make_cutouts, normalize, losses, clip_model, tgt, **kw):
    return types.SimpleNamespace(diffusion=odiff, current_timestep=14, make_cutouts=make_cutouts, clip_util=normalize, losses=losses,
                                 clip_model=clip_model, target_embeds=tgt, weights=th.ones(1, device="cuda"), num_cutouts=16,
                                 clip_guidance_scale=1000, tv_scale=150, range_scale=50, sat_scale=0, use_magnitude=False, **kw)


@pytest.mark.parametrize("mode", ["ancestral", "ddim"])
def test_cfg2_step_everything_on_the_package(mode):
    from clip_guided_diffusion_b200 import gaussian_diffusion as pgd
    from clip_guided_diffusion_b200 import guidance as pg
    from clip_guided_diffusion_b200 import lpips as plp
    from oracle import diffusion as od
    from oracle import lpips as ol
    from tests.test_gpu_lpips_autograd import _natural
    m = _cfg2()
    lsd = ol.seeded_state_dict()
    odiff = od.create_gaussian_diffusion(1000, "linear", "ddim25" if mode == "ddim" else "25")
    th.manual_seed(0)
    tgt = th.randn(1, 512, device="cuda")
    coords = og.MakeCutouts(224, 16)._generate_coords(256, 256, 16)
    g = th.Generator().manual_seed(3)
    x, y = th.randn(1, 3, 256, 256, generator=g).cuda(), th.randint(0, 1000, (1,), generator=g).cuda()
    init = _natural(1, 256, 7)
    mk = MakeCutouts(m.clip_size, 16)
    mk.cached_coords = coords
    omk = og.MakeCutouts(224, 16)
    e = _step(odiff, mode, m.eng.model, _ns(odiff, lambda t, **kw: mk(t, use_cache=True, **kw), clip_util, pl, m.clip_model, tgt,
                                           lpips_vgg=plp.LPIPS(net="vgg", lpips_state_dict=lsd).to("cuda"), init_tensor=init, init_scale=1000.0), x, y)
    o = _step(odiff, mode, m.ounet, _ns(odiff, lambda t, **kw: omk(t, coords=coords, **kw), types.SimpleNamespace(CLIP_NORMALIZE=og.clip_normalize),
                                       og, m.oclip, tgt, lpips_vgg=ol.LPIPSVgg({k: v.cuda() for k, v in lsd.items()}).cuda(), init_tensor=init,
                                       init_scale=1000.0), x, y)
    vals = (_cos(e["g"], o["g"]), _rel(e["g"], o["g"]), _rel(e["pred_xstart"], o["pred_xstart"]), _rel(e["sample"], o["sample"]))
    print(f"\ncfg2-size {mode} step, every piece on the package vs the fp32 oracle: cos(g) {vals[0]:.5f} rel(g) {vals[1]:.3e} "
          f"rel(pred_xstart) {vals[2]:.3e} rel(sample) {vals[3]:.3e} terms {e['terms']} vs {o['terms']}")
    assert vals[0] > 0.995 and vals[1] < 2e-2 and vals[2] < 2e-2 and vals[3] < 2e-2, vals
    del m
    th.cuda.empty_cache()
    from clip_guided_diffusion_b200 import unet as pu
    from clip_guided_diffusion_b200 import vit as pv
    from clip_guided_diffusion_b200 import weights as pw
    ucfg, vcfg = pu.config_for(256, True), pv.VIT_CONFIGS["ViT-B/32"]
    pdiff = pgd.create_gaussian_diffusion(1000, "linear", "ddim25" if mode == "ddim" else "25")
    feng = pg.GuidedStepB200(ucfg, pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234), vcfg, pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 1235),
                             batch=1, num_cutouts=16, device="cuda", lpips_sd=lsd, init_scale=1000.0)
    feng.set_targets(tgt, th.ones(1))
    feng.set_init_image(init)
    feng.stage_step(pdiff.scalar_table(14, 14, 0.0), coords, pdiff.model_timestep(14), y)
    feng.img(feng.unet.x_in).copy_(x)
    feng.img(feng.noise).zero_()
    feng.replay(mode, 16)
    th.cuda.synchronize()
    f = dict(g=feng.img(feng.g).float().clone(), pred_xstart=feng.img(feng.x0).float().clone())
    fused = (_cos(e["g"], f["g"]), _rel(e["g"], f["g"]), _rel(e["pred_xstart"], f["pred_xstart"]))
    print(f"cfg2-size {mode} step, every piece on the package vs the fused CondFnB200: cos(g) {fused[0]:.5f} rel(g) {fused[1]:.3e} "
          f"rel(pred_xstart) {fused[2]:.3e}")
    assert fused[0] > 0.995 and fused[1] < 2e-2 and fused[2] < 2e-2, fused


def test_cfg2_use_augs_step_vs_oracle():
    from oracle import diffusion as od
    m = _cfg2()
    odiff = od.create_gaussian_diffusion(1000, "linear", "ddim25")
    th.manual_seed(0)
    tgt = th.randn(1, 512, device="cuda")
    g = th.Generator().manual_seed(3)
    x, y = th.randn(1, 3, 256, 256, generator=g).cuda(), th.randint(0, 1000, (1,), generator=g).cuda()
    mk = MakeCutouts(m.clip_size, 16, use_augs=True)
    drawn = {}

    def oracle_cutouts(t, num_cutouts_override=None):
        th.manual_seed(77)  # the draws the package's call made: windows, then per cutout the parameters and the noise (CUDA generator)
        coords = mk._generate_coords(256, 256, 16)
        noise = th.zeros(16, 4, 1, 3, 256, 256, device="cuda")
        prm = augs.draw_aug_params(coords, 1, 256, 256, noise_device="cuda", noise_out=noise)
        drawn["coords"] = coords
        return og.MakeCutouts(224, 16)(t, coords=coords, aug_params=prm, aug_noise=noise)

    def package_cutouts(t, num_cutouts_override=None):
        th.manual_seed(77)
        return mk(t, num_cutouts_override=num_cutouts_override)
    e = _step(odiff, "ddim", m.eng.model, _ns(odiff, package_cutouts, clip_util, pl, m.clip_model, tgt), x, y)
    o = _step(odiff, "ddim", m.ounet, _ns(odiff, oracle_cutouts, types.SimpleNamespace(CLIP_NORMALIZE=og.clip_normalize), og, m.oclip, tgt), x, y)
    vals = (_cos(e["g"], o["g"]), _rel(e["g"], o["g"]), _rel(e["pred_xstart"], o["pred_xstart"]), _rel(e["sample"], o["sample"]))
    print(f"\ncfg2-size use_augs ddim step vs the fp32 oracle with the same draws: cos(g) {vals[0]:.5f} rel(g) {vals[1]:.3e} "
          f"rel(pred_xstart) {vals[2]:.3e} rel(sample) {vals[3]:.3e}")
    assert len(drawn["coords"]) == 16
    assert vals[0] > 0.995 and vals[1] < 2e-2 and vals[2] < 2e-2 and vals[3] < 2e-2, vals
