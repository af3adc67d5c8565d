"""GPU: the engine's UNet under torch.autograd (GuidedStepB200(..., input_grad=True)) on the H100.

The three bridge kernels one by one against float64 references (GRAD_SEED and GRAD_UNSCALE bit for bit, PMV_BWD within a few fp32
ulps, with all-zero images, inf and NaN in the inputs), `model()`'s input gradient against the fp32 oracle UNet at the tiny, 64x64 and
256x256 architectures, the oracle's *_with_grad steps at cfg2's size with model = engine.model, a 25-step chain of the package's loop
with a plain PyTorch cond_fn, and a fused step after a generic one on the same engine."""
from __future__ import annotations

import numpy as np
import pytest
import torch as th

from clip_guided_diffusion_b200 import _lib
from clip_guided_diffusion_b200 import gaussian_diffusion as pgd
from clip_guided_diffusion_b200 import guidance as pg
from clip_guided_diffusion_b200 import unet as pu
from clip_guided_diffusion_b200 import vit as pv
from clip_guided_diffusion_b200 import weights as pw
from clip_guided_diffusion_b200._lib import SC
from oracle import diffusion as od
from oracle import guidance as og
from tests.step_parity import cos, prod_unet_cfg, psnr, rel

pytestmark = pytest.mark.gpu
LD = pu.IN_PAD
SENTINEL = 7.0  # seed channels 6.. must be left alone


# ---------------------------------------------------------------------- 1. kernels
def _d_out(B, HW, seed):
    g = th.Generator().manual_seed(seed)
    d = th.randn(B, 6, HW, generator=g) * th.exp2(th.randint(-30, 30, (B, 1, 1), generator=g).float())
    if B > 1:
        d[0] = 0.0  # an all-zero image: scale 1
    d[-1, 4, 7] = float("inf")
    d[-1, 1, 3] = float("nan")
    return d


def _scale_ref(m: np.ndarray) -> np.ndarray:
    """SEED_QUANT's rule in float64: the largest element lands in (2048, 4096], exponent clamped to +-60"""
    with np.errstate(divide="ignore"):
        e = np.clip(np.floor(np.log2(4096.0 / m.astype(np.float64))), -60, 60)
    return np.where(m > 0, np.exp2(e), 1.0).astype(np.float32)


@pytest.mark.parametrize("B", [1, 2, 8])
@pytest.mark.parametrize("size", [64, 256, 512])
def test_bridge_kernels(size, B):
    HW = size * size
    d = _d_out(B, HW, seed=size + B)
    dev = d.cuda()
    dyn = th.zeros(2 * B, device="cuda")
    seed = th.full((B, HW, LD), SENTINEL, dtype=th.float16, device="cuda")
    _lib.run_op("GRAD_SEED", i=[B, HW, LD], p=[dev, dyn, seed])
    th.cuda.synchronize()
    dn = d.numpy()
    a = np.abs(dn).reshape(B, -1)
    m = np.minimum(np.where(np.isnan(a), 0, a).max(1), np.float32(3.0e38)).astype(np.float32)
    dyn_h = dyn.cpu().numpy()
    assert np.array_equal(dyn_h[:B], m), (dyn_h[:B], m)
    scale = _scale_ref(m)
    assert np.array_equal(dyn_h[B:], scale), (dyn_h[B:], scale)
    ok = m > 0
    assert np.all((m * scale)[ok & (m < 1e30)] > 2048) and np.all((m * scale)[ok & (m < 1e30)] <= 4096)
    v = np.nan_to_num(dn * scale[:, None, None], nan=-60000.0, posinf=np.inf, neginf=-np.inf)  # the kernel's fmaxf turns NaN into -60000
    want = np.clip(v, -60000, 60000).astype(np.float16).transpose(0, 2, 1)
    got = seed.cpu().numpy()
    assert np.array_equal(got[:, :, :6].view(np.uint16), want.view(np.uint16))
    assert np.all(got[:, :, 6:] == SENTINEL)

    for direct in (False, True):
        g = th.Generator().manual_seed(7 + direct)
        dxu, dxd = th.randn(B, 3, HW, generator=g) * 1e3, th.randn(B, 3, HW, generator=g)
        dx = th.empty(B, 3, HW, device="cuda")
        dyn_c, seed_c = dyn.clone(), seed.clone()
        _lib.run_op("GRAD_UNSCALE", i=[B, HW, LD], p=[dxu.cuda(), dxd.cuda() if direct else None, dyn_c, seed_c, dx])
        th.cuda.synchronize()
        ref = dxu.numpy() * (np.float32(1.0) / scale)[:, None, None]
        if direct:
            ref = (ref + dxd.numpy()).astype(np.float32)
        assert np.array_equal(dx.cpu().numpy(), ref)
        assert np.all(dyn_c[:B].cpu().numpy() == 0) and np.array_equal(dyn_c[B:].cpu().numpy(), scale)
        sc = seed_c.cpu().numpy()
        assert np.all(sc[:, :, :6] == 0) and np.all(sc[:, :, 6:] == SENTINEL)

    diff = pgd.create_gaussian_diffusion(1000, "linear", "25")
    s = th.from_numpy(diff.scalar_table(11, 11))
    g = th.Generator().manual_seed(size * 3 + B)
    var = th.rand(B, 3, HW, generator=g) + 0.01
    ups = [th.randn(B, 3, HW, generator=g) for _ in range(4)]
    for present in ((True, False, False, False), (False, True, False, False), (False, False, True, False), (False, False, False, True),
                    (True, True, True, True)):
        gs = [u.cuda() if p else None for u, p in zip(ups, present)]
        d_out, dxd = th.empty(B, 6, HW, device="cuda"), th.empty(B, 3, HW, device="cuda")
        _lib.run_op("PMV_BWD", i=[B, HW], p=[s.cuda(), var.cuda(), *gs, d_out, dxd])
        th.cuda.synchronize()
        k = {n: float(s[SC[n]]) for n in SC if n != "COUNT"}
        z = np.zeros((B, 3, HW))
        gx0, gm, gv, gl = (u.double().numpy() if p else z for u, p in zip(ups, present))
        G = gx0 + k["POST_COEF1"] * gm
        hr = (np.float64(np.float32(k["MAX_LOG"]) - np.float32(k["MIN_LOG"]))) * 0.5
        lv = gl + var.double().numpy() * gv
        refs = [(-k["SQRT_RECIPM1_AC"] * G, abs(k["SQRT_RECIPM1_AC"]) * (np.abs(gx0) + abs(k["POST_COEF1"]) * np.abs(gm))),
                (hr * lv, abs(hr) * (np.abs(gl) + var.double().numpy() * np.abs(gv))),
                (k["SQRT_RECIP_AC"] * G + k["POST_COEF2"] * gm,
                 abs(k["SQRT_RECIP_AC"]) * (np.abs(gx0) + abs(k["POST_COEF1"]) * np.abs(gm)) + abs(k["POST_COEF2"]) * np.abs(gm))]
        gots = [d_out[:, :3].double().cpu().numpy(), d_out[:, 3:].double().cpu().numpy(), dxd.double().cpu().numpy()]
        for got_, (ref_, mag) in zip(gots, refs):
            err = np.abs(got_ - ref_)
            assert np.all(err <= 4 * np.finfo(np.float32).eps * mag + 1e-30), (present, float((err / (mag + 1e-30)).max()))


# ---------------------------------------------------------------------- 2. model() input gradient
def _arch(name):
    from oracle.unet import UNetModel, config_for, seeded_init_, tiny_config
    if name == "tiny":
        ocfg = tiny_config(image_size=64, model_channels=64, channel_mult=(1, 2), num_res_blocks=1, attention_resolutions=(32,), class_cond=True)
        ounet = seeded_init_(UNetModel(ocfg)).eval()
        return prod_unet_cfg(ocfg), ounet.state_dict(), ounet, 2
    size = {"cfg1_64": 64, "full_256": 256}[name]
    ucfg = pu.config_for(size, True)
    usd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234)
    ounet = UNetModel(config_for(size, True)).eval()
    ounet.load_state_dict(usd)
    return ucfg, usd, ounet, 1


@pytest.mark.parametrize("name", ["tiny", "cfg1_64", "full_256"])
def test_model_input_gradient_vs_oracle(name):
    ucfg, usd, ounet, B = _arch(name)
    eng = pg.GuidedStepB200(ucfg, usd, batch=B, device="cuda", input_grad=True)
    ounet = ounet.cuda()
    for prm in ounet.parameters():
        prm.requires_grad_(False)
    g = th.Generator().manual_seed(1)
    S = ucfg.image_size
    x, w = th.randn(B, 3, S, S, generator=g).cuda(), th.randn(B, 6, S, S, generator=g).cuda()
    t, y = th.full((B,), 400.0, device="cuda"), th.randint(0, ucfg.num_classes, (B,), generator=g).cuda()
    xe = x.clone().requires_grad_()
    out = eng.model(xe, t, y)
    (ge,) = th.autograd.grad((w * out).sum(), xe, retain_graph=True)
    (ge2,) = th.autograd.grad((w * out).sum(), xe)
    xo = x.clone().requires_grad_()
    (go,) = th.autograd.grad((w * ounet(xo, t, y=y)).sum(), xo)
    c, r = cos(ge, go), rel(ge, go)
    print(f"\nmodel() input gradient {name}: cos {c:.6f} rel {r:.3e}")
    assert th.equal(ge, ge2), "the UNet backward is not repeatable (retain_graph=True)"
    assert c >= 0.999 and r <= 2e-2, (c, r)


# ---------------------------------------------------------------------- 3. the oracle's steps at cfg2's size
@pytest.mark.parametrize("mode", ["ancestral", "ddim"])
def test_oracle_steps_cfg2_size(mode):
    from oracle.clip_vit import VIT_CONFIGS, CLIPVisualOnly
    from oracle.unet import UNetModel, config_for
    ucfg, vcfg = pu.config_for(256, True), pv.VIT_CONFIGS["ViT-B/32"]
    usd, vsd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234), pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 1235)
    eng = pg.GuidedStepB200(ucfg, usd, batch=1, device="cuda", input_grad=True)
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
    res = []
    for model in (eng.model, ounet):
        cf = og.OracleCondFn(odiff, oclip, tgt, th.ones(1, device="cuda"), cut_size=224, num_cutouts=16)
        cf.current_timestep = 14
        seen = {}

        def cond_fn(xx, tt, out, y=None, cf=cf, seen=seen):
            seen["g"] = cf(xx, tt, out, y=y, coords=coords)
            return seen["g"]
        th.manual_seed(21)
        fn = odiff.p_sample_with_grad if mode == "ancestral" else odiff.ddim_sample_with_grad
        o = fn(model, x, th.full((1,), 14, dtype=th.long, device="cuda"), clip_denoised=False, cond_fn=cond_fn, model_kwargs={"y": y})
        res.append(dict(o, g=seen["g"].detach()))
    e, o = res
    vals = (cos(e["g"], o["g"]), rel(e["pred_xstart"], o["pred_xstart"]), rel(e["sample"], o["sample"]))
    print(f"\ncfg2-size {mode} step, engine.model vs oracle UNet: cos(g) {vals[0]:.5f} rel(pred_xstart) {vals[1]:.3e} rel(sample) {vals[2]:.3e}")
    assert vals[0] > 0.995 and vals[1] < 2e-2 and vals[2] < 2e-2, vals


# ---------------------------------------------------------------------- 4. 25-step chain of the package's loop, generic cond_fn
def _tiny_tower(input_grad=True):
    from oracle.clip_vit import CLIPVisualOnly, ViTConfig as OViTConfig
    from oracle.unet import UNetModel, seeded_init_, tiny_config
    ocfg = tiny_config(image_size=64, model_channels=64, channel_mult=(1, 2), num_res_blocks=1, attention_resolutions=(32,), class_cond=True)
    ounet = seeded_init_(UNetModel(ocfg)).eval()
    oclip = seeded_init_(CLIPVisualOnly(OViTConfig(32, 16, 128, 2, 64)), seed=5).eval()
    for prm in list(ounet.parameters()) + list(oclip.parameters()):
        prm.requires_grad_(False)
    eng = pg.GuidedStepB200(prod_unet_cfg(ocfg), ounet.state_dict(), pv.ViTConfig(32, 16, 128, 2, 64), oclip.state_dict(), batch=2, num_cutouts=3,
                            use_magnitude=True, device="cuda", input_grad=input_grad)
    tgt = th.randn(1, 64, generator=th.Generator().manual_seed(99))
    eng.set_targets(tgt, th.ones(1))
    return eng, ounet.cuda(), oclip.cuda(), tgt.cuda()


@pytest.mark.parametrize("mode", ["ancestral", "ddim"])
def test_package_loop_generic_cond_fn_chain(mode):
    eng, ounet, oclip, tgt = _tiny_tower()
    odiff, pdiff = od.create_gaussian_diffusion(1000, "linear", "25"), pgd.create_gaussian_diffusion(1000, "linear", "25")
    outs = []
    for diff, model in ((pdiff, eng.model), (odiff, ounet)):
        cf = og.OracleCondFn(odiff, oclip, tgt, th.ones(1, device="cuda"), cut_size=32, num_cutouts=3, use_magnitude=True)
        th.manual_seed(11)  # x_T, the noise (device generator) and the cutout windows (CPU generator) drawn alike on both sides
        name = "p_sample_loop_progressive" if mode == "ancestral" else "ddim_sample_loop_progressive"
        seq = []
        for out in getattr(diff, name)(model, (2, 3, 64, 64), clip_denoised=False, cond_fn=cf, cond_fn_with_grad=True, device="cuda",
                                       model_kwargs={"y": th.tensor([1, 2], device="cuda")}):
            cf.step_done()
            seq.append((out["sample"].detach().float().cpu(), out["pred_xstart"].detach().float().cpu()))
        outs.append(seq)
    assert len(outs[0]) == len(outs[1]) == 25
    drift = [rel(e[0], o[0]) for e, o in zip(*outs)]
    res = dict(drift_max=max(drift), psnr_sample=psnr(outs[0][-1][0], outs[1][-1][0]), psnr_x0=psnr(outs[0][-1][1], outs[1][-1][1]))
    print(f"\n25-step {mode} chain, package loop + PyTorch cond_fn vs oracle: {res}")
    assert th.isfinite(outs[0][-1][0]).all() and res["drift_max"] < 3e-2 and res["psnr_sample"] > 40.0 and res["psnr_x0"] > 40.0, res


# ---------------------------------------------------------------------- 5. a fused step after a generic one
def _fused(eng, pdiff, x, y, noise, coords):
    eng.stage_step(pdiff.scalar_table(14, 14, 0.0), coords, pdiff.model_timestep(14), y)
    eng.img(eng.unet.x_in).copy_(x)
    eng.img(eng.noise).copy_(noise)
    eng.replay("ddim", 3)
    th.cuda.synchronize()
    return eng.img(eng.sample).clone(), eng.img(eng.g).clone(), eng.img(eng.x0).clone()


def test_fused_step_after_generic_step_is_unchanged():
    eng, _, oclip, tgt = _tiny_tower()
    pdiff, odiff = pgd.create_gaussian_diffusion(1000, "linear", "25"), od.create_gaussian_diffusion(1000, "linear", "25")
    g = th.Generator().manual_seed(5)
    x, noise = th.randn(2, 3, 64, 64, generator=g).cuda(), th.randn(2, 3, 64, 64, generator=g).cuda()
    y, coords = th.tensor([3, 4], device="cuda"), [(0, 0, 64), (5, 9, 40), (20, 3, 33)]
    cf = og.OracleCondFn(odiff, oclip, tgt, th.ones(1, device="cuda"), cut_size=32, num_cutouts=3)
    cf.current_timestep = 20
    for mode in ("ancestral", "ddim"):  # generic steps leave the shared seed / maxima as they found them
        fn = pdiff.p_sample_with_grad if mode == "ancestral" else pdiff.ddim_sample_with_grad
        fn(eng.model, x * 0.3, th.full((2,), 20, dtype=th.long), clip_denoised=False, model_kwargs={"y": y},
           cond_fn=lambda xx, tt, out, y=None: cf(xx, tt, out, y=y, coords=coords))
    after = _fused(eng, pdiff, x, y, noise, coords)
    fresh = _fused(_tiny_tower()[0], pdiff, x, y, noise, coords)
    assert all(th.equal(a, b) for a, b in zip(after, fresh))
