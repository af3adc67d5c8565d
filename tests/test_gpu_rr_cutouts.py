"""GPU: ResizeRight (lanczos3) cutouts on non-square images, with progressive cutout counts and after the use_augs pipeline.

* Every launch signature the new modes make at production sizes (tests/test_rr_cutouts_cpu.py asserts the list below covers them), one
  launch at a time: CUTOUTS_RR_FWD / _BWD flags 1 (x-axis tables) and 2 (augmented-crop workspace) against float64 with the bound form of
  tests/test_gpu_lpips_cutout_kernels.py (one fp16 ulp plus taps x u x magnitude); CUTOUTS_AUG_FWD / _BWD flags 1 against the fp32
  torchvision pipeline (oracle.guidance.apply_augs: its nearest-neighbour and bilinear index decisions are fp32 decisions, which a float64
  twin would not reproduce).  Workspaces, outputs and unused table slots are NaN before the launch.
* Teacher-forced full-size steps (cfg2 architecture) against the fp32 oracle, graph replay against eager for every cutout count, and a
  free-running 25-step chain at 64 x 96."""
import math

import pytest
import torch as th

from clip_guided_diffusion_b200 import resize_right as rr
from clip_guided_diffusion_b200.augs import draw_aug_params
from clip_guided_diffusion_b200.guidance import CLIP_MEAN, CLIP_STD
from clip_guided_diffusion_b200.plan import Plan
from oracle import guidance as og
from tests.kernel_check import D64, U, check, run, ulp16
from tests.rr_cutouts import AugResizeMakeCutouts, axis_matrix, crops

# (B, H, W, cutn, cs, patch, Kpad, use_augs): the production geometries of tests/test_rr_cutouts_cpu.py PROD
B32, B16, L14, L14_336 = (224, 32, 3072), (224, 16, 768), (224, 14, 640), (336, 14, 640)
CASES = {
    "b32-256x320": (1, 256, 320, 16, *B32, False), "b32-320x256": (1, 320, 256, 16, *B32, False), "b32-192x256": (1, 192, 256, 16, *B32, False),
    "b32-256-c4": (1, 256, 256, 4, *B32, False), "b32-256-c8": (1, 256, 256, 8, *B32, False), "b32-256-c16": (1, 256, 256, 16, *B32, False),
    "b32-256-augs": (1, 256, 256, 16, *B32, True), "b32-256x320-augs": (1, 256, 320, 16, *B32, True),
    "b32-320x256-augs": (1, 320, 256, 16, *B32, True),
    "b16-512-augs-c4": (1, 512, 512, 4, *B16, True), "b16-512-augs-c8": (1, 512, 512, 8, *B16, True), "b16-512-augs": (1, 512, 512, 16, *B16, True),
    "b16-512x576": (1, 512, 576, 16, *B16, False),
    "l14-256x320-augs": (1, 256, 320, 16, *L14, True), "l14-336-512x448-augs": (1, 512, 448, 16, *L14_336, True),
    "hand-B2-96x64-augs-kpad": (2, 96, 64, 5, 32, 4, 64, True), "hand-B2-64x100-kpad": (2, 64, 100, 6, 64, 2, 16, False),
}


def check_mostly(what, got, ref, tol, max_frac=1e-4):
    """check() that lets a fraction `max_frac` of the elements miss `tol` (but not be NaN): torchvision's affine step samples the nearest
    pixel, and a source coordinate within a few fp32 ulps of a half-integer rounds one way in the kernel's arithmetic order and the other
    way in torchvision's, which moves that one sample (and, in the backward, that one scatter) to the neighbouring pixel"""
    got, ref = got.to(D64), ref.to(D64)
    bad = ~((got - ref).abs() <= tol)
    assert not bool(got.isnan().any()), f"{what}: NaN"
    assert int(bad.sum()) <= max_frac * bad.numel(), f"{what}: {int(bad.sum())} of {bad.numel()} elements outside tolerance"


def case_signatures(case) -> set:
    """(code, flags, B, H, W, cutn, cs, patch, Kpad, Smax | 0) of the launches one case runs (tests/test_rr_cutouts_cpu.py's form)"""
    B, H, W, cutn, cs, P, kpad, augs = case
    geo, S, xf = (B, H, W, cutn, cs, P, kpad), min(H, W), 1 if H != W else 0
    if augs:
        return {("CUTOUTS_AUG_FWD", 1, *geo, S), ("CUTOUTS_RR_FWD", 2 | xf, *geo, S), ("CUTOUTS_RR_BWD", 2 | xf, *geo, S), ("CUTOUTS_AUG_BWD", 1, *geo, S)}
    return {("CUTOUTS_RR_FWD", xf, *geo, 0), ("CUTOUTS_RR_BWD", xf, *geo, S)}


def covered_signatures() -> set:
    return set().union(*(case_signatures(c) for c in CASES.values()))


def windows(H, W, cs, cutn, seed, sliver=1):
    """the whole image's largest window, windows clipped to slivers at the right and bottom border (down to `sliver` pixels: up-sampling),
    one at S == cs when it fits, then the reference's own draws with swapped sides (cgd/modules.py:52) whose crop is not empty"""
    mx, mn = min(H, W), min(H, W, cs)
    out = [(0, 0, mx), (W - sliver, 0, mx), (0, H - sliver - 2, mx), (W - sliver, H - sliver, mn), (W - mn, H - mn, mn)]
    if H == W:  # a square image's windows lie inside it (the swapped sides are equal): one table set serves both axes
        out = [(0, 0, mx), (W - mn, H - mn, mn)]
    g = th.Generator().manual_seed(seed)
    while len(out) < cutn:
        s = int(th.rand([], generator=g) * (mx - mn) + mn)
        ox, oy = int(th.randint(0, H - s + 1, (), generator=g)), int(th.randint(0, W - s + 1, (), generator=g))
        if ox < W and oy < H:
            out.append((ox, oy, s))
    return out[:cutn]


def axis_tables(ext, cs, Smax):
    """device tables of one axis for the crop extents `ext` (one per cutout): weight slots past T are NaN, inverse rows past the extent
    are empty"""
    n = len(ext)
    left, wt = th.zeros(n, cs, dtype=th.int32), th.full((n, cs, rr.T_MAX), math.nan)
    taps, inv = th.zeros(n, dtype=th.int32), th.tensor([1, 0], dtype=th.int32).repeat(n, Smax, 1)
    mats = []
    for k, S in enumerate(ext):
        l, w, T = rr.tables(S, cs)
        left[k], taps[k] = l, T
        wt[k, :, :T] = w[:, :T]
        inv[k, :S] = rr.inverse_ranges(l, T, S)
        mats.append(axis_matrix(l, w, T, S, cs, D64))
    return (left, wt, taps, inv), mats


def to_patches(img, P, kpad):
    n, _, cs, _ = img.shape
    g = cs // P
    t = img.reshape(n, 3, g, P, g, P).permute(0, 2, 4, 1, 3, 5).reshape(n, g * g, 3 * P * P)
    return th.nn.functional.pad(t, (0, kpad - 3 * P * P))


def from_patches(t, P, cs):
    n, g = t.shape[0], cs // P
    return t[:, :, :3 * P * P].reshape(n, g, g, 3, P, P).permute(0, 3, 1, 4, 2, 5).reshape(n, 3, cs, cs)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_cutout_launch_vs_reference(name):
    B, H, W, cutn, cs, P, kpad, augs = CASES[name]
    S = min(H, W)
    # use_augs: slivers of 8 px, as torchvision's perspective fit is rank-deficient on a 1-pixel-wide crop (in the reference as well)
    coords = windows(H, W, cs, cutn, seed=H * 7 + W + cutn, sliver=8 if augs else 1)
    cr = crops(coords, H, W)
    ty, Ay = axis_tables([c[3] for c in cr], cs, S)
    tx, Ax = axis_tables([c[4] for c in cr], cs, S)
    rect = H != W
    g = th.Generator().manual_seed(H * W + cutn)
    x = (th.randn(B, 3, H, W, generator=g) * 0.7).float()
    G2 = (cs // P) ** 2
    dpatch = (th.randn(cutn * B, G2, kpad, generator=g) * 0.01).half()
    nan_ws = th.full((cutn, B, 3, S, S), math.nan)
    mean, sd = th.tensor(CLIP_MEAN, dtype=D64).view(1, 3, 1, 1), th.tensor(CLIP_STD, dtype=D64).view(1, 3, 1, 1)
    scale = 0.25
    plan = Plan()
    bx, bc, bo, bd = plan.new(x.numel(), "f"), plan.new(cutn * 3, "i32"), plan.new(cutn * B * G2 * kpad, "h"), plan.new(dpatch.numel(), "h")
    by = [plan.new(t.numel(), "i32" if t.dtype == th.int32 else "f") for t in ty]
    bxt = [plan.new(t.numel(), "i32" if t.dtype == th.int32 else "f") for t in tx] if rect else []
    fwd_t = [(b, 0) for b in by[:3]] + [(b, 0) for b in bxt[:3]]
    bwd_t = [(b, 0) for b in (by[0], by[1], by[3])] + ([(b, 0) for b in (bxt[0], bxt[1], bxt[3])] if rect else [])
    geo, xf = [B, H, W, cutn, cs, P, kpad], 1 if rect else 0
    inputs = [(bx, x), (bc, th.tensor(coords, dtype=th.int32)), (bo, th.full((cutn * B * G2 * kpad,), 7.0).half()), (bd, dpatch)]
    inputs += list(zip(by, ty)) + (list(zip(bxt, tx)) if rect else [])
    if not augs:
        bg = plan.new(x.numel(), "f")
        plan.emit("CUTOUTS_RR_FWD", flags=xf, i=geo, f=[*CLIP_MEAN, *CLIP_STD], p=[(bx, 0), (bc, 0), (bo, 0), *fwd_t])
        plan.emit("CUTOUTS_RR_BWD", flags=xf, i=geo + [S], f=[0, 0, 0, *CLIP_STD, scale], p=[(bd, 0), (bc, 0), (bg, 0), *bwd_t])
        rd = run(plan, "cuda", inputs + [(bg, th.full((x.numel(),), math.nan))])
        src64 = x.to(D64)
    else:
        # one launch each, on its own input: AUG_FWD x -> crops; RR_FWD from a random crop workspace (NaN outside every crop);
        # RR_BWD d patches -> d crops; AUG_BWD from random d crops (NaN outside every crop) into a zeroed dx
        noise = th.zeros(cutn, 4, B, 3, S, S)
        th.manual_seed(11)
        prm = draw_aug_params(coords, B, H, W, noise_out=noise)
        ws_in, dws_in = nan_ws.clone(), nan_ws.clone()
        for k, _, _, sy, sx in cr:
            ws_in[k, :, :, :sy, :sx] = th.rand(B, 3, sy, sx, generator=g)
            dws_in[k, :, :, :sy, :sx] = th.randn(B, 3, sy, sx, generator=g)
        bp, bn, bwa, bwi, bwb, bdi, bg = (plan.new(prm.numel(), "f"), plan.new(noise.numel(), "f"), plan.new(nan_ws.numel(), "f"),
                                          plan.new(nan_ws.numel(), "f"), plan.new(nan_ws.numel(), "f"), plan.new(nan_ws.numel(), "f"),
                                          plan.new(x.numel(), "f"))
        plan.emit("CUTOUTS_AUG_FWD", flags=1, i=geo + [S], p=[(bx, 0), (bc, 0), (bwa, 0), (bp, 0), (bn, 0)])
        plan.emit("CUTOUTS_RR_FWD", flags=2 | xf, i=geo + [S], f=[*CLIP_MEAN, *CLIP_STD], p=[(bwi, 0), (bc, 0), (bo, 0), *fwd_t])
        plan.emit("CUTOUTS_RR_BWD", flags=2 | xf, i=geo + [S], f=[0, 0, 0, *CLIP_STD, scale], p=[(bd, 0), (bc, 0), (bwb, 0), *bwd_t])
        plan.emit("CUTOUTS_AUG_BWD", flags=1, i=geo + [S], f=[0, 0, 0, 1, 1, 1, scale], p=[(bdi, 0), (bc, 0), (bg, 0), (bp, 0)])
        rd = run(plan, "cuda", inputs + [(bp, prm), (bn, noise), (bwa, nan_ws), (bwi, ws_in), (bwb, nan_ws), (bdi, dws_in),
                                         (bg, th.zeros(x.numel()))])
        src64 = ws_in.to(D64)
        # AUG_FWD: every crop pixel against the fp32 pipeline (values in [0, 1] plus noise).  The kernel computes each sampling position in
        # another fp32 order than torchvision's grid, so positions agree to a few ulps of coordinates up to Smax; between neighbouring
        # pixels of random data that moves a bilinear sample by up to ~1e-4 (an index error would be O(1))
        got = rd(bwa, nan_ws.shape)
        x01 = (x + 1) * 0.5
        for k, ox, oy, sy, sx in cr:
            ref = og.apply_augs(x01[:, :, oy:oy + sy, ox:ox + sx], prm[k], noise[k][..., :sy, :sx])
            check_mostly(f"cutouts_aug_fwd crops[{k}]", got[k, :, :, :sy, :sx], ref, 3e-4)
        # AUG_BWD: the fp32 autograd of the pipeline, summed over the crops, times scale; fp32 atomics in another order and bilinear weights
        # from the same few-ulp positions as above
        xr = th.zeros(B, 3, H, W, requires_grad=True)
        tot = sum((og.apply_augs(((xr + 1) * 0.5)[:, :, oy:oy + sy, ox:ox + sx], prm[k]) * dws_in[k, :, :, :sy, :sx]).sum()
                  for k, ox, oy, sy, sx in cr)
        (gref,) = th.autograd.grad(tot, xr)
        gmag = gref.abs().max()
        check_mostly("cutouts_aug_bwd", rd(bg, x.shape), gref * scale, (1e-3 * gref.abs() + 1e-4 * gmag) * scale, max_frac=1e-3)
    # ResizeRight forward: a row pass of T_x fmas and a column pass of T_y fmas, then the normalisation: (T_y + T_x + 8) u of the magnitude
    Tmax = int(max(ty[2].max(), tx[2].max()))

    def resized(src, absval=False):
        out = []
        for k, ox, oy, sy, sx in cr:
            c = src[k, :, :, :sy, :sx] if augs else src[:, :, oy:oy + sy, ox:ox + sx]
            ay, ax = (Ay[k].abs(), Ax[k].abs()) if absval else (Ay[k], Ax[k])
            out.append(ay @ (c.abs() if absval else c) @ ax.t())
        return th.cat(out)
    # the image mode resamples x in [-1, 1] and maps (acc + 1) / 2; the crop mode resamples the augmented crop in [0, 1]
    to01 = (lambda v: v) if augs else (lambda v: (v + 1) / 2)  # noqa: E731
    ref = to_patches((to01(resized(src64)) - mean) / sd, P, kpad)
    mag = to_patches((to01(resized(src64, True)) + mean) / sd, P, kpad)
    got = rd(bo, (cutn * B, G2, kpad))
    check("cutouts_rr_fwd", got, ref, ulp16(ref) + (2 * Tmax + 8) * U * mag)
    assert bool((got[:, :, 3 * P * P:] == 0).all()), "patch-vector padding not zeroed"
    # backward: per crop pixel a gather over <= T outputs per axis, two fmas deep, then two products; summed over the crops holding an
    # image pixel in the image-space form
    dimg = from_patches(dpatch.to(D64), P, cs).view(cutn, B, 3, cs, cs)
    if augs:
        got = rd(bwb, nan_ws.shape)
        for k, _, _, sy, sx in cr:
            r = Ay[k].t() @ dimg[k] @ Ax[k] / sd * scale
            m = Ay[k].abs().t() @ dimg[k].abs() @ Ax[k].abs() / sd * scale
            check(f"cutouts_rr_bwd d crops[{k}]", got[k, :, :, :sy, :sx], r, (2 * Tmax + 6) * U * m + 1e-30)
            assert bool(got[k, :, :, sy:, :].isnan().all() and got[k, :, :, :, sx:].isnan().all()), "wrote outside the crop"
    else:
        gref, gmag = th.zeros(B, 3, H, W, dtype=D64), th.zeros(B, 3, H, W, dtype=D64)
        for k, ox, oy, sy, sx in cr:
            gref[:, :, oy:oy + sy, ox:ox + sx] += Ay[k].t() @ dimg[k] @ Ax[k]
            gmag[:, :, oy:oy + sy, ox:ox + sx] += Ay[k].abs().t() @ dimg[k].abs() @ Ax[k].abs()
        check("cutouts_rr_bwd", rd(bg, x.shape), gref * 0.5 / sd * scale, (2 * Tmax * cutn + 6) * U * gmag * 0.5 / sd * scale + 1e-30)


# ------------------------------------------------------------------------------------------------ whole steps
def _fullsize_ctx(H, W, cutn, cutn_variants=(), use_augs=False):
    """the cfg2 architecture (256² UNet family, ViT-B/32) at H x W, seeded weights; its fp32 oracle on the same device"""
    from clip_guided_diffusion_b200 import gaussian_diffusion as pgd
    from clip_guided_diffusion_b200 import guidance as pg
    from clip_guided_diffusion_b200 import unet as pu
    from clip_guided_diffusion_b200 import vit as pv
    from clip_guided_diffusion_b200 import weights as pw
    from oracle import diffusion as od
    from oracle.clip_vit import VIT_CONFIGS, CLIPVisualOnly
    from oracle.unet import UNetModel, config_for
    ucfg, vcfg = pu.config_for(256, True), pv.VIT_CONFIGS["ViT-B/32"]
    usd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234)
    vsd = pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 1235)
    ounet = UNetModel(config_for(256, True)).eval()
    ounet.load_state_dict(usd)
    oclip = CLIPVisualOnly(VIT_CONFIGS["ViT-B/32"]).eval()
    oclip.load_state_dict(vsd)
    for p in list(ounet.parameters()) + list(oclip.parameters()):
        p.requires_grad_(False)
    tgt = th.randn(1, 512, generator=th.Generator().manual_seed(0))
    eng = pg.GuidedStepB200(ucfg, usd, vcfg, vsd, batch=1, height=H, width=W, num_cutouts=cutn, cutn_variants=cutn_variants, device="cuda",
                            cutout_resize="lanczos3", use_augs=use_augs)
    eng.set_targets(tgt, th.ones(1))
    return dict(ounet=ounet.cuda(), oclip=oclip.cuda(), odiff=od.create_gaussian_diffusion(1000, "linear", "25"),
                pdiff=pgd.create_gaussian_diffusion(1000, "linear", "25"), eng=eng, targets=tgt.cuda(), weights=th.ones(1).cuda(),
                kw=dict(clip_guidance_scale=1000.0, tv_scale=150.0, range_scale=50.0, sat_scale=0.0), use_magnitude=False, cutout_resize="lanczos3")


def _fullsize_step(ctx, cutn, use_augs, seed=3, mode="ddim", t_index=14):
    from oracle.guidance import OracleCondFn
    eng = ctx["eng"]
    H, W = eng.H, eng.W
    g = th.Generator().manual_seed(seed)
    x, y = th.randn(1, 3, H, W, generator=g), th.randint(0, 1000, (1,), generator=g)
    th.manual_seed(seed + 200)
    coords = og.MakeCutouts(224, cutn)._generate_coords(H, W, cutn)
    th.manual_seed(seed + 100)
    noise = th.randn(1, 3, H, W)
    pdiff, odiff = ctx["pdiff"], ctx["odiff"]
    th.manual_seed(4242)
    eng.stage_step(pdiff.scalar_table(t_index, t_index, 0.0), coords, pdiff.model_timestep(t_index), y)
    eng.img(eng.unet.x_in).copy_(x)
    eng.img(eng.noise).copy_(noise)
    eng.replay(mode, cutn)
    th.cuda.synchronize()
    e = dict(g=eng.img(eng.g).cpu().clone(), pred_xstart=eng.img(eng.x0).cpu().clone(), sample=eng.img(eng.sample).cpu().clone())
    aug = {}
    if use_augs:
        aug = dict(aug_params=eng.v(eng.aug_prm, (eng.cutn, 20))[:cutn].cpu().clone(),
                   aug_noise=eng.v(eng.aug_noise, (eng.cutn, 4, 1, 3, eng.aug_smax, eng.aug_smax))[:cutn].clone())
    cond = OracleCondFn(odiff, ctx["oclip"], ctx["targets"], ctx["weights"], cut_size=224, num_cutouts=cutn, cutout_resize="lanczos3", **ctx["kw"])
    cond.current_timestep = t_index
    grabbed = {}

    def cond_fn(xx, tt, out, y=None):
        grabbed["g"] = cond(xx, tt, out, y=y, coords=coords, **aug).detach().clone()
        return grabbed["g"]
    xo = x.cuda()
    o = odiff.ddim_sample_with_grad(ctx["ounet"], xo, th.full((1,), t_index, device="cuda"), clip_denoised=False, cond_fn=cond_fn,
                                    model_kwargs={"y": y.cuda()}, eta=0.0)
    o = dict(g=grabbed["g"].cpu(), pred_xstart=o["pred_xstart"].detach().cpu(), sample=o["sample"].detach().cpu())
    from tests.step_parity import compare
    return compare(o, e)


@pytest.mark.gpu
@pytest.mark.parametrize("hw,cutn,variants,augs", [((256, 320), 16, (), False), ((320, 256), 16, (), False), ((256, 256), 16, (4, 8), False),
                                                   ((256, 320), 16, (), True), ((256, 256), 8, (4,), True)],
                         ids=["256x320", "320x256", "progressive", "augs-256x320", "augs-progressive"])
def test_fullsize_step_vs_oracle(hw, cutn, variants, augs, monkeypatch):
    """teacher-forced cfg2-architecture step (graph replay) against the fp32 oracle at protocol-3 thresholds, every cutout count"""
    monkeypatch.setattr(og, "MakeCutouts", AugResizeMakeCutouts)
    ctx = _fullsize_ctx(*hw, cutn, variants, augs)
    for c in sorted({cutn, *variants}):
        res = _fullsize_step(ctx, c, augs)
        assert res["cos_g"] > 0.995 and res["rel_x0"] < 2e-2 and res["rel_sample"] < 2e-2, (c, res)


@pytest.mark.gpu
@pytest.mark.parametrize("augs", [False, True])
def test_graph_replay_equals_eager_for_every_count(augs):
    """one step per cutout count from the CUDA graph and launched op by op: bitwise equal without use_augs; with use_augs the gradient
    scatter uses fp32 atomics, whose order may differ, so equal to a few fp32 ulps"""
    from tests.step_parity import build_tiny
    ctx = build_tiny("cuda", image=64, hw=(64, 96), B=2, cutn=8, cutn_variants=(2, 4), cutout_resize="lanczos3", use_augs=augs, use_graph=True)
    eng, pdiff = ctx["eng"], ctx["pdiff"]
    for c in (2, 4, 8):
        outs = []
        for fused in (False, True):
            g = th.Generator().manual_seed(c)
            x, y = th.randn(2, 3, 64, 96, generator=g), th.randint(0, 10, (2,), generator=g)
            th.manual_seed(c + 1)
            coords = og.MakeCutouts(32, c)._generate_coords(64, 96, c)
            eng.stage_step(pdiff.scalar_table(10, 10, 0.0), coords, pdiff.model_timestep(10), y)
            eng.img(eng.unet.x_in).copy_(x)
            eng.img(eng.noise).zero_()
            for _ in range(2 if fused else 1):  # the first replay captures after an eager run; the second is a pure replay
                eng.replay("ddim", c) if fused else eng._run_all("ddim", None, c)
            th.cuda.synchronize()
            outs.append((eng.img(eng.g).cpu().clone(), eng.img(eng.sample).cpu().clone()))
        (g0, s0), (g1, s1) = outs
        if augs:
            assert th.allclose(g0, g1, rtol=1e-5, atol=1e-6 * float(g0.abs().max())) and th.allclose(s0, s1, rtol=1e-5, atol=1e-6), c
        else:
            assert th.equal(g0, g1) and th.equal(s0, s1), c


@pytest.mark.gpu
def test_free_running_chain_64x96():
    """25 steps at 64 x 96 with lanczos3 cutouts, each side feeding its own sample back: final-sample PSNR above 40 dB (use_magnitude keeps
    the seeded tiny model's gradient bounded, as in tests/test_step_cpu.py's chain)"""
    from tests.step_parity import run_tiny_chain
    res = run_tiny_chain(device="cuda", mode="ancestral", image=64, hw=(64, 96), B=1, cutn=4, cutout_resize="lanczos3", fused=True,
                         use_graph=True, use_magnitude=True)
    assert res["finite"] and res["steps"] == 25 and res["psnr_sample"] > 40.0, res
