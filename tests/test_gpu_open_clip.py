"""GPU: the OpenCLIP towers (``"open_clip:<arch>"``) on the device kernels.

- every row of tests/open_clip_plan_table.py as one launch on the existing float64 harnesses; CONV flags 8 (acc * GELU'(u)) in the
  randn regime against a float64 GELU'; the padded ViT-H attention's padded columns of out, dq, dk and dv exactly zero;
- QGELU_FWD flags 1 (exact GELU) against float64 at every size the plans run;
- the five towers at 16 images (ViT-B-32 also at 1 and 2), forward and input gradient through load_clip's autograd bridge, against the
  fp32 oracle;
- teacher-forced cfg2-size guided steps with open_clip:ViT-H-14 (DDIM and ancestral, eager and graph replay) and with the ensemble
  ViT-B/32 + open_clip:ViT-H-14, against the fp32 oracle;
- clip_guided_diffusion(clip_model_name="open_clip:ViT-B-32", text_encoder="device") end to end."""
from __future__ import annotations

import math
import unittest.mock as mock

import pytest
import torch as th

from clip_guided_diffusion_b200 import clip_model as cm
from clip_guided_diffusion_b200 import gaussian_diffusion as pgd
from clip_guided_diffusion_b200 import guidance as pg
from clip_guided_diffusion_b200 import unet as pu
from clip_guided_diffusion_b200 import vit as pv
from clip_guided_diffusion_b200 import weights as pw
from clip_guided_diffusion_b200.plan import Plan
from tests import test_gpu_conv_kernels as KC
from tests import test_gpu_kernels_fullshape as KF
from tests.kernel_check import D64, U, check, check16, run, ulp16
from tests.open_clip_oracle import gelu_f64, gelu_grad_f64, vision_oracle
from tests.open_clip_plan_table import OPEN_CLIP_CONV_PLAN, OPEN_CLIP_GELU_SIZES, OPEN_CLIP_OP_PLAN, OPEN_CLIP_OTHER_PLAN
from tests.step_parity import cos, rel

pytestmark = pytest.mark.gpu
ARCHS = list(pv.OPEN_CLIP_CONFIGS)


def no_tf32():
    saved = (th.backends.cuda.matmul.allow_tf32, th.backends.cudnn.allow_tf32)
    th.backends.cuda.matmul.allow_tf32 = th.backends.cudnn.allow_tf32 = False
    return saved


# ---------------------------------------------------------------------------------------------------------------- one launch per table row
def gelu_grad_tol(u):
    """absolute error of the device's GELU'(u) = Phi(u) + u phi(u), Phi = erfcf(-u / sqrt 2) / 2 and phi through the __expf intrinsic (ex2.approx
    of a pre-scaled argument): a few ulp each, their fp32 arguments off by 2 U |arg|, and the four roundings of the products and the fma"""
    u = u.double()
    cdf, pdf = 0.5 * (1 + th.erf(u / math.sqrt(2))), th.exp(-0.5 * u * u) / math.sqrt(2 * math.pi)
    return 8 * U * (cdf + u.abs() * pdf * (2 + u * u)) + 4 * U * gelu_grad_f64(u).abs()


@pytest.mark.parametrize("case", OPEN_CLIP_CONV_PLAN, ids=[KC.conv_id(s) for s in OPEN_CLIP_CONV_PLAN])
def test_conv_rows(case):
    if not case[10] & 8:
        KC.test_conv_exact("cuda", case)
        KC.test_conv_randn("cuda", case)
        return
    x, w, bias, res, _ = KC.conv_data(th.device("cuda"), case, "randn")
    _, mag, acc = KC.reference(case, x, w, None, None)
    u = res.to(D64)
    ref = acc * gelu_grad_f64(u)
    tol = KC.C_ACC * U * mag * gelu_grad_f64(u).abs() + acc.abs() * gelu_grad_tol(u)
    got, what = KC.launch("cuda", case, x, w, bias, res)
    check(what, got, ref, tol + ulp16(ref))


@pytest.mark.parametrize("n", [1, 2])
def test_conv_rows_of_small_b32_batches(n):
    """open_clip:ViT-B-32 at 1 and 2 images: the c_proj dgrad spans one pixel tile, the planner forces BN >= 64 and no split-K for the
    GELU' epilogue; every CONV flags 8 signature of that plan, one launch each"""
    from tests.test_conv_coverage_cpu import plan_conv_signatures
    cfg = pv.OPEN_CLIP_CONFIGS["ViT-B-32"].vision
    plan = pv.ViTB200(cfg, pw.seeded_state_dict(pw.vit_param_shapes(cfg), 1235), n_images=n, device="cpu").plan
    rows = [s for s in plan_conv_signatures(plan) if s[10] & 8]
    assert rows
    for case in rows:
        test_conv_rows(case)


@pytest.mark.parametrize("sig", OPEN_CLIP_OTHER_PLAN, ids=[repr(s) for s in OPEN_CLIP_OTHER_PLAN])
def test_other_rows(sig, monkeypatch):
    from tests.test_gpu_clip_autograd import test_tower_other_launches
    test_tower_other_launches(sig, monkeypatch)


def _op_row(s):
    code, r = s[0], s[1:]
    if code == "LN_FWD":
        return KF.test_layernorm("cuda", (*r, r[1], r[1]))
    if code == "LN_BWD":
        return KF.test_layernorm("cuda", (r[0], r[1], r[3], r[1], r[2], r[4]))
    if code == "LINEAR_SMALL":
        return KF.test_linear_small("cuda", (r[:7],))
    if code == "VIT_EMBED":
        return KF.test_vit_embed("cuda", (r[0], tuple(r[1:])))
    if code == "QGELU_FWD":
        return KF.test_qgelu("cuda", r[0])
    if code in ("CUTOUTS_FWD", "CUTOUTS_BWD"):
        return KF.test_cutouts_fwd_bwd("cuda", (*r[:4], tuple(r[4:7]), ()))
    if code == "SPHERICAL":
        return KF.test_spherical("cuda", (*r, "random"))
    pytest.fail(f"no GPU harness for {code}")


@pytest.mark.parametrize("sig", OPEN_CLIP_OP_PLAN, ids=[repr(s) for s in OPEN_CLIP_OP_PLAN])
def test_op_rows(sig):
    _op_row(sig)


@pytest.mark.parametrize("n", OPEN_CLIP_GELU_SIZES)
def test_exact_gelu_fwd(n):
    """QGELU_FWD flags 1: 0.5 u (1 + erf(u / sqrt 2)) from fp16 u over [-70, 70], one fp16 rounding (test_qgelu's tolerance form)"""
    g = th.Generator().manual_seed(1)
    u = th.rand(n, generator=g) * 140 - 70
    u[:12] = th.tensor([0.0, -0.0, 60.0, -60.0, 1e-4, -1e-4, 3.0, -3.0, 6.0, -6.0, 30.0, -30.0])
    u[12:n // 2] = th.randn(n // 2 - 12, generator=g) * 3
    u = u.half()
    plan = Plan()
    bu, ba = plan.new(n, "h"), plan.new(n, "h")
    plan.emit("QGELU_FWD", flags=1, i=[n], p=[(bu, 0), (ba, 0)])
    rd = run(plan, "cuda", [(bu, u)])
    a = gelu_f64(u)
    check16(f"gelu_fwd n={n}", rd(ba), a, 2.0 ** -24 + 16 * U * a.abs())


@pytest.mark.parametrize("B", sorted({s[1] for s in OPEN_CLIP_OTHER_PLAN if s[0] == "ATTN_FWD" and s[4] == 128}))
def test_padded_attention_columns_stay_zero(B):
    """ViT-H's heads: 80 live columns of 128 in q, k, v and d out; out, dq, dk and dv are exactly zero in the other 48"""
    heads, T, d, live, C = 16, 257, 128, 80, 2048
    g = th.Generator(device="cuda").manual_seed(B)
    qkv = th.randn(B * T, 3, heads, d, device="cuda", generator=g)
    qkv[..., live:] = 0
    do = th.randn(B * T, heads, d, device="cuda", generator=g)
    do[..., live:] = 0
    plan = Plan()
    bqkv, bo, blse, bdo, bd, bdel = (plan.new(B * T * 3 * C, "h"), plan.new(B * T * C, "h"), plan.new(B * heads * T, "f"), plan.new(B * T * C, "h"),
                                     plan.new(B * T * 3 * C, "h"), plan.new(B * heads * T, "f"))
    ii = [B, heads, T, d, T * 3 * C, 3 * C, d, T * C, C, d]
    sc = [1.0 / math.sqrt(live)]
    q, k, v = (bqkv, 0), (bqkv, C), (bqkv, 2 * C)
    plan.emit("ATTN_FWD", i=ii, f=sc, p=[q, k, v, (bo, 0), (blse, 0)])
    plan.emit("ATTN_BWD", i=ii, f=sc, p=[q, k, v, (bo, 0), (bdo, 0), (blse, 0), (bd, 0), (bd, C), (bd, 2 * C), (bdel, 0)])
    rd = run(plan, "cuda", [(bqkv, qkv.half()), (bdo, do.half()), (bd, th.full((B * T * 3 * C,), float("nan")))])
    out, dqkv = rd(bo, (B * T, heads, d)), rd(bd, (B * T, 3, heads, d))
    assert th.isfinite(out).all() and th.isfinite(dqkv).all()
    assert not out[..., live:].any() and not dqkv[..., live:].any()
    # the live columns are the unpadded 80-wide attention's
    q64, k64, v64 = (qkv[:, j, :, :live].double().view(B, T, heads, live).transpose(1, 2) for j in range(3))
    ref = th.softmax(q64 @ k64.transpose(-1, -2) * sc[0], -1) @ v64
    assert rel(out[..., :live].view(B, T, heads, live).transpose(1, 2).cuda(), ref) < 2e-3


# ---------------------------------------------------------------------------------------------------------------- towers through load_clip
@pytest.mark.parametrize("arch,n", [(a, 16) for a in ARCHS] + [("ViT-B-32", 1), ("ViT-B-32", 2)])
def test_tower_forward_and_input_gradient_vs_fp32_oracle(arch, n):
    cfg = pv.OPEN_CLIP_CONFIGS[arch].vision
    sd = pw.seeded_state_dict(pw.vit_param_shapes(cfg), 1235)
    saved = no_tf32()
    try:
        model, res = cm.load_clip(f"open_clip:{arch}", "cuda", max_images=n, clip_state_dict=sd)
        assert res == 224 and model.cfg.act == cfg.act
        g = th.Generator(device="cuda").manual_seed(5)
        img = th.randn(n, 3, 224, 224, device="cuda", generator=g).requires_grad_()
        seed = th.randn(n, cfg.output_dim, device="cuda", generator=g)
        emb = model.encode_image(img)
        (gi,) = th.autograd.grad((emb * seed).sum(), img)
        del model
        oracle = vision_oracle(cfg, sd).cuda()
        for p in oracle.parameters():
            p.requires_grad_(False)
        x = img.detach().clone().requires_grad_()
        ref = oracle.encode_image(x)
        (gr,) = th.autograd.grad((ref * seed).sum(), x)
        r = dict(cos_e=cos(emb, ref), rel_e=rel(emb, ref), cos_g=cos(gi, gr), rel_g=rel(gi, gr))
        print(arch, r)
        assert r["cos_e"] > 0.999 and r["rel_e"] < 2e-2 and r["cos_g"] > 0.999 and r["rel_g"] < 4e-2, (arch, r)
    finally:
        th.backends.cuda.matmul.allow_tf32, th.backends.cudnn.allow_tf32 = saved


# ---------------------------------------------------------------------------------------------------------------- full-size guided steps
def _full_step(names, mode, t_index=180, size=256, cutn=16):
    from oracle import diffusion as od
    from oracle.clip_vit import VIT_CONFIGS, CLIPVisualOnly
    from oracle.unet import UNetModel, config_for
    from tests.ensemble_oracle import ensemble_loss
    dev = th.device("cuda:0")
    ucfg = pu.config_for(size, True)
    cfgs = [pv.OPEN_CLIP_CONFIGS[n[len("open_clip:"):]].vision if n.startswith("open_clip:") else pv.VIT_CONFIGS[n] for n in names]
    usd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234)
    sds = [pw.seeded_state_dict(pw.vit_param_shapes(c), 1235 + k) for k, c in enumerate(cfgs)]
    g = th.Generator().manual_seed(17)
    tgts = [th.randn(1, c.output_dim, generator=g) for c in cfgs]
    x = th.randn(1, 3, size, size, generator=g)
    noise = th.randn(1, 3, size, size, generator=g)
    y = th.tensor([417])
    th.manual_seed(23)
    coords = [pg.MakeCutouts(c.input_resolution, cutn)._generate_coords(size, size, cutn) for c in cfgs]
    respacing = "ddim250" if mode == "ddim" else "250"
    one = len(cfgs) == 1
    eng = pg.GuidedStepB200(ucfg, usd, cfgs[0] if one else cfgs, sds[0] if one else sds, batch=1, num_cutouts=cutn, device=dev)
    eng.set_targets(tgts[0] if one else tgts, th.ones(1))
    pdiff = pgd.create_gaussian_diffusion(1000, "linear", respacing, rescale_timesteps=ucfg.rescale_timesteps)
    outs = {}
    for how in ("eager", "graph"):
        eng.stage_step(pdiff.scalar_table(t_index, t_index, 0.0), coords if not one else coords[0], pdiff.model_timestep(t_index), y)
        eng.img(eng.unet.x_in).copy_(x)
        eng.img(eng.noise).copy_(noise)
        if how == "eager":
            eng._launch(eng.schedule(mode, None, True))
        else:
            eng.replay(mode)
        th.cuda.synchronize()
        outs[how] = {k: eng.img(b).float().cpu().clone() for k, b in (("sample", eng.sample), ("pred_xstart", eng.x0), ("g", eng.g))}
    del eng
    th.cuda.empty_cache()
    ounet = UNetModel(config_for(size, True)).eval()
    ounet.load_state_dict(usd)
    models = [vision_oracle(c, sd) if n.startswith("open_clip:") else CLIPVisualOnly(VIT_CONFIGS[n]).eval() for n, c, sd in zip(names, cfgs, sds)]
    for n, m, sd in zip(names, models, sds):
        if not n.startswith("open_clip:"):
            m.load_state_dict(sd)
    ounet = ounet.to(dev)
    models = [m.to(dev) for m in models]
    for p in list(ounet.parameters()) + [p for m in models for p in m.parameters()]:
        p.requires_grad_(False)
    odiff = od.create_gaussian_diffusion(1000, "linear", respacing, rescale_timesteps=ucfg.rescale_timesteps)
    fac = float(odiff.sqrt_one_minus_alphas_cumprod[t_index])
    towers = [(c, None, m) for c, m in zip(cfgs, models)]
    grabbed = {}

    def cond_fn(xx, tt, out, y=None):
        loss, _ = ensemble_loss(xx, out["pred_xstart"], fac, coords, towers, [t.to(dev) for t in tgts], th.ones(1, device=dev),
                                clip_guidance_scale=1000.0, tv_scale=150.0, range_scale=50.0, sat_scale=0.0)
        grabbed["g"] = -th.autograd.grad(loss, xx)[0].detach()
        return grabbed["g"]

    step = odiff.ddim_sample_with_grad if mode == "ddim" else odiff.p_sample_with_grad
    with mock.patch.object(th, "randn_like", lambda t, **k: noise.to(t.device)):
        o = step(ounet, x.to(dev), th.tensor([t_index], device=dev), clip_denoised=False, cond_fn=cond_fn, model_kwargs={"y": y.to(dev)})
    o = dict(sample=o["sample"].detach().float().cpu(), pred_xstart=o["pred_xstart"].detach().float().cpu(), g=grabbed["g"].float().cpu())
    for how, e in outs.items():
        res = dict(cos_g=cos(e["g"], o["g"]), rel_x0=rel(e["pred_xstart"], o["pred_xstart"]), rel_sample=rel(e["sample"], o["sample"]))
        print(names, mode, how, {k: round(v, 5) for k, v in res.items()})
        assert all(th.isfinite(v).all() for v in e.values()), (how, res)
        assert res["cos_g"] > 0.995 and res["rel_x0"] < 2e-2 and res["rel_sample"] < 2e-2, (how, res)


@pytest.mark.parametrize("mode", ["ddim", "ancestral"])
def test_vit_h_cfg2_step_vs_fp32_oracle(mode):
    saved = no_tf32()
    try:
        _full_step(["open_clip:ViT-H-14"], mode)
    finally:
        th.backends.cuda.matmul.allow_tf32, th.backends.cudnn.allow_tf32 = saved


def test_b32_plus_vit_h_ensemble_step_vs_fp32_oracle():
    saved = no_tf32()
    try:
        _full_step(["ViT-B/32", "open_clip:ViT-H-14"], "ddim")
    finally:
        th.backends.cuda.matmul.allow_tf32, th.backends.cudnn.allow_tf32 = saved


# ---------------------------------------------------------------------------------------------------------------- the entry point
def test_clip_guided_diffusion_open_clip_b32_device_text(tmp_path, monkeypatch):
    """a short DDIM run at 64² with open_clip:ViT-B-32 and a text prompt encoded on the device text tower (synthetic vocabulary)"""
    from clip_guided_diffusion_b200 import cgd
    from tests import clip_text_oracle as oct
    v, t = pv.OPEN_CLIP_CONFIGS["ViT-B-32"]
    oct.write_vocab(tmp_path / "bpe.txt.gz", oct.synthetic_merges(200))  # ids below 49408: the checkpoint's table rows
    sd = {**pw.seeded_state_dict(pw.vit_param_shapes(v), 1235), **pw.seeded_state_dict(pw.text_param_shapes(t), 1236)}
    encoded = []
    real = cgd._encode_text_device
    monkeypatch.setattr(cgd, "_encode_text_device", lambda *a, **k: encoded.append(k.get("act")) or real(*a, **k))
    monkeypatch.chdir(tmp_path)
    ucfg = pu.config_for(64, True)
    out = list(cgd.clip_guided_diffusion(image_size=64, num_cutouts=4, prompts=["a lighthouse"], clip_model_name="open_clip:ViT-B-32",
                                         clip_state_dict=sd, unet_state_dict=pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234),
                                         text_encoder="device", bpe_path=str(tmp_path / "bpe.txt.gz"), timestep_respacing="ddim4",
                                         diffusion_steps=1000, save_frequency=1, prefix_path=tmp_path / "out", progress=False))
    assert encoded == ["gelu"] and len(out) >= 4 and all(p.endswith(".png") for _, p in out)
