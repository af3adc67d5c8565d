"""Test side of the CLIP-tower ensemble (several towers guiding one step): an fp32 oracle made of oracle/guidance.py pieces -- the
reference's CLIP block (cutouts, CLIP_NORMALIZE, encode_image, spherical_dist_loss) once per tower, the CLIP losses summed, tv / range /
sat / LPIPS once, the RMS clamp on the total gradient -- and a tiny two-tower engine (the tiny ViT at 32 px and a tiny ModifiedResNet
at 64 px with another output width) to run against it.  Shared by tests/test_ensemble_cpu.py (op-list interpreter) and
tests/test_gpu_ensemble.py."""
import torch as th

from clip_guided_diffusion_b200 import gaussian_diffusion as pgd
from clip_guided_diffusion_b200 import guidance as pg
from clip_guided_diffusion_b200 import rn as prn
from clip_guided_diffusion_b200 import vit as pv
from clip_guided_diffusion_b200 import weights as pw
from oracle import clip_rn as orn
from oracle import diffusion as od
from oracle import guidance as og
from oracle.clip_vit import CLIPVisualOnly, ViTConfig as OViTConfig
from oracle.unet import UNetModel, seeded_init_, tiny_config
from tests.plan_interp import Interp
from tests.step_parity import compare, prod_unet_cfg

RN_RES, RN_DIM = 64, 48  # the second tower: another input resolution and another embedding width than the ViT's (32, 64)


class EnsembleInterp(Interp):
    """the plan interpreter plus CUTOUTS_BWD flags 2 (add the cutout gradient into dx instead of storing it)"""

    def op_CUTOUTS_BWD(self, op):
        if not op.flags & 2:
            return super().op_CUTOUTS_BWD(op)
        B, H, W = op.i[:3]
        dst = self.V(op.p[2], (B, 3, H, W), (3 * H * W, H * W, W, 1))
        old = dst.clone()
        super().op_CUTOUTS_BWD(op)
        dst.add_(old)


def interp_runner(eng):
    return EnsembleInterp(eng.plan).run_range


def tiny_towers():
    """[(engine config, state_dict, oracle tower)]: the tiny ViT of tests/step_parity.py and a one-bottleneck-per-stage RN"""
    vcfg = pv.ViTConfig(32, 16, 128, 2, 64)
    ovit = seeded_init_(CLIPVisualOnly(OViTConfig(32, 16, 128, 2, 64)), seed=5).eval()
    rcfg = prn.RNConfig(layers=(1, 1, 1, 1), output_dim=RN_DIM, input_resolution=RN_RES, width=64)
    rsd = pw.seeded_rn_state_dict(rcfg, seed=6)
    orn_ = orn.CLIPVisualRN(orn.RNConfig(layers=(1, 1, 1, 1), output_dim=RN_DIM, input_resolution=RN_RES, width=64)).eval()
    orn_.visual.load_state_dict({k[len("visual."):]: v for k, v in rsd.items()}, strict=False)
    for m in (ovit, orn_):
        for prm in m.parameters():
            prm.requires_grad_(False)
    return [(vcfg, ovit.state_dict(), ovit), (rcfg, rsd, orn_)]


def build_ensemble(device, B=2, P=1, cutn=3, image=32, hw=None, use_magnitude=False, sat_scale=0.0, init_scale=0.0, cutn_variants=(),
                   run_cutn=None, use_graph=False, towers=None, respacing="25"):
    ocfg = tiny_config(image_size=image, model_channels=64, channel_mult=(1, 2), num_res_blocks=1, attention_resolutions=(image // 2,),
                       class_cond=True)
    ounet = seeded_init_(UNetModel(ocfg)).eval()
    for prm in ounet.parameters():
        prm.requires_grad_(False)
    towers = towers or tiny_towers()
    g = th.Generator().manual_seed(99)
    targets = [th.randn(P, cfg.output_dim, generator=g) for cfg, _, _ in towers]
    weights = th.rand(P, generator=g) + 0.5
    weights = weights / weights.sum()
    kw = dict(clip_guidance_scale=1000.0, tv_scale=150.0, range_scale=50.0, sat_scale=sat_scale)
    lp_sd = init = olp = None
    if init_scale:
        from oracle import lpips as ol
        lp_sd = ol.seeded_state_dict()
        olp = ol.LPIPSVgg(lp_sd)
        init = th.rand(1, 3, image, image, generator=th.Generator().manual_seed(7)) * 2 - 1
    H, W = hw or (image, image)
    eng = pg.GuidedStepB200(prod_unet_cfg(ocfg), ounet.state_dict(), [c for c, _, _ in towers], [sd for _, sd, _ in towers], batch=B,
                            height=H, width=W, num_cutouts=cutn, max_prompts=P, use_magnitude=use_magnitude, device=device,
                            use_graph=use_graph, cutn_variants=cutn_variants, lpips_sd=lp_sd, init_scale=init_scale, **kw)
    eng.set_targets(targets, weights)
    return dict(ounet=ounet, towers=towers, targets=targets, weights=weights, kw=kw, olp=olp, init=init, init_scale=init_scale,
                use_magnitude=use_magnitude, cutn=run_cutn or cutn, B=B, hw=(H, W), eng=eng,
                odiff=od.create_gaussian_diffusion(1000, "linear", respacing), pdiff=pgd.create_gaussian_diffusion(1000, "linear", respacing))


def ensemble_loss(x, pred_xstart, fac, per_tower_coords, towers, targets, weights, *, clip_guidance_scale, tv_scale, range_scale, sat_scale,
                  lpips_model=None, init_tensor=None, init_scale=0.0):
    """cond_fn's loss (cgd/cgd.py:177-226) with the CLIP block repeated per tower: -> (total loss, {"clip": [per tower], ...})"""
    n = x.shape[0]
    x_in = pred_xstart * fac + x * (1 - fac)
    clip_terms = []
    for (cfg, _, model), tgt, coords in zip(towers, targets, per_tower_coords):
        cutn = len(coords)
        mk = og.MakeCutouts(cfg.input_resolution, cutn)
        clip_in = og.clip_normalize(mk(x_in.add(1).div(2), coords=coords))
        embeds = model.encode_image(clip_in).float().view([cutn, n, -1])
        dists = og.spherical_dist_loss(embeds.unsqueeze(0), tgt.unsqueeze(0)).view([cutn, n, -1])
        clip_terms.append(dists.mul(weights).sum(2).mean(0).sum() * clip_guidance_scale)
    range_l = og.range_loss(pred_xstart).sum() * range_scale
    tv_l = og.tv_loss(x_in).sum() * tv_scale
    loss = sum(clip_terms) + tv_l + range_l
    if sat_scale != 0:
        loss = loss + th.abs(x_in - x_in.clamp(min=-1, max=1)).mean() * sat_scale
    if lpips_model is not None and init_tensor is not None and init_scale != 0:
        loss = loss + lpips_model(x_in, init_tensor).sum() * init_scale
    return loss, {"clip": [float(c.detach()) for c in clip_terms], "tv": float(tv_l.detach()), "range": float(range_l.detach())}


def oracle_step(ctx, mode, x, t_index, y, noise_seed, per_tower_coords, fac_index):
    odiff = ctx["odiff"]
    fac = float(odiff.sqrt_one_minus_alphas_cumprod[fac_index])
    grabbed = {}

    def cond_fn(xx, tt, out, y=None):
        loss, terms = ensemble_loss(xx, out["pred_xstart"], fac, per_tower_coords, ctx["towers"], ctx["targets"], ctx["weights"],
                                    lpips_model=ctx["olp"], init_tensor=ctx["init"], init_scale=ctx["init_scale"], **ctx["kw"])
        g = -th.autograd.grad(loss, xx)[0]
        if ctx["use_magnitude"]:
            g = og.magnitude_clamp(g)
        grabbed.update(g=g.detach().clone(), terms=terms)
        return g

    t = th.full((x.shape[0],), t_index, dtype=th.long)
    th.manual_seed(noise_seed)
    fn = odiff.p_sample_with_grad if mode == "ancestral" else odiff.ddim_sample_with_grad
    out = fn(ctx["ounet"], x, t, clip_denoised=False, cond_fn=cond_fn, model_kwargs={"y": y})
    out.update(grabbed)
    return out


def engine_step(ctx, mode, x, t_index, y, noise, per_tower_coords, fac_index, runner=None, fused=False):
    eng, pdiff = ctx["eng"], ctx["pdiff"]
    eng.stage_step(pdiff.scalar_table(t_index, fac_index, 0.0), per_tower_coords, pdiff.model_timestep(t_index), y)
    eng.img(eng.unet.x_in).copy_(x)
    eng.img(eng.noise).copy_(noise)
    cutn = len(per_tower_coords[0])
    if fused:
        eng.replay(mode, cutn)
    else:
        eng._run_all(mode, runner, cutn)
    if eng.device.type == "cuda":
        th.cuda.synchronize()
    return dict(sample=eng.img(eng.sample).float().cpu().clone(), pred_xstart=eng.img(eng.x0).float().cpu().clone(),
                g=eng.img(eng.g).float().cpu().clone(), losses={k: v.clone() for k, v in eng.losses().items()})


def make_inputs(ctx, seed=3):
    """x_t, classes, noise and every tower's windows, drawn in tower order with the tower's own cut size"""
    B, (H, W) = ctx["B"], ctx["hw"]
    g = th.Generator().manual_seed(seed)
    x = th.randn(B, 3, H, W, generator=g)
    y = th.randint(0, 10, (B,), generator=g)
    th.manual_seed(seed + 100)
    noise = th.randn_like(x)
    th.manual_seed(seed + 200)
    coords = [og.MakeCutouts(cfg.input_resolution, ctx["cutn"])._generate_coords(H, W, ctx["cutn"]) for cfg, _, _ in ctx["towers"]]
    return x, y, noise, seed + 100, coords


def run_ensemble_step(ctx, mode="ancestral", t_index=14, runner=None, fused=False):
    if ctx["init"] is not None:
        ctx["eng"].set_init_image(ctx["init"], runner)
    x, y, noise, nseed, coords = make_inputs(ctx)
    o = oracle_step(ctx, mode, x, t_index, y, nseed, coords, fac_index=t_index)
    e = engine_step(ctx, mode, x, t_index, y, noise, coords, fac_index=t_index, runner=runner, fused=fused)
    res = compare(o, e)
    per = e["losses"]["clip_per_tower"].sum(1)
    res["clip_loss_rel"] = max(abs(float(a) - b) / (abs(b) + 1e-9) for a, b in zip(per, o["terms"]["clip"]))
    res["clip_sum_rel"] = abs(float(e["losses"]["clip"].sum()) - sum(o["terms"]["clip"])) / (abs(sum(o["terms"]["clip"])) + 1e-9)
    res["tv_loss_rel"] = abs(float(e["losses"]["tv"].sum()) - o["terms"]["tv"]) / (abs(o["terms"]["tv"]) + 1e-9)
    res["range_loss_rel"] = abs(float(e["losses"]["range"].sum()) - o["terms"]["range"]) / (abs(o["terms"]["range"]) + 1e-9)
    return res
