"""GPU: every BASELINE.json configuration at FULL architecture size, teacher-forced single guided step vs the fp32 oracle.

The oracle (oracle/: fp32 PyTorch restatement, eager autograd) runs on the same GPU with TF32 switched off -- cuDNN / cuBLAS fp32
FMA paths, i.e. the arithmetic of its CPU run, in seconds instead of minutes -- and receives the same weights (one seeded
state_dict in upstream key layout), x_t, timestep, class label, noise and cutout windows as the engine's CUDA-graph replay:

    cfg2  256x256, ddim250,            1 image, 16 cutouts, ViT-B/32      (the benchmarked configuration)
    cfg3  256x256, "1000" (ancestral), 1 image, 32 cutouts, ViT-B/32      (per-GPU shard of batch 8)
    cfg4  512x512, ddim250,            1 image, 16 cutouts, ViT-B/16      (per-GPU shard of batch 4)
    cfg5  512x512, "1000" (ancestral), 1 image, 64 cutouts, ViT-L/14, init image + LPIPS init_scale 1000 (shard of batch 8)
    default128  128x128, "1000" (ancestral), 1 image, 16 cutouts, ViT-B/32: the reference's default arguments (cgd/cgd.py:20-33)
    vit_l14_336  256x256, ddim250, 1 image, 4 cutouts of 336 px, ViT-L/14@336px

Tolerances (SURVEY.md 8c protocol item 2, the same as tests/test_gpu_ops.py): cos(g) > 0.995, rel L2 of pred_xstart and of the
sample < 2e-2 (fp16 storage with fp32 accumulation against fp32 everywhere), the loss terms within 2 %."""
import pytest
import torch as th

from clip_guided_diffusion_b200 import gaussian_diffusion as pgd
from clip_guided_diffusion_b200 import guidance as pg
from clip_guided_diffusion_b200 import unet as pu
from clip_guided_diffusion_b200 import vit as pv
from clip_guided_diffusion_b200 import weights as pw
from tests.step_parity import cos, rel

pytestmark = pytest.mark.gpu

CASES = {
    "cfg2": dict(size=256, respacing="ddim250", cutn=16, clip="ViT-B/32", lpips=False, t_index=180),
    "cfg3": dict(size=256, respacing="1000", cutn=32, clip="ViT-B/32", lpips=False, t_index=700),
    "cfg4": dict(size=512, respacing="ddim250", cutn=16, clip="ViT-B/16", lpips=False, t_index=120),
    "cfg5": dict(size=512, respacing="1000", cutn=64, clip="ViT-L/14", lpips=True, t_index=400),
    # not a BASELINE configuration: the reference's DEFAULT call (cgd/cgd.py:20-33: image_size 128, "1000", 16 cutouts, ViT-B/32) -- the
    # 128x128 checkpoint, whose four heads attend with 128 / 192 / 256 channels each (csrc/attention_flash.cu)
    "default128": dict(size=128, respacing="1000", cutn=16, clip="ViT-B/32", lpips=False, t_index=500),
    # the one CLIP_MODEL_URLS entry (cgd/clip_util.py:28) whose cutouts are not 224 px: 336 px, 24 x 24 patches of 14, 577 tokens
    "vit_l14_336": dict(size=256, respacing="ddim250", cutn=4, clip="ViT-L/14@336px", lpips=False, t_index=180),
}


def _oracle_on_gpu(c, usd, vsd, lsd, init, tgt, dev):
    from oracle import diffusion as od
    from oracle import guidance as og
    from oracle import lpips as ol
    from oracle.clip_vit import VIT_CONFIGS, CLIPVisualOnly
    from oracle.unet import UNetModel, config_for
    ounet = UNetModel(config_for(c["size"], True)).eval()
    ounet.load_state_dict(usd)
    oclip = CLIPVisualOnly(VIT_CONFIGS[c["clip"]]).eval()
    oclip.load_state_dict(vsd)
    ounet, oclip = ounet.to(dev), oclip.to(dev)
    for p in list(ounet.parameters()) + list(oclip.parameters()):
        p.requires_grad_(False)
    ucfg = pu.config_for(c["size"], True)
    odiff = od.create_gaussian_diffusion(1000, "linear", c["respacing"], rescale_timesteps=ucfg.rescale_timesteps)
    olp = ol.LPIPSVgg({k: v.to(dev) for k, v in lsd.items()}).to(dev) if lsd is not None else None
    cond = og.OracleCondFn(odiff, oclip, tgt.to(dev), th.ones(1, device=dev), cut_size=VIT_CONFIGS[c["clip"]].input_resolution,
                           num_cutouts=c["cutn"], lpips_model=olp,
                           init_tensor=init.to(dev) if init is not None else None, init_scale=1000.0 if lsd is not None else 0.0)
    return ounet, odiff, cond


@pytest.mark.parametrize("name", list(CASES))
def test_full_size_step_vs_fp32_oracle(name):
    c = CASES[name]
    dev = th.device("cuda:0")
    tf32 = (th.backends.cuda.matmul.allow_tf32, th.backends.cudnn.allow_tf32)
    th.backends.cuda.matmul.allow_tf32 = False
    th.backends.cudnn.allow_tf32 = False
    try:
        size, mode = c["size"], ("ddim" if c["respacing"].startswith("ddim") else "ancestral")
        ucfg, vcfg = pu.config_for(size, True), pv.VIT_CONFIGS[c["clip"]]
        usd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234)
        vsd = pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 1235)
        lsd = pw.seeded_lpips_state_dict() if c["lpips"] else None
        g = th.Generator().manual_seed(17)
        tgt = th.randn(1, vcfg.output_dim, generator=g)
        init = (th.rand(1, 3, size, size, generator=g) * 2 - 1) if c["lpips"] else None
        x = th.randn(1, 3, size, size, generator=g)
        noise = th.randn(1, 3, size, size, generator=g)
        y = th.tensor([417])
        th.manual_seed(23)
        coords = pg.MakeCutouts(vcfg.input_resolution, c["cutn"])._generate_coords(size, size, c["cutn"])
        t_index = c["t_index"]

        # ---- engine: one CUDA-graph replay of the fused step
        extra = dict(lpips_sd=lsd, init_scale=1000.0) if c["lpips"] else {}
        eng = pg.GuidedStepB200(ucfg, usd, vcfg, vsd, batch=1, num_cutouts=c["cutn"], device=dev, **extra)
        eng.set_targets(tgt, th.ones(1))
        if c["lpips"]:
            eng.set_init_image(init.to(dev))
        pdiff = pgd.create_gaussian_diffusion(1000, "linear", c["respacing"], rescale_timesteps=ucfg.rescale_timesteps)
        eng.stage_step(pdiff.scalar_table(t_index, t_index, 0.0), coords, pdiff.model_timestep(t_index), y)
        eng.img(eng.unet.x_in).copy_(x)
        eng.img(eng.noise).copy_(noise)
        eng.replay(mode)
        th.cuda.synchronize()
        e = {k: eng.img(b).float().cpu().clone() for k, b in (("sample", eng.sample), ("pred_xstart", eng.x0), ("g", eng.g))}
        e_losses = {k: float(v.sum()) for k, v in eng.losses().items()}
        del eng
        th.cuda.empty_cache()

        # ---- oracle: fp32, eager autograd, same device, TF32 off
        ounet, odiff, cond = _oracle_on_gpu(c, usd, vsd, lsd, init, tgt, dev)
        cond.current_timestep = t_index
        grabbed = {}

        def cond_fn(xx, tt, out, y=None):
            grabbed["g"] = cond(xx, tt, out, y=y, coords=coords).detach()
            return grabbed["g"]

        fn = odiff.ddim_sample_with_grad if mode == "ddim" else odiff.p_sample_with_grad
        import unittest.mock as mock
        with mock.patch.object(th, "randn_like", lambda t, **k: noise.to(t.device)):
            o = fn(ounet, x.to(dev), th.tensor([t_index], device=dev), clip_denoised=False, cond_fn=cond_fn, model_kwargs={"y": y.to(dev)})
        o = dict(sample=o["sample"].detach().float().cpu(), pred_xstart=o["pred_xstart"].detach().float().cpu(), g=grabbed["g"].float().cpu())
        res = dict(cos_g=cos(e["g"], o["g"]), rel_g=rel(e["g"], o["g"]), rel_x0=rel(e["pred_xstart"], o["pred_xstart"]),
                   rel_sample=rel(e["sample"], o["sample"]))
        for k in ("clip", "tv", "range") + (("init",) if c["lpips"] else ()):
            res["loss_" + k] = abs(e_losses[k] - cond.last_terms[k]) / (abs(cond.last_terms[k]) + 1e-9)
        print(name, {k: round(v, 5) for k, v in res.items()})
        assert all(th.isfinite(v).all() for v in e.values()), res
        assert res["cos_g"] > 0.995 and res["rel_x0"] < 2e-2 and res["rel_sample"] < 2e-2, res
        assert max(v for k, v in res.items() if k.startswith("loss_")) < 2e-2, res
    finally:
        th.backends.cuda.matmul.allow_tf32, th.backends.cudnn.allow_tf32 = tf32
