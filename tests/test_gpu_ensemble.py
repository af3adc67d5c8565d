"""GPU: several CLIP towers guiding one step.  CUTOUTS_BWD flags 2 (add into dx) bit for bit on both kernels, the tiny two-tower step
against the fp32 ensemble oracle (eager and replayed from the CUDA graph), one full-size 256x256 step with ViT-B/32 + ViT-B/16 + RN50
against the oracle with TF32 off, and the entry end to end with two towers and device-encoded text prompts."""
import os
import unittest.mock as mock

import pytest
import torch as th
import torch.nn.functional as F

from clip_guided_diffusion_b200 import _lib, cgd
from clip_guided_diffusion_b200 import gaussian_diffusion as pgd
from clip_guided_diffusion_b200 import guidance as pg
from clip_guided_diffusion_b200 import rn as prn
from clip_guided_diffusion_b200 import text as ptx
from clip_guided_diffusion_b200 import tokenizer as ptok
from clip_guided_diffusion_b200 import unet as pu
from clip_guided_diffusion_b200 import vit as pv
from clip_guided_diffusion_b200 import weights as pw
from tests import clip_text_oracle as oct
from tests.ensemble_oracle import build_ensemble, ensemble_loss, run_ensemble_step
from tests.step_parity import cos, rel

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------- CUTOUTS_BWD flags 2
def _cut_bwd(dp, coords, dx, B, H, W, cutn, cs, P, kpad, flags):
    _lib.run_op("CUTOUTS_BWD", flags=flags, i=[B, H, W, cutn, cs, P, kpad], f=[0.0, 0.0, 0.0, 0.26862954, 0.26130258, 0.27577711, 0.37],
                p=[dp, coords, dx])


@pytest.mark.parametrize("B,H,W,cutn,cs,P", [(2, 64, 64, 16, 32, 16),     # row-per-block kernel
                                             (1, 48, 80, 9, 32, 16),      # non-square image
                                             (2, 40, 56, 130, 32, 16),    # cutn > 128: the element-per-thread kernel
                                             (1, 96, 64, 24, 224, 32)])   # up-sampling windows (ViT-B/32 geometry)
def test_cutouts_bwd_accumulate_is_old_plus_store(B, H, W, cutn, cs, P):
    g = th.Generator().manual_seed(cutn)
    kpad = 3 * P * P
    dp = (th.randn(cutn * B, (cs // P) ** 2, kpad, generator=g) * 0.1).half().cuda()
    side = min(H, W)
    coords = []
    for _ in range(cutn):
        s = int(th.randint(min(side, cs) // 2, side + 1, (), generator=g))
        coords.append((int(th.randint(0, W - s + 1, (), generator=g)), int(th.randint(0, H - s + 1, (), generator=g)), s))
    cdev = th.tensor(coords, dtype=th.int32).cuda()
    old = th.randn(B, 3, H, W, generator=g).cuda()
    stored = th.full_like(old, float("nan"))
    _cut_bwd(dp, cdev, stored, B, H, W, cutn, cs, P, kpad, flags=0)
    acc = old.clone()
    _cut_bwd(dp, cdev, acc, B, H, W, cutn, cs, P, kpad, flags=2)
    th.cuda.synchronize()
    assert bool(th.isfinite(stored).all()) and float(stored.abs().max()) > 0
    assert th.equal(acc, old + stored)  # bitwise: one IEEE fp32 addition per element


# ---------------------------------------------------------------- the tiny two-tower step
@pytest.mark.parametrize("mode,kw", [("ancestral", dict(B=2, P=1)), ("ddim", dict(B=1, P=3, cutn=2)),
                                     ("ancestral", dict(B=2, sat_scale=30.0, use_magnitude=True)),
                                     ("ddim", dict(B=2, cutn=2, init_scale=1000.0)),
                                     ("ancestral", dict(B=1, cutn=8, cutn_variants=(2, 4), run_cutn=4))])
def test_two_tower_step_vs_oracle_eager_and_graph(mode, kw):
    ctx = build_ensemble("cuda", use_graph=True, **kw)
    for fused in (False, True):
        res = run_ensemble_step(ctx, mode, fused=fused)
        assert res["cos_g"] > 0.995 and res["rel_x0"] < 2e-2 and res["rel_sample"] < 2e-2, (fused, res)
        assert res["clip_loss_rel"] < 2e-2 and res["clip_sum_rel"] < 2e-2 and res["tv_loss_rel"] < 1e-3, (fused, res)
    eng = ctx["eng"]
    assert eng.launches_per_step(mode) > 0 and eng.losses()["clip_per_tower"].shape == (2, ctx["B"])


# ---------------------------------------------------------------- full size: ViT-B/32 + ViT-B/16 + RN50 at 256 x 256
def test_full_size_three_tower_step_vs_fp32_oracle():
    from oracle import clip_rn as orn
    from oracle import diffusion as od
    from oracle.clip_vit import VIT_CONFIGS, CLIPVisualOnly
    from oracle.unet import UNetModel, config_for
    dev = th.device("cuda:0")
    tf32 = (th.backends.cuda.matmul.allow_tf32, th.backends.cudnn.allow_tf32)
    th.backends.cuda.matmul.allow_tf32 = False
    th.backends.cudnn.allow_tf32 = False
    try:
        size, cutn, t_index = 256, 16, 180
        ucfg = pu.config_for(size, True)
        cfgs = [pv.VIT_CONFIGS["ViT-B/32"], pv.VIT_CONFIGS["ViT-B/16"], prn.RN_CONFIGS["RN50"]]
        usd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234)
        sds = [pw.seeded_state_dict(pw.vit_param_shapes(cfgs[0]), 1235), pw.seeded_state_dict(pw.vit_param_shapes(cfgs[1]), 1236),
               pw.seeded_rn_state_dict(cfgs[2], seed=1237)]
        g = th.Generator().manual_seed(17)
        tgts = [th.randn(1, c.output_dim, generator=g) for c in cfgs]
        x = th.randn(1, 3, size, size, generator=g)
        noise = th.randn(1, 3, size, size, generator=g)
        y = th.tensor([417])
        th.manual_seed(23)
        coords = [pg.MakeCutouts(c.input_resolution, cutn)._generate_coords(size, size, cutn) for c in cfgs]

        eng = pg.GuidedStepB200(ucfg, usd, cfgs, sds, batch=1, num_cutouts=cutn, device=dev)
        eng.set_targets(tgts, th.ones(1))
        pdiff = pgd.create_gaussian_diffusion(1000, "linear", "ddim250", rescale_timesteps=ucfg.rescale_timesteps)
        eng.stage_step(pdiff.scalar_table(t_index, t_index, 0.0), coords, pdiff.model_timestep(t_index), y)
        eng.img(eng.unet.x_in).copy_(x)
        eng.img(eng.noise).copy_(noise)
        eng.replay("ddim")
        th.cuda.synchronize()
        e = {k: eng.img(b).float().cpu().clone() for k, b in (("sample", eng.sample), ("pred_xstart", eng.x0), ("g", eng.g))}
        e_losses = eng.losses()
        del eng
        th.cuda.empty_cache()

        ounet = UNetModel(config_for(size, True)).eval()
        ounet.load_state_dict(usd)
        models = []
        for name, sd in zip(("ViT-B/32", "ViT-B/16"), sds[:2]):
            m = CLIPVisualOnly(VIT_CONFIGS[name]).eval()
            m.load_state_dict(sd)
            models.append(m)
        rc = cfgs[2]
        m = orn.CLIPVisualRN(orn.RNConfig(layers=tuple(rc.layers), output_dim=rc.output_dim, input_resolution=rc.input_resolution,
                                          width=rc.width)).eval()
        m.visual.load_state_dict({k[len("visual."):]: v for k, v in sds[2].items()}, strict=False)
        models.append(m)
        ounet = ounet.to(dev)
        models = [m.to(dev) for m in models]
        for p in list(ounet.parameters()) + [p for m in models for p in m.parameters()]:
            p.requires_grad_(False)
        odiff = od.create_gaussian_diffusion(1000, "linear", "ddim250", rescale_timesteps=ucfg.rescale_timesteps)
        fac = float(odiff.sqrt_one_minus_alphas_cumprod[t_index])
        towers = [(c, None, m) for c, m in zip(cfgs, models)]
        grabbed = {}

        def cond_fn(xx, tt, out, y=None):
            loss, terms = ensemble_loss(xx, out["pred_xstart"], fac, coords, towers, [t.to(dev) for t in tgts], th.ones(1, device=dev),
                                        clip_guidance_scale=1000.0, tv_scale=150.0, range_scale=50.0, sat_scale=0.0)
            grabbed.update(g=-th.autograd.grad(loss, xx)[0].detach(), terms=terms)
            return grabbed["g"]

        with mock.patch.object(th, "randn_like", lambda t, **k: noise.to(t.device)):
            o = odiff.ddim_sample_with_grad(ounet, x.to(dev), th.tensor([t_index], device=dev), clip_denoised=False, cond_fn=cond_fn,
                                            model_kwargs={"y": y.to(dev)})
        o = dict(sample=o["sample"].detach().float().cpu(), pred_xstart=o["pred_xstart"].detach().float().cpu(), g=grabbed["g"].float().cpu())
        res = dict(cos_g=cos(e["g"], o["g"]), rel_g=rel(e["g"], o["g"]), rel_x0=rel(e["pred_xstart"], o["pred_xstart"]),
                   rel_sample=rel(e["sample"], o["sample"]))
        for m, ref in enumerate(grabbed["terms"]["clip"]):
            res[f"loss_clip{m}"] = abs(float(e_losses["clip_per_tower"][m].sum()) - ref) / (abs(ref) + 1e-9)
        print("three towers", {k: round(v, 5) for k, v in res.items()})
        assert all(th.isfinite(v).all() for v in e.values()), res
        assert res["cos_g"] > 0.995 and res["rel_x0"] < 2e-2 and res["rel_sample"] < 2e-2, res
        assert max(v for k, v in res.items() if k.startswith("loss_")) < 2e-2, res
    finally:
        th.backends.cuda.matmul.allow_tf32, th.backends.cudnn.allow_tf32 = tf32


# ---------------------------------------------------------------- the entry, two towers, device text encoder
def test_clip_guided_diffusion_with_two_towers_and_device_text(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    vpath = str(tmp_path / ptok.VOCAB_FILE)
    V = oct.write_vocab(vpath, oct.synthetic_merges(400))
    ucfg = pu.config_for(64, True)
    usd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234)
    vcfg, rcfg = pv.VIT_CONFIGS["ViT-B/32"], prn.RN_CONFIGS["RN50"]
    csds = [{**pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 1235),
             **pw.seeded_state_dict(pw.text_param_shapes(ptx.TextConfig(width=512, layers=12, vocab_size=V, output_dim=512)), 1236)},
            {**pw.seeded_rn_state_dict(rcfg, seed=1237),
             **pw.seeded_state_dict(pw.text_param_shapes(ptx.TextConfig(width=512, layers=12, vocab_size=V, output_dim=1024)), 1238)}]
    seen = []

    class Engine(pg.GuidedStepB200):
        def set_targets(self, target_embeds, weights):
            seen.append(([t.detach().float().cpu().clone() for t in target_embeds], th.as_tensor(weights).clone()))
            super().set_targets(target_embeds, weights)

    monkeypatch.setattr(cgd, "GuidedStepB200", Engine)
    monkeypatch.setattr(cgd, "_encode_text", lambda *a, **k: pytest.fail("text_encoder='device' must not use the clip package"))
    prompts = ["a lighthouse on a rocky coast:2", "oil painting of a fox"]
    got = list(cgd.clip_guided_diffusion(image_size=64, num_cutouts=4, prompts=prompts, batch_size=1, timestep_respacing="25",
                                         skip_timesteps=22, save_frequency=2, prefix_path=tmp_path / "out", progress=False, seed=0,
                                         clip_model_name=["ViT-B/32", "RN50"], unet_state_dict=usd, clip_state_dict=csds,
                                         text_encoder="device", bpe_path=vpath))
    assert [b for b, _ in got] == [0, 0] and all(os.path.exists(p) for _, p in got)
    (targets, weights), = seen
    ids = ptok.tokenize(["a lighthouse on a rocky coast", "oil painting of a fox"], bpe_path=vpath)
    for t, csd, D in zip(targets, csds, (512, 1024)):
        ref = oct.encode_text(csd, ids)
        assert t.shape == (2, D) and float(F.cosine_similarity(t.double(), ref.double(), dim=-1).min()) > 0.999
    assert th.allclose(weights.float(), th.tensor([2.0, 1.0]) / 3.0, atol=1e-7)
