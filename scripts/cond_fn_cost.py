#!/usr/bin/env python
"""What a guided step costs with the reference's cond_fn written in PyTorch, at cfg2's size (256x256, ViT-B/32, 16 cutouts, seeded
weights, batch 1, DDIM), on one GPU.  Three arms, timed alternating:

- fused: the package's own CondFnB200 step (one CUDA graph);
- package: a cond_fn written like the reference's (tests/cond_fn_autograd_interp.py, reference_style_cond_fn) on engine.model,
  load_clip's model, the package's MakeCutouts, clip_util.CLIP_NORMALIZE and losses, through ddim_sample_with_grad on an input_grad engine;
- eager_cutouts_losses: the same cond_fn with the oracle's eager MakeCutouts, normalisation and losses (everything else as `package`).

CUDA events around each step, warmed up, medians over the timed steps.  Prints one JSON line with the card's name and power limit.

    python scripts/cond_fn_cost.py [--steps 30] [--warmup 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import types

import torch as th

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from clip_guided_diffusion_b200 import clip_util  # noqa: E402
from clip_guided_diffusion_b200 import gaussian_diffusion as pgd  # noqa: E402
from clip_guided_diffusion_b200 import guidance as pg  # noqa: E402
from clip_guided_diffusion_b200 import losses as pl  # noqa: E402
from clip_guided_diffusion_b200 import unet as pu  # noqa: E402
from clip_guided_diffusion_b200 import vit as pv  # noqa: E402
from clip_guided_diffusion_b200 import weights as pw  # noqa: E402
from scripts.autograd_step_cost import card, timed_alternating  # noqa: E402
from tests.cond_fn_autograd_interp import reference_style_cond_fn  # noqa: E402


def main():
    from oracle import guidance as og
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not th.cuda.is_available():
        raise SystemExit("needs a GPU: the timings are CUDA events")
    ucfg, vcfg = pu.config_for(256, True), pv.VIT_CONFIGS["ViT-B/32"]
    usd, vsd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234), pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 1235)
    diff = pgd.create_gaussian_diffusion(1000, "linear", "ddim50")
    th.manual_seed(0)
    tgt = th.randn(1, 512)
    y = th.zeros(1, dtype=th.long, device="cuda")
    res = {"card": card(), "size": "cfg2: 256x256, ViT-B/32, 16 cutouts, batch 1, DDIM", "steps": args.steps, "warmup": args.warmup}

    eng = pg.GuidedStepB200(ucfg, usd, vcfg, vsd, batch=1, num_cutouts=16, device="cuda")
    eng.set_targets(tgt, th.ones(1))
    cond = pg.CondFnB200(eng, diff, pg.MakeCutouts(224, 16))
    x = eng.draw_initial_noise()
    geng = pg.GuidedStepB200(ucfg, usd, batch=1, device="cuda", input_grad=True)
    clip_model, clip_size = clip_util.load_clip("ViT-B/32", "cuda", clip_state_dict=vsd, max_images=16)
    t = th.full((1,), 30, dtype=th.long, device="cuda")

    def cond_fn(make_cutouts, normalize, losses):
        return reference_style_cond_fn(types.SimpleNamespace(
            diffusion=diff, current_timestep=30, make_cutouts=make_cutouts, clip_util=normalize, losses=losses, clip_model=clip_model,
            target_embeds=tgt.cuda(), weights=th.ones(1, device="cuda"), num_cutouts=16, clip_guidance_scale=1000, tv_scale=150,
            range_scale=50, sat_scale=0, use_magnitude=False))
    arms = {"package": cond_fn(pg.MakeCutouts(clip_size, 16), clip_util, pl),
            "eager_cutouts_losses": cond_fn(og.MakeCutouts(clip_size, 16), types.SimpleNamespace(CLIP_NORMALIZE=og.clip_normalize), og)}
    fns = {"fused": lambda: eng.fused_step(diff, "ddim", 30, x, y, cond)}
    for k, cf in arms.items():
        fns[k] = lambda cf=cf: diff.ddim_sample_with_grad(geng.model, x, t, clip_denoised=False, cond_fn=cf, model_kwargs={"y": y})
    res["step_ms"] = timed_alternating(fns, args.steps, args.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
