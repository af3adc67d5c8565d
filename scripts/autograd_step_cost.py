#!/usr/bin/env python
"""What a guided step costs when the guidance is a PyTorch cond_fn on the engine's autograd bridge, at cfg2's size (256x256, ViT-B/32,
16 cutouts, seeded weights, batch 1, DDIM), on one GPU:

- fused: the package's own CondFnB200 step (one CUDA graph);
- generic: the same guidance written in PyTorch -- the oracle's cond_fn with the CLIP tower in fp16 (LayerNorm in fp32, like the
  reference's clip.model.convert_weights) -- through the package's ddim_sample_with_grad on an input_grad engine: UNet forward +
  p_mean_variance on the engine, CLIP forward / backward in PyTorch, the UNet input gradient on the engine;
- unet_fwd_bwd: `model()` forward + `th.autograd.grad` alone, no guidance.

CUDA events around each step, warmed up, medians over the timed steps.  Prints one JSON line with the card's name and power limit.

    python scripts/autograd_step_cost.py [--steps 20] [--warmup 5]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch as th

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from clip_guided_diffusion_b200 import gaussian_diffusion as pgd  # noqa: E402
from clip_guided_diffusion_b200 import guidance as pg  # noqa: E402
from clip_guided_diffusion_b200 import unet as pu  # noqa: E402
from clip_guided_diffusion_b200 import vit as pv  # noqa: E402
from clip_guided_diffusion_b200 import weights as pw  # noqa: E402


def timed(fn, steps, warmup):
    """median ms of fn() between CUDA events, after `warmup` untimed calls"""
    for _ in range(warmup):
        fn()
    th.cuda.synchronize()
    ms = []
    for _ in range(steps):
        a, b = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else th.cuda.get_device_name(0)


def main():
    from oracle import guidance as og
    from oracle.clip_vit import VIT_CONFIGS, CLIPVisualOnly
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
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
    res["fused_step_ms"] = timed(lambda: eng.fused_step(diff, "ddim", 30, x, y, cond), args.steps, args.warmup)
    res["launches_per_step_fused"] = eng.launches_per_step("ddim")
    del eng, cond
    th.cuda.empty_cache()

    geng = pg.GuidedStepB200(ucfg, usd, batch=1, device="cuda", input_grad=True)
    clip = CLIPVisualOnly(VIT_CONFIGS["ViT-B/32"]).eval()
    clip.load_state_dict(vsd)
    clip = clip.cuda().half()
    for m in clip.modules():
        if isinstance(m, th.nn.LayerNorm):
            m.float()
    for prm in clip.parameters():
        prm.requires_grad_(False)
    ocond = og.OracleCondFn(diff, clip, tgt.cuda(), th.ones(1, device="cuda"), cut_size=224, num_cutouts=16)
    ocond.current_timestep = 30
    t = th.full((1,), 30, dtype=th.long, device="cuda")
    res["generic_step_ms"] = timed(lambda: diff.ddim_sample_with_grad(geng.model, x, t, clip_denoised=False, cond_fn=ocond,
                                                                       model_kwargs={"y": y}), args.steps, args.warmup)
    w = th.randn(1, 6, 256, 256, device="cuda")
    ts = th.full((1,), float(diff.model_timestep(30)), device="cuda")

    def unet_fwd_bwd():
        xe = x.detach().requires_grad_()
        return th.autograd.grad((w * geng.model(xe, ts, y)).sum(), xe)
    res["unet_fwd_bwd_ms"] = timed(unet_fwd_bwd, args.steps, args.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
