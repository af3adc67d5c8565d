#!/usr/bin/env python
"""What a guided step costs when the guidance is a PyTorch cond_fn on the engine's autograd bridge, at cfg2's size (256x256, ViT-B/32,
16 cutouts, seeded weights, batch 1, DDIM), on one GPU:

- fused: the package's own CondFnB200 step (one CUDA graph);
- generic: the same guidance written in PyTorch -- the oracle's cond_fn with the CLIP tower in fp16 (LayerNorm in fp32, like the
  reference's clip.model.convert_weights) -- through the package's ddim_sample_with_grad on an input_grad engine: UNet forward +
  p_mean_variance on the engine, CLIP forward / backward in PyTorch, the UNet input gradient on the engine;
- unet_fwd_bwd: `model()` forward + `th.autograd.grad` alone, no guidance;
- generic_engine_clip: the generic step with load_clip's model (clip_model.py) in place of the eager fp16 tower, so both networks run on
  the engine's kernels (timed alternating with a second run of the generic step);
- clip_fwd_bwd: `encode_image` + `th.autograd.grad` alone, load_clip's model against the eager fp16 tower, for ViT-B/32, ViT-B/16,
  ViT-L/14 and RN50 at 16 and 64 images (timed alternating);
- lpips_fwd_bwd: `LPIPS()(x_in, init)` + `th.autograd.grad` into x_in alone (init one broadcast image), lpips.py's LPIPS against the eager
  fp32 oracle.lpips.LPIPSVgg (torch's default cuDNN settings; the same F.conv2d sequence as the `lpips` package), at 256^2 and 512^2,
  batch 1 and 4 (timed alternating);
- init_step: the generic step with an init image (init_scale 1000): the oracle's cond_fn on load_clip's model, LPIPS and engine.model,
  against the fused step of an engine built with the same LPIPS weights (timed alternating).

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


def timed_alternating(fns: dict, steps, warmup):
    """{name: median ms}: every fn warmed up, then the timed calls interleaved (a, b, a, b, ...) so that clock or thermal drift hits
    all arms alike"""
    for fn in fns.values():
        for _ in range(warmup):
            fn()
    th.cuda.synchronize()
    ms = {k: [] for k in fns}
    for _ in range(steps):
        for k, fn in fns.items():
            a, b = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ms[k].append(a.elapsed_time(b))
    return {k: statistics.median(v) for k, v in ms.items()}


def eager_fp16(tower):
    """the oracle tower the way the reference runs CLIP on CUDA: fp16 weights, normalisation layers in fp32"""
    tower = tower.cuda().half()
    for m in tower.modules():
        if isinstance(m, (th.nn.LayerNorm, th.nn.BatchNorm2d)):
            m.float()
    for prm in tower.parameters():
        prm.requires_grad_(False)
    return tower


def clip_fwd_bwd(steps, warmup):
    """encode_image + autograd.grad of the input, engine (load_clip) vs eager fp16, per tower and image count"""
    from clip_guided_diffusion_b200 import clip_util
    from clip_guided_diffusion_b200 import rn as prn
    from oracle import clip_rn as orn
    from oracle.clip_vit import VIT_CONFIGS, CLIPVisualOnly
    out = {}
    for name in ("ViT-B/32", "ViT-B/16", "ViT-L/14", "RN50"):
        if name in pv.VIT_CONFIGS:
            cfg = pv.VIT_CONFIGS[name]
            sd = pw.seeded_state_dict(pw.vit_param_shapes(cfg), 1235)
            eager = CLIPVisualOnly(VIT_CONFIGS[name]).eval()
            eager.load_state_dict(sd)
        else:
            cfg = prn.RN_CONFIGS[name]
            sd = pw.seeded_rn_state_dict(cfg, seed=3)
            eager = orn.CLIPVisualRN(orn.RNConfig(tuple(cfg.layers), cfg.output_dim, cfg.input_resolution, cfg.width)).eval()
            eager.load_state_dict(sd, strict=False)
        eager = eager_fp16(eager)
        R, D = cfg.input_resolution, cfg.output_dim
        for n in (16, 64):
            model, _ = clip_util.load_clip(name, "cuda", clip_state_dict=sd, max_images=n)
            x = th.randn(n, 3, R, R, device="cuda")
            w = th.randn(n, D, device="cuda")

            def run(m):
                def fn():
                    xe = x.detach().requires_grad_()
                    return th.autograd.grad((w * m.encode_image(xe).float()).sum(), xe)
                return fn
            out[f"{name} x{n}"] = timed_alternating({"engine": run(model), "eager_fp16": run(eager)}, steps, warmup)
            del model
            th.cuda.empty_cache()
    return out


def lpips_fwd_bwd(steps, warmup):
    """LPIPS forward + autograd.grad into x_in, lpips.py's LPIPS vs the eager fp32 oracle, per size and batch"""
    from clip_guided_diffusion_b200 import lpips as pl
    from oracle import lpips as ol
    sd = ol.seeded_state_dict()
    eager = ol.LPIPSVgg({k: v.cuda() for k, v in sd.items()}).cuda()
    out = {}
    for size in (256, 512):
        for n in (1, 4):
            model = pl.LPIPS(lpips_state_dict=sd)
            x, init = th.rand(n, 3, size, size, device="cuda") * 2 - 1, th.rand(1, 3, size, size, device="cuda") * 2 - 1

            def run(m):
                def fn():
                    xe = x.detach().requires_grad_()
                    return th.autograd.grad(m(xe, init).sum() * 1000.0, xe)
                return fn
            out[f"{size}x{size} x{n}"] = timed_alternating({"engine": run(model), "eager_fp32": run(eager)}, steps, warmup)
            del model
            th.cuda.empty_cache()
    return out


def init_step(steps, warmup, ucfg, usd, vcfg, vsd, diff, tgt, x, y):
    """cfg2 DDIM step with an init image: fused (CondFnB200 with LPIPS) vs generic (OracleCondFn, load_clip, LPIPS, engine.model)"""
    from clip_guided_diffusion_b200 import clip_util
    from clip_guided_diffusion_b200 import lpips as pl
    from oracle import guidance as og
    from oracle import lpips as ol
    lsd = ol.seeded_state_dict()
    init = th.rand(1, 3, 256, 256, device="cuda") * 2 - 1
    eng = pg.GuidedStepB200(ucfg, usd, vcfg, vsd, batch=1, num_cutouts=16, device="cuda", lpips_sd=lsd, init_scale=1000.0)
    eng.set_targets(tgt, th.ones(1))
    eng.set_init_image(init)
    cond = pg.CondFnB200(eng, diff, pg.MakeCutouts(224, 16))
    geng = pg.GuidedStepB200(ucfg, usd, batch=1, device="cuda", input_grad=True)
    eclip, _ = clip_util.load_clip("ViT-B/32", "cuda", clip_state_dict=vsd, max_images=16)
    ocond = og.OracleCondFn(diff, eclip, tgt.cuda(), th.ones(1, device="cuda"), cut_size=224, num_cutouts=16, lpips_model=pl.LPIPS(lpips_state_dict=lsd),
                            init_tensor=init, init_scale=1000.0)
    ocond.current_timestep = 30
    t = th.full((1,), 30, dtype=th.long, device="cuda")
    res = timed_alternating({"fused": lambda: eng.fused_step(diff, "ddim", 30, x, y, cond),
                             "generic": lambda: diff.ddim_sample_with_grad(geng.model, x, t, clip_denoised=False, cond_fn=ocond, model_kwargs={"y": y})},
                            steps, warmup)
    del eng, cond, geng, eclip, ocond
    th.cuda.empty_cache()
    return res


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else th.cuda.get_device_name(0)


def main():
    from oracle import guidance as og
    from oracle.clip_vit import VIT_CONFIGS, CLIPVisualOnly
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", choices=["lpips"], help="only the LPIPS arms (lpips_fwd_bwd, init_step)")
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
    if args.only == "lpips":
        x = th.randn(1, 3, 256, 256, device="cuda")
        res["init_step_ms"] = init_step(args.steps, args.warmup, ucfg, usd, vcfg, vsd, diff, tgt, x, y)
        res["lpips_fwd_bwd_ms"] = lpips_fwd_bwd(args.steps, args.warmup)
        print(json.dumps(res))
        return

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

    from clip_guided_diffusion_b200 import clip_util
    eclip, _ = clip_util.load_clip("ViT-B/32", "cuda", clip_state_dict=vsd, max_images=16)
    econd = og.OracleCondFn(diff, eclip, tgt.cuda(), th.ones(1, device="cuda"), cut_size=224, num_cutouts=16)
    econd.current_timestep = 30
    pair = timed_alternating({c: (lambda c=c: diff.ddim_sample_with_grad(geng.model, x, t, clip_denoised=False, cond_fn=c, model_kwargs={"y": y}))
                              for c in (ocond, econd)}, args.steps, args.warmup)
    res["generic_step_ms_alternating"], res["generic_engine_clip_step_ms"] = pair[ocond], pair[econd]
    del geng, eclip
    th.cuda.empty_cache()
    res["clip_fwd_bwd_ms"] = clip_fwd_bwd(args.steps, args.warmup)
    res["init_step_ms"] = init_step(args.steps, args.warmup, ucfg, usd, vcfg, vsd, diff, tgt, x, y)
    res["lpips_fwd_bwd_ms"] = lpips_fwd_bwd(args.steps, args.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
