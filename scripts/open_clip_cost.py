"""What the OpenCLIP towers cost the guided step, printed as one JSON line beside the card's name, power limit and SM clock.

1. The step of `bench.py`'s cfg2 (256x256, ddim250, one image, 16 cutouts, seeded weights), replayed from its CUDA graph with windows and
   scalars staged per step, for OpenAI ViT-B/32, open_clip:ViT-B-32, open_clip:ViT-L-14 and open_clip:ViT-H-14.  All engines are built
   first; the rounds alternate between them, so a slow phase of a shared machine hits every arm alike.  Medians of CUDA-event times.
2. The ViT-H-14 tower alone at 16 cutouts: forward + input-gradient backward (vit_fwd .. vit_end) eagerly, CUDA events around `reps`
   runs, next to the padded (heads at 128) and unpadded (heads at 80) multiply-add counts computed from shapes.

    python scripts/open_clip_cost.py [--rounds 5] [--steps 20] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys

import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.ensemble_cost import card, time_steps  # noqa: E402

ARMS = {"openai:ViT-B/32": "ViT-B/32", "open_clip:ViT-B-32": "open_clip:ViT-B-32", "open_clip:ViT-L-14": "open_clip:ViT-L-14",
        "open_clip:ViT-H-14": "open_clip:ViT-H-14"}


def tower_cfg(name):
    from clip_guided_diffusion_b200.vit import OPEN_CLIP_CONFIGS, VIT_CONFIGS
    return OPEN_CLIP_CONFIGS[name[len("open_clip:"):]].vision if name.startswith("open_clip:") else VIT_CONFIGS[name]


def vit_flops(cfg, n, head_dim):
    """2 x multiply-adds of one forward of n images with every head `head_dim` wide (q / k / v / attention / out_proj at that width;
    the backward's dgrads cost 2x this, weight gradients do not exist); patch embedding, LayerNorms and the projection included"""
    T, w, L = cfg.tokens, cfg.width, cfg.layers
    a = cfg.heads * head_dim
    per_layer = T * (3 * a * w + a * w + 8 * w * w) + 2 * T * T * a
    return 2.0 * n * (L * per_layer + cfg.grid ** 2 * 3 * cfg.patch_size ** 2 * w + w * cfg.output_dim)


def tower_alone(name, n=16, reps=20):
    from clip_guided_diffusion_b200 import weights as pw
    from clip_guided_diffusion_b200.vit import ViTB200
    cfg = tower_cfg(name)
    net = ViTB200(cfg, pw.seeded_state_dict(pw.vit_param_shapes(cfg), 1235), n_images=n, device="cuda")
    net.plan.view(net.patches).copy_(th.randn(net.patches.numel, device="cuda").half())
    net.plan.view(net.d_embeds).copy_(th.randn(net.d_embeds.numel, device="cuda"))
    for _ in range(3):
        net.plan.run_range("vit_fwd", "vit_end")
    times = []
    for _ in range(5):
        t0, t1 = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(reps):
            net.plan.run_range("vit_fwd", "vit_end")
        t1.record()
        th.cuda.synchronize()
        times.append(t0.elapsed_time(t1) / reps)
    ms = statistics.median(times)
    padded, unpadded = vit_flops(cfg, n, cfg.head_pad), vit_flops(cfg, n, cfg.head_width)
    del net
    th.cuda.empty_cache()
    return {"tower": name, "images": n, "fwd_bwd_ms_median": round(ms, 3), "fwd_bwd_ms_all": [round(t, 3) for t in times],
            "gflop_fwd_bwd_padded": round(3 * padded / 1e9, 1), "gflop_fwd_bwd_unpadded": round(3 * unpadded / 1e9, 1),
            "padded_over_unpadded": round(padded / unpadded, 4), "tflops_executed": round(3 * padded / (ms * 1e-3) / 1e12, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/open_clip_cost.json")
    args = ap.parse_args()
    if not th.cuda.is_available():
        raise SystemExit("open_clip_cost.py times the step on a CUDA device; none found")
    from clip_guided_diffusion_b200 import gaussian_diffusion as pgd
    from clip_guided_diffusion_b200 import guidance as pg
    from clip_guided_diffusion_b200 import unet as pu
    from clip_guided_diffusion_b200 import weights as pw
    ucfg = pu.config_for(256, True)
    usd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234)
    diff = pgd.create_gaussian_diffusion(1000, "linear", "ddim250", rescale_timesteps=ucfg.rescale_timesteps)
    engines = {}
    for k, name in ARMS.items():
        cfg = tower_cfg(name)
        eng = pg.GuidedStepB200(ucfg, usd, cfg, pw.seeded_state_dict(pw.vit_param_shapes(cfg), 1235), batch=1, num_cutouts=16, device="cuda")
        eng.set_targets(th.randn(1, cfg.output_dim, generator=th.Generator().manual_seed(1)), th.ones(1))
        engines[k] = (eng, [pg.MakeCutouts(cfg.input_resolution, 16)])
    th.manual_seed(0)
    for eng, mks in engines.values():  # warm-up: graph capture, module load
        time_steps(eng, mks, diff, 3)
    times = {k: [] for k in ARMS}
    for _ in range(args.rounds):
        for k, (eng, mks) in engines.items():
            times[k].append(time_steps(eng, mks, diff, args.steps))
    med = {k: statistics.median(v) for k, v in times.items()}
    launches = {k: eng.launches_per_step("ddim") for k, (eng, _) in engines.items()}
    del engines
    th.cuda.empty_cache()
    res = {**card(), "workload": "256x256 ddim250, batch 1, 16 cutouts, seeded weights, guided step from its CUDA graph",
           "rounds": args.rounds, "steps_per_round": args.steps,
           "step_ms_median": {k: round(v, 3) for k, v in med.items()},
           "step_ms_all": {k: [round(t, 3) for t in v] for k, v in times.items()},
           "launches_per_step": launches,
           "vit_h_tower": tower_alone("open_clip:ViT-H-14")}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "open_clip_cost.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
