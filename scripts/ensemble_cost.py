"""What each extra CLIP tower costs the guided step, printed as one JSON line beside the card's name, power limit and SM clock.

The step of `bench.py`'s cfg2 -- 256x256, ddim250, one image, 16 cutouts, seeded weights -- replayed from its CUDA graph (windows and
scalars staged per step as the sampling loop does) for ViT-B/32, ViT-B/16 and RN50 alone, ViT-B/32 + ViT-B/16, and
ViT-B/32 + ViT-B/16 + RN50.  All five engines are built first; the rounds then alternate between them, so a slow phase of a shared
machine hits every configuration alike.

    python scripts/ensemble_cost.py [--rounds 5] [--steps 20] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = {"B/32": ["ViT-B/32"], "B/16": ["ViT-B/16"], "RN50": ["RN50"], "B/32+B/16": ["ViT-B/32", "ViT-B/16"],
           "B/32+B/16+RN50": ["ViT-B/32", "ViT-B/16", "RN50"]}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm, sm_max = (v.strip() for v in q.split(","))
        return {"gpu": name, "power_limit": power, "sm_clock": sm, "max_sm_clock": sm_max}
    except Exception as e:  # noqa: BLE001 -- the numbers stay valid, only their label is missing
        return {"gpu": th.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def build(names, ucfg, usd, tower_sds):
    from clip_guided_diffusion_b200 import guidance as pg
    from clip_guided_diffusion_b200.rn import RN_CONFIGS
    from clip_guided_diffusion_b200.vit import VIT_CONFIGS
    cfgs = [{**VIT_CONFIGS, **RN_CONFIGS}[n] for n in names]
    sds = [tower_sds[n] for n in names]
    one = len(names) == 1
    eng = pg.GuidedStepB200(ucfg, usd, cfgs[0] if one else cfgs, sds[0] if one else sds, batch=1, num_cutouts=16, device="cuda")
    g = th.Generator().manual_seed(1)
    tg = [th.randn(1, c.output_dim, generator=g) for c in cfgs]
    eng.set_targets(tg[0] if one else tg, th.ones(1))
    mks = [pg.MakeCutouts(c.input_resolution, 16) for c in cfgs]
    return eng, mks


def time_steps(eng, mks, diff, steps):
    """ms per guided step: `steps` stage + replay pairs between two CUDA events"""
    x = th.randn(1, 3, 256, 256, device="cuda")
    y = th.zeros(1, dtype=th.long)
    eng.img(eng.unet.x_in).copy_(x)
    t0, t1 = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
    t0.record()
    for k in range(steps):
        t = 200 - k % 50
        per = [mk._generate_coords(256, 256, 16) for mk in mks]
        eng.stage_step(diff.scalar_table(t, t, 0.0), per[0] if len(per) == 1 else per, diff.model_timestep(t), y)
        eng.replay("ddim")
    t1.record()
    th.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/ensemble_cost.json")
    args = ap.parse_args()
    if not th.cuda.is_available():
        raise SystemExit("ensemble_cost.py times the step on a CUDA device; none found")
    from clip_guided_diffusion_b200 import gaussian_diffusion as pgd
    from clip_guided_diffusion_b200 import unet as pu
    from clip_guided_diffusion_b200 import weights as pw
    from clip_guided_diffusion_b200.rn import RN_CONFIGS
    from clip_guided_diffusion_b200.vit import VIT_CONFIGS
    ucfg = pu.config_for(256, True)
    usd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234)
    tower_sds = {"ViT-B/32": pw.seeded_state_dict(pw.vit_param_shapes(VIT_CONFIGS["ViT-B/32"]), 1235),
                 "ViT-B/16": pw.seeded_state_dict(pw.vit_param_shapes(VIT_CONFIGS["ViT-B/16"]), 1236),
                 "RN50": pw.seeded_rn_state_dict(RN_CONFIGS["RN50"], seed=1237)}
    diff = pgd.create_gaussian_diffusion(1000, "linear", "ddim250", rescale_timesteps=ucfg.rescale_timesteps)
    engines = {k: build(v, ucfg, usd, tower_sds) for k, v in CONFIGS.items()}
    th.manual_seed(0)
    for eng, mks in engines.values():  # warm-up: graph capture, module load
        time_steps(eng, mks, diff, 3)
    times = {k: [] for k in CONFIGS}
    for _ in range(args.rounds):
        for k, (eng, mks) in engines.items():
            times[k].append(time_steps(eng, mks, diff, args.steps))
    med = {k: statistics.median(v) for k, v in times.items()}
    res = {**card(), "workload": "256x256 ddim250, batch 1, 16 cutouts, seeded weights, guided step from its CUDA graph",
           "rounds": args.rounds, "steps_per_round": args.steps,
           "step_ms_median": {k: round(v, 3) for k, v in med.items()},
           "step_ms_all": {k: [round(t, 3) for t in v] for k, v in times.items()},
           "launches_per_step": {k: eng.launches_per_step("ddim") for k, (eng, _) in engines.items()},
           "extra_ms": {"+B/16 on B/32": round(med["B/32+B/16"] - med["B/32"], 3),
                        "+RN50 on B/32+B/16": round(med["B/32+B/16+RN50"] - med["B/32+B/16"], 3)}}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ensemble_cost.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
