"""Cost of the cutout resampling modes on the GPU: pool (adaptive_avg_pool2d, the reference's), lanczos3 (ResizeRight) and lanczos3 after
the use_augs pipeline, at cfg2 (256², ViT-B/32, 16 cutouts) and cfg4 (512², ViT-B/16) sizes, square and with a +64 width offset.

Per engine: the cutout forward launches (cut_fwd -> sph ranges) plus the cutout backward launches (cut_bwd -> cut_end), and one whole guided
DDIM step from its CUDA graph, each timed with CUDA events; the arms alternate round by round on the same windows, and the median over the
rounds is reported.  The card's name and power limit are read in the same run.  Prints one JSON line (and writes it to
DIR/rr_cutout_cost.json with --out DIR).

    python scripts/rr_cutout_cost.py [--rounds 20] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys

import torch as th

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from clip_guided_diffusion_b200 import gaussian_diffusion as pgd  # noqa: E402
from clip_guided_diffusion_b200 import guidance as pg  # noqa: E402
from clip_guided_diffusion_b200 import unet as pu  # noqa: E402
from clip_guided_diffusion_b200 import vit as pv  # noqa: E402
from clip_guided_diffusion_b200 import weights as pw  # noqa: E402

SIZES = {"cfg2_256x256": (256, 256, 256, "ViT-B/32"), "cfg2_256x320": (256, 256, 320, "ViT-B/32"), "cfg4_512x512": (512, 512, 512, "ViT-B/16")}
ARMS = {"pool": dict(), "lanczos3": dict(cutout_resize="lanczos3"), "lanczos3_augs": dict(cutout_resize="lanczos3", use_augs=True)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else th.cuda.get_device_name()


def timed(fn, reps=5):
    a, b = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/rr_cutout_cost.json")
    args = ap.parse_args()
    if not th.cuda.is_available():
        sys.exit("rr_cutout_cost.py measures on the GPU; no CUDA device found")
    out = {"card": card(), "rounds": args.rounds, "ms": {}}
    pdiff = pgd.create_gaussian_diffusion(1000, "linear", "25")
    for size, (res, H, W, clip) in SIZES.items():
        ucfg, vcfg = pu.config_for(res, True), pv.VIT_CONFIGS[clip]
        usd, vsd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234), pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 1235)
        engines = {}
        for arm, kw in ARMS.items():
            eng = pg.GuidedStepB200(ucfg, usd, vcfg, vsd, batch=1, height=H, width=W, num_cutouts=16, device="cuda", **kw)
            eng.set_targets(th.randn(1, vcfg.output_dim), th.ones(1))
            engines[arm] = eng
        th.manual_seed(0)
        coords = pg.MakeCutouts(224, 16)._generate_coords(H, W, 16)
        coords = [(min(ox, W - 1), min(oy, H - 1), s) for ox, oy, s in coords]  # keep every window non-empty on the offset image
        for arm, eng in engines.items():
            th.manual_seed(1)
            eng.stage_step(pdiff.scalar_table(12, 12, 0.0), coords, pdiff.model_timestep(12), th.zeros(1, dtype=th.long))
            eng.img(eng.unet.x_in).normal_()
            eng.replay("ddim", 16)  # eager run + capture
            for _ in range(3):
                eng.replay("ddim", 16)
        th.cuda.synchronize()
        samples = {arm: {"cutouts": [], "step": []} for arm in engines}
        for _ in range(args.rounds):
            for arm, eng in engines.items():
                run = eng.plan.run_range
                samples[arm]["cutouts"].append(timed(lambda: (run("cut_fwd", "sph"), run("cut_bwd", "cut_end"))))
                samples[arm]["step"].append(timed(lambda: eng.replay("ddim", 16), reps=3))
        for arm, s in samples.items():
            out["ms"][f"{size}/{arm}"] = {k: round(sorted(v)[len(v) // 2], 4) for k, v in s.items()}
        del engines
        th.cuda.empty_cache()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "rr_cutout_cost.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
