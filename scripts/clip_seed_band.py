#!/usr/bin/env python
"""Choose CLIP_SEED's BAND (clip_model.py CLIP_SEED_BAND): the target magnitude of the largest seed value of the CLIP tower backward.

For each tower (ViT-B/32, ViT-B/16, ViT-L/14, RN50; seeded weights, 16 images) one forward, then one backward per candidate band
2^0 .. 2^15 with the seed written as CLIP_SEED writes it (each row scaled by the power of two that puts its max |.| in (band / 2,
band]).  The arena holds every intermediate gradient of the backward, so for each band it records:
- max16: the largest |fp16| over the tower's gradient buffers (the fp16 buffers the backward writes), inf if one overflowed;
- headroom: 65504 / max16;
- flushed: the fraction of d_patches (real columns) that are zero or subnormal in fp16.
The chosen band is the largest one that leaves at least 2^4 of headroom in every tower.  Seeded weights are not the published
checkpoints: the band rests on seeded towers.

    python scripts/clip_seed_band.py                     # prints one JSON line, with the card's name and power limit
    python scripts/clip_seed_band.py open_clip:ViT-H-14  # other towers: any VIT_CONFIGS / RN_CONFIGS / "open_clip:<arch>" names
"""
from __future__ import annotations

import json
import math
import os
import sys

import torch as th

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from clip_guided_diffusion_b200 import clip_model as cm  # noqa: E402
from clip_guided_diffusion_b200 import rn as prn  # noqa: E402
from clip_guided_diffusion_b200 import vit as pv  # noqa: E402
from clip_guided_diffusion_b200 import weights as pw  # noqa: E402
from scripts.autograd_step_cost import card  # noqa: E402

TOWERS = ("ViT-B/32", "ViT-B/16", "ViT-L/14", "RN50")
BANDS = [2.0 ** k for k in range(16)]


def measure(name, n=16):
    if name.startswith("open_clip:"):
        cfg = pv.OPEN_CLIP_CONFIGS[name[len("open_clip:"):]].vision
        sd = pw.seeded_state_dict(pw.vit_param_shapes(cfg), 1235)
    elif name in pv.VIT_CONFIGS:
        cfg = pv.VIT_CONFIGS[name]
        sd = pw.seeded_state_dict(pw.vit_param_shapes(cfg), 1235)
    else:
        cfg = prn.RN_CONFIGS[name]
        sd = pw.seeded_rn_state_dict(cfg, seed=3)
    model = cm.ClipModelB200(cfg, sd, n, "cuda")
    plan, R, D, P = model.plan, cfg.input_resolution, cfg.output_dim, cfg.patch_size
    g = th.Generator(device="cuda").manual_seed(0)
    model.forward(th.randn(n, 3, R, R, device="cuda", generator=g))
    d = th.randn(n, D, device="cuda", generator=g)
    consts = {off for _, off, _ in plan.const_index}
    halves = [b for b in plan.bufs if b.dt == "h" and b.off not in consts]
    before = [plan.view(b).clone() for b in halves]
    plan.view(model.tower.d_embeds, (n, D)).copy_(d)
    plan.run_range("vit_bwd", "vit_end")
    th.cuda.synchronize()
    grads = [b for b, v in zip(halves, before) if not th.equal(plan.view(b).view(th.int16), v.view(th.int16))]
    dp = plan.view(model.tower.d_patches, (n, cfg.grid ** 2, cfg.kpad))[:, :, :3 * P * P]
    m = d.abs().amax(1, keepdim=True)
    rows = []
    for band in BANDS:
        scale = th.exp2(th.floor(th.log2(band / m)))
        plan.view(model.tower.d_embeds, (n, D)).copy_(d * scale)
        plan.run_range("vit_bwd", "vit_end")
        mx = max(float(plan.view(b).float().abs().nan_to_num(nan=math.inf).max()) for b in grads)
        flushed = float((dp.float().abs() < 2.0 ** -14).double().mean())
        rows.append({"band": band, "max16": mx, "headroom_log2": math.log2(65504 / mx) if math.isfinite(mx) and mx > 0 else None,
                     "flushed": flushed})
    del model
    th.cuda.empty_cache()
    return {"grad_buffers": len(grads), "bands": rows}


def main():
    if not th.cuda.is_available():
        raise SystemExit("needs a GPU")
    res = {"card": card(), "images": 16, "weights": "seeded (pw.seeded_state_dict / seeded_rn_state_dict), not the published checkpoints"}
    res["towers"] = {name: measure(name) for name in (sys.argv[1:] or TOWERS)}
    ok = [b for b in BANDS if all(r["headroom_log2"] is not None and r["headroom_log2"] >= 4
                                  for t in res["towers"].values() for r in t["bands"] if r["band"] == b)]
    res["chosen_band"] = max(ok) if ok else None
    if ok:
        res["headroom_log2_at_chosen"] = min(r["headroom_log2"] for t in res["towers"].values() for r in t["bands"] if r["band"] == max(ok))
    # every tower's headroom at the band the package ships
    res["headroom_log2_at_shipped_band"] = {name: next(r["headroom_log2"] for r in t["bands"] if r["band"] == cm.CLIP_SEED_BAND)
                                           for name, t in res["towers"].items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
