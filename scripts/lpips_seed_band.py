#!/usr/bin/env python
"""Choose LPIPS_SEED's BAND (lpips.py LPIPS_SEED_BAND): the target of |d_loss| * scale, the factor every seed of the LPIPS trunk backwards
is multiplied by.

On seeded LPIPS weights (oracle.lpips.seeded_state_dict), for 64^2, 256^2 and 512^2 images (batch 2, in1 one broadcast init image) and three
kinds of in0 (natural-looking: smooth random fields; random: uniform noise in [-1, 1]; flat: one grey value), one forward, then one
backward of both trunks per candidate band 2^10 .. 2^30: LPIPS_SEED runs, then its scales are overwritten by band / |d_loss| (d_loss = 1)
so each candidate is one backward of the same plan.  For each band it records, over the fp16 buffers the backward writes:
- max16: the largest |fp16| over the gradient buffers (the fp16 buffers the backward writes, found as those whose bits one backward
  changes; the forward activations it reads are not among them), inf if one overflowed, with the seeds' +-60000 saturation (all-zero
  feature pixels) counted separately;
- headroom_log2: log2(65504 / max16) over the non-saturated values;
- flushed: the fraction of the first layer's input gradient (the 3 image channels) that is zero or subnormal in fp16.
The chosen band is the largest with at least 2^4 of headroom in every case.  Seeded weights are not the published checkpoints.

    python scripts/lpips_seed_band.py      # prints one JSON line, with the card's name and power limit
"""
from __future__ import annotations

import json
import math
import os
import sys

import torch as th

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from clip_guided_diffusion_b200 import lpips as pl  # noqa: E402
from scripts.autograd_step_cost import card  # noqa: E402

BANDS = [2.0 ** k for k in range(10, 31)]
SIZES = (64, 256, 512)


def inputs(kind, n, size, seed):
    g = th.Generator(device="cuda").manual_seed(seed)
    if kind == "natural":
        low = th.randn(n, 3, max(2, size // 16), max(2, size // 16), device="cuda", generator=g)
        return th.tanh(th.nn.functional.interpolate(low, size=(size, size), mode="bicubic", align_corners=False))
    if kind == "random":
        return th.rand(n, 3, size, size, device="cuda", generator=g) * 2 - 1
    return th.full((n, 3, size, size), 0.1, device="cuda")


def measure(model, size, kind):
    a, b = inputs(kind, 2, size, 1), inputs("natural", 1, size, 2)
    pp = model.plan_for(size, size, 2, 1)
    p = pp.plan
    pp.forward(a, b)
    consts = {off for _, off, _ in p.const_index}
    halves = [bf for bf in p.bufs if bf.dt == "h" and bf.off not in consts]
    # the gradient buffers: the fp16 buffers whose bits one backward changes (the forward activations it reads stay as they are)
    before = [p.view(bf).clone() for bf in halves]
    p.view(pp.d_loss, (2,)).fill_(1.0)
    p.run_range("lp_seed", "lp_seed0")
    p.run_range("lp_bwd0", "lp_end")
    th.cuda.synchronize()
    grads = [bf for bf, v in zip(halves, before) if not th.equal(p.view(bf).view(th.int16), v.view(th.int16))]
    del before
    first = p.ops[p.marks["lp_bwd1"] - 1].p[0]  # PM_TO_NCHW of trunk 0: its source is d (pixel-major input), 64 channels
    rows = []
    for band in BANDS:
        p.view(pp.d_loss, (2,)).fill_(1.0)
        p.run_range("lp_seed", "lp_seed01")
        p.view(pp.dyn).fill_(band)
        p.run_range("lp_seed01", "lp_seed0")
        p.run_range("lp_bwd0", "lp_end")
        th.cuda.synchronize()
        mx, sat = 0.0, 0
        for bf in grads:
            v = p.view(bf).float().abs().nan_to_num(nan=math.inf)
            sat += int((v == 60000).sum())
            mx = max(mx, float(v[v != 60000].max()) if bool((v != 60000).any()) else 0.0)
        dx = p.arena[first[0].off:first[0].off + first[0].nbytes].view(th.float16).view(2, size * size, 64)[:, :, :3].float()
        rows.append({"band": band, "max16": mx, "saturated": sat, "flushed": float((dx.abs() < 2.0 ** -14).double().mean()),
                     "headroom_log2": math.log2(65504 / mx) if math.isfinite(mx) and mx > 0 else None})
    model.plans.clear()
    th.cuda.empty_cache()
    return {"grad_buffers": len(grads), "bands": rows}


def main():
    if not th.cuda.is_available():
        raise SystemExit("needs a GPU")
    from oracle.lpips import seeded_state_dict
    model = pl.LPIPS(lpips_state_dict=seeded_state_dict())
    res = {"card": card(), "batch": "in0 2 images, in1 1 (broadcast)", "weights": "seeded (oracle.lpips.seeded_state_dict), not the published checkpoints"}
    res["cases"] = {f"{size}-{kind}": measure(model, size, kind) for size in SIZES for kind in ("natural", "random", "flat")}
    ok = [b for b in BANDS if all(r["headroom_log2"] is not None and r["headroom_log2"] >= 4 for c in res["cases"].values() for r in c["bands"]
                                  if r["band"] == b)]
    res["chosen_band"] = max(ok) if ok else None
    if ok:
        res["headroom_log2_at_chosen"] = {c: next(r["headroom_log2"] for r in v["bands"] if r["band"] == max(ok)) for c, v in res["cases"].items()}
        res["flushed_at_chosen"] = {c: next(r["flushed"] for r in v["bands"] if r["band"] == max(ok)) for c, v in res["cases"].items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
