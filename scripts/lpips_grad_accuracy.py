#!/usr/bin/env python
"""How close the input gradient of LPIPS(x_in, init) comes to the fp32 oracle (oracle.lpips.LPIPSVgg), by kind of input, and why.

For 256^2 images (batch 1, one init image; seeded weights) and two kinds of input -- smooth (bicubic-upsampled noise, closer to real
images) and uniform noise in [-1, 1] -- d (1000 * LPIPS) / d x_in of:
- lpips.py's LPIPS (fp16 trunks, LPIPS_PAIR_BWD seeds, BAND);
- the fused LpipsB200 (the same fp16 trunk with the LPIPS_TAP seeds and a fixed gradient scale: no LPIPS_SEED, no BAND);
- the fp32 oracle run under torch.autocast(fp16): any VGG16 with fp16 activations;
- the oracle in float64 (how well-conditioned the fp32 reference itself is);
each as cos / rel against the fp32 oracle, and the number of all-zero pixels of each tap (where 1 / (||f|| + 1e-10) explodes).

    python scripts/lpips_grad_accuracy.py      # prints one JSON line, with the card's name and power limit
"""
from __future__ import annotations

import json
import os
import sys

import torch as th

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from clip_guided_diffusion_b200 import lpips as pl  # noqa: E402
from oracle import lpips as ol  # noqa: E402
from scripts.autograd_step_cost import card  # noqa: E402


def inputs(kind, size, seed):
    g = th.Generator(device="cuda").manual_seed(seed)
    if kind == "smooth":
        low = th.randn(1, 3, size // 16, size // 16, device="cuda", generator=g)
        return th.tanh(th.nn.functional.interpolate(low, size=(size, size), mode="bicubic", align_corners=False))
    return th.rand(1, 3, size, size, device="cuda", generator=g) * 2 - 1


def grad(fn, x, init):
    xe = x.clone().requires_grad_()
    return th.autograd.grad(fn(xe, init).sum() * 1000.0, xe)[0].double()


def metrics(a, b):
    return {"cos": float(th.nn.functional.cosine_similarity(a.flatten(), b.flatten(), dim=0)), "rel": float((a - b).norm() / b.norm())}


def fused_grad(sd, x, init):
    from tests.test_lpips_cpu import build
    _, plan, lp, x_src, g_dst = build("cuda", 1, x.shape[2], x.shape[3], 1000.0)
    lp.set_init_image(init)
    plan.view(x_src, tuple(x.shape)).copy_(x)
    plan.view(g_dst, tuple(x.shape)).zero_()
    plan.run_range("lpips", "lpips_end")
    th.cuda.synchronize()
    return plan.view(g_dst, tuple(x.shape)).double().clone()


def main():
    if not th.cuda.is_available():
        raise SystemExit("needs a GPU")
    sd = ol.seeded_state_dict()
    oracle = ol.LPIPSVgg({k: v.cuda() for k, v in sd.items()}).cuda()
    oracle64 = ol.LPIPSVgg(sd).cuda().double()
    oracle64.sd = {k: v.cuda().double() for k, v in sd.items()}  # LPIPSVgg keeps its weights in fp32
    model = pl.LPIPS(lpips_state_dict=sd)
    res = {"card": card(), "size": "256x256, batch 1, one init image", "weights": "seeded (oracle.lpips.seeded_state_dict)"}
    for kind in ("smooth", "uniform"):
        x, init = inputs(kind, 256, 1), inputs(kind, 256, 2)
        ref = grad(oracle, x, init)

        def eager16(a, b):
            with th.autocast("cuda", dtype=th.float16):
                return oracle(a, b).float()
        taps = oracle.features(x)
        res[kind] = {"LPIPS": metrics(grad(model, x, init), ref), "fused LpipsB200": metrics(fused_grad(sd, x, init), ref),
                     "eager fp16 (autocast)": metrics(grad(eager16, x, init), ref),
                     "oracle float64": metrics(grad(oracle64, x.double(), init.double()), ref),
                     "all-zero tap pixels": [int((t.abs().amax(1) == 0).sum()) for t in taps]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
