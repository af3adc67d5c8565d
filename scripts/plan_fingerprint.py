#!/usr/bin/env python
"""Digests of the guided-step engine's plan for a set of configurations, built on the CPU (no GPU, no native plan).

    python scripts/plan_fingerprint.py [NAME ...]

For each configuration it prints one row of digests:
- ops: the op list (code, flags, ints, floats, and each pointer as (buffer number, name, dtype, numel, element offset)), the buffers
  numbered in order of first use, so that the order in which the engine allocates them does not change the digest;
- marks: the range marks and the op indices they point at;
- bufs: the multiset of buffers (name, dtype, numel);
- consts: the multiset of packed constants (name, bytes);
- lower: the C structs `plan.lower(0)` builds, which also depend on the arena offsets.

Two engine versions that must build the same plans are compared by running this script on both and diffing the output."""
from __future__ import annotations

import hashlib
import os
import sys

import torch as th

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from clip_guided_diffusion_b200 import guidance as pg  # noqa: E402
from clip_guided_diffusion_b200 import rn as prn  # noqa: E402
from clip_guided_diffusion_b200 import unet as pu  # noqa: E402
from clip_guided_diffusion_b200 import vit as pv  # noqa: E402
from clip_guided_diffusion_b200 import weights as pw  # noqa: E402


def _h(obj) -> str:
    return hashlib.sha256(repr(obj).encode() if not isinstance(obj, bytes) else obj).hexdigest()[:12]


def digests(plan) -> dict:
    order = {}

    def ptr(p):
        if p is None:
            return None
        b, eoff = p
        k = order.setdefault(id(b), len(order))
        return (k, b.name, b.dt, b.numel, eoff)
    ops = [(op.code, op.flags, list(op.i), [float(v) for v in op.f], [ptr(p) for p in op.p]) for op in plan.ops]
    arena = plan.arena.numpy()
    consts = sorted((name, hashlib.sha256(arena[off:off + n].tobytes()).hexdigest()) for name, off, n in plan.const_index)
    return dict(ops=_h(ops), marks=_h(sorted(plan.marks.items())), bufs=_h(sorted((b.name, b.dt, b.numel) for b in plan.bufs)),
                consts=_h(consts), lower=_h(bytes(plan.lower(0))))


def _vit(name_or_cfg):
    cfg = pv.VIT_CONFIGS[name_or_cfg] if isinstance(name_or_cfg, str) else name_or_cfg
    return cfg, pw.seeded_state_dict(pw.vit_param_shapes(cfg), 1235)


def _rn(cfg):
    return cfg, pw.seeded_rn_state_dict(cfg, seed=5)


TINY_UNET = pu.UNetConfig(image_size=32, model_channels=64, num_res_blocks=1, channel_mult=(1, 2), attention_resolutions=(16,),
                          num_classes=10)
TINY_VIT = pv.ViTConfig(32, 16, 64, 1, 32)
TINY_VIT2 = pv.ViTConfig(64, 32, 64, 1, 48)
TINY_RN = prn.RNConfig(layers=(1, 1, 1, 1), output_dim=48, input_resolution=32, width=64)


def _unet(cfg):
    return cfg, pw.seeded_state_dict(pw.unet_param_shapes(cfg), 1234)


def full(size, clip, cutn, lpips=False):
    extra = dict(lpips_sd=pw.seeded_lpips_state_dict(), init_scale=1000.0) if lpips else {}
    return (*_unet(pu.config_for(size, class_cond=True)), *_vit(clip)), dict(batch=1, num_cutouts=cutn, **extra)


def tiny(towers=(TINY_VIT,), **kw):
    """towers: a tuple is one tower per entry (a single tower passed as a plain config), a list is passed as a list"""
    cfgs, sds = zip(*[(_rn(c) if isinstance(c, prn.RNConfig) else _vit(c)) for c in towers])
    plain = isinstance(towers, tuple) and len(towers) == 1
    kw.setdefault("batch", 2)
    kw.setdefault("num_cutouts", 4)
    return (*_unet(TINY_UNET), cfgs[0] if plain else list(cfgs), sds[0] if plain else list(sds)), kw


CONFIGS = {
    "cfg2": lambda: full(256, "ViT-B/32", 16),
    "cfg3": lambda: full(256, "ViT-B/32", 32),
    "cfg4": lambda: full(512, "ViT-B/16", 16),
    "cfg5-lpips": lambda: full(512, "ViT-L/14", 64, lpips=True),
    "tiny": lambda: tiny(),
    "tiny-list1": lambda: tiny(towers=[TINY_VIT]),
    "cutn_variants": lambda: tiny(num_cutouts=8, cutn_variants=(2, 4)),
    "lanczos3": lambda: tiny(num_cutouts=3, cutout_resize="lanczos3"),
    "use_augs": lambda: tiny(use_augs=True),
    "vit_streams2": lambda: tiny(vit_streams=2),
    "rn": lambda: tiny(towers=(TINY_RN,)),
    "non-square": lambda: tiny(height=32, width=64, batch=1),
    "seed_scale": lambda: tiny(seed_scale=1024.0),
    "magnitude-ws2": lambda: tiny(batch=1, use_magnitude=True, world_size=2, rank=1),
    "magnitude-sat-P3": lambda: tiny(batch=1, use_magnitude=True, sat_scale=30.0, max_prompts=3),
    "lpips": lambda: tiny(lpips_sd=pw.seeded_lpips_state_dict(), init_scale=1000.0),
    "no-clip": lambda: ((*_unet(TINY_UNET), None, None), dict(batch=2)),
    "three-towers": lambda: tiny(towers=(TINY_VIT, TINY_RN, TINY_VIT2), num_cutouts=8, cutn_variants=(2, 4)),
    "two-towers-ws2-streams": lambda: tiny(towers=(TINY_VIT, TINY_VIT2), use_magnitude=True, world_size=2, vit_streams=2),
}


def main(names):
    th.set_num_threads(min(8, os.cpu_count() or 1))
    cols = ("ops", "marks", "bufs", "consts", "lower")
    print("| config | " + " | ".join(cols) + " |")
    print("|---" * (len(cols) + 1) + "|")
    for name in names or CONFIGS:
        args, kw = CONFIGS[name]()
        eng = pg.GuidedStepB200(*args, device="cpu", **kw)
        d = digests(eng.plan)
        print(f"| {name} | " + " | ".join(d[c] for c in cols) + " |", flush=True)
        del eng


if __name__ == "__main__":
    main(sys.argv[1:])
