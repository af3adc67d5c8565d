"""Every GroupNorm, attention and glue-op signature the shipped guided-step plans emit is a case of tests/test_gpu_unet_kernels.py.

The cfg2, cfg4, cfg5, default128 and 64x64 engines are built on the CPU with seeded weights (as scripts/plan_fingerprint.py does); the
signature of every GN_*, ATTN_*, POOL2, UP2, ADD, COPY, NCHW_TO_PM and PM_TO_NCHW op -- shape, leading dimensions, flags and, for the
GroupNorms, the engine the plan chose -- is looked up in the GPU file's case tables.  A plan change that introduces an untested shape
fails here, on a machine without a GPU."""
from __future__ import annotations

import functools

import pytest
import torch as th

from clip_guided_diffusion_b200 import guidance as pg
from clip_guided_diffusion_b200 import unet as pu
from clip_guided_diffusion_b200 import vit as pv
from clip_guided_diffusion_b200 import weights as pw
from clip_guided_diffusion_b200._lib import OP
from tests import test_gpu_unet_kernels as K

CODE = {v: k for k, v in OP.items()}


def _full(size, clip, cutn, lpips=False):
    ucfg, vcfg = pu.config_for(size, class_cond=True), pv.VIT_CONFIGS[clip]
    extra = dict(lpips_sd=pw.seeded_lpips_state_dict(), init_scale=1000.0) if lpips else {}
    return lambda: pg.GuidedStepB200(ucfg, pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234), vcfg,
                                     pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 1235), device="cpu", batch=1, num_cutouts=cutn,
                                     **extra)


ENGINES = {  # the configurations of tests/test_gpu_baseline_configs.py, and the 64x64 checkpoint
    "cfg2": _full(256, "ViT-B/32", 16),
    "cfg4": _full(512, "ViT-B/16", 16),
    "cfg5": _full(512, "ViT-L/14", 64, lpips=True),
    "default128": _full(128, "ViT-B/32", 16),
    "64x64": _full(64, "ViT-B/32", 16),
}


def plan_signatures(eng) -> set:
    """{(kind, *signature)} of the ops of the engine's plan that tests/test_gpu_unet_kernels.py covers"""
    out = set()
    for op in eng.plan.ops:
        name, i, f = CODE[op.code], op.i, op.f
        if name in ("GN_FWD_FUSED", "GN_FWD_GRID", "GN_APPLY"):
            engine = {"GN_FWD_FUSED": "cluster", "GN_FWD_GRID": "grid", "GN_APPLY": "twopass"}[name]
            ldy = i[5] if name == "GN_APPLY" else i[4]
            emb = (op.p[4] if name == "GN_APPLY" else op.p[3]) is not None
            out.add(("GN_FWD", engine, i[0], i[1], i[2], i[3], ldy, emb, op.flags & 1))
        elif name in ("GN_BWD_FUSED", "GN_BWD_GRID", "GN_BWD_APPLY"):
            engine = {"GN_BWD_FUSED": "cluster", "GN_BWD_APPLY": "twopass"}.get(name) or K.gn_bwd_grid_engine(i[1], i[2])
            ld_dx = i[6] if name == "GN_BWD_APPLY" else i[5]
            out.add(("GN_BWD", engine, i[0], i[1], i[2], i[3], i[4], ld_dx, op.p[5] is not None, op.flags & 1, (op.flags >> 1) & 1))
        elif name in ("ATTN_FWD", "ATTN_BWD"):
            B, heads, T, d, qbs, qrs, qhs, obs, ors, ohs = i[:10]
            assert qbs == T * qrs and obs == T * ors and ohs == d, (name, list(i[:10]))
            legacy = qhs == 3 * d
            assert legacy or qhs == d, (name, list(i[:10]))
            out.add((name, B, heads, T, d, qrs, ors, bool(legacy), op.flags & 1))
        elif name in ("POOL2", "UP2"):
            out.add((name, *i[:6], float(f[0])))
        elif name == "ADD":
            out.add((name, *i[:5]))
        elif name == "COPY":
            out.add((name, *i[:4]))
        elif name == "NCHW_TO_PM":  # flags 4: per-channel shift f1..3 and multiplier f4..6
            out.add((name, *i[:4], op.flags, *(float(v) for v in f[:7 if op.flags & 4 else 1])))
        elif name == "PM_TO_NCHW":  # flags 1: fp32 source, 2: accumulate, 4: per-channel multiplier f1..3
            out.add((name, *i[:4], op.flags, *(float(v) for v in f[:4 if op.flags & 4 else 1])))
    return out


@functools.lru_cache(maxsize=None)
def _signatures(name):
    th.manual_seed(0)
    eng = ENGINES[name]()
    try:
        return frozenset(plan_signatures(eng))
    finally:
        del eng


@pytest.mark.parametrize("name", list(ENGINES))
def test_plan_signatures_are_tested(name):
    sigs = _signatures(name)
    assert any(s[0] == "GN_FWD" for s in sigs) and any(s[0] == "ATTN_FWD" for s in sigs), "no GroupNorm / attention op found"
    covered = K.covered_signatures()
    missing = sorted((s for s in sigs if s not in covered), key=repr)
    assert not missing, f"{name}: {len(missing)} op signature(s) without a case in tests/test_gpu_unet_kernels.py:\n" + \
        "\n".join(map(repr, missing))
