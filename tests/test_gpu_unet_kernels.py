"""The UNet's GroupNorm, attention and glue kernels one by one, at every shape the shipped plans run, against float64 references written
from the op definitions (include/cgd_b200.h; guided-diffusion GroupNorm32 + SiLU + scale-shift, QKVAttention(Legacy), the 2x2 average
pool / nearest up-sampling of Downsample / Upsample and their adjoints, channel concatenation and gradient sums).

Each case is a stand-alone plan.  On CUDA it runs the native kernels (`gpu` tests, production shapes; the references are computed on
the device); on a plan finalized on the CPU it runs through tests/plan_interp.py at a reduced size, which validates the references on a
machine without a GPU.  The references never call the interpreter.  tests/test_unet_kernel_coverage_cpu.py checks that every signature
the cfg2 / cfg4 / cfg5 / default128 / 64x64 plans emit is in the tables below.

Tolerances are element-wise: one fp16 ulp of the float64 value (a correctly rounded result is within half an ulp; the other half
absorbs the fp32 arithmetic before the rounding) plus an fp32 floor derived per op from the kernel's arithmetic -- the summation chain
lengths and the approximate transcendental instructions it uses.

GroupNorm engines and the |mean| / std ratio they are known to be good to.  Every case draws its groups with |mean| / std cycling
through 0, 0.5, 2, 16 and 64, and every engine meets the same bounds at all of them:
* cluster (csrc/norm_fused.cu): exact two-pass statistics (mean, then the sum of (x - mean)^2);
* grid (csrc/norm_grid.cu) and two-pass (csrc/norm.cu): E[(x - p)^2] - (mean - p)^2 about a per-group pivot p, the group's first
  element.  Without the pivot the variance loses ~log2(1 + mean^2 / var) bits: rstd of groups at 16 and 64 std missed its bound.
  The tests draw the pivot from the group's own distribution; a pivot k std from the mean would cost ~log2(1 + k^2) bits again.
"""
import math

import pytest
import torch as th
import torch.nn.functional as F

from clip_guided_diffusion_b200.lpips import SCALE as LPIPS_SCALE
from clip_guided_diffusion_b200.lpips import SHIFT as LPIPS_SHIFT
from clip_guided_diffusion_b200.plan import Plan, gn_fused_cluster, gn_grid_ctas
from tests.kernel_check import D64, U, cases, check, check16, run, ulp16

RATIOS = (0.0, 0.5, 2.0, 16.0, 64.0)  # |mean| / std of the groups, cycled over (image, group)
SENTINEL = 7.0  # guard channels / rows of outputs: must be left alone


def gen(device, seed):
    return th.Generator(device=device).manual_seed(seed)


def dev_of(device):
    return th.device("cuda" if device == "cuda" else "cpu")


def reader(plan, device):
    """Buf -> tensor on the device the references run on"""
    return lambda b, shape=None: plan.view(b, shape).clone()


def strided(t, ld, fill):
    """[..., C] -> [..., ld] with channels C..ld set to `fill`"""
    out = th.full((*t.shape[:-1], ld), fill, dtype=t.dtype, device=t.device)
    out[..., :t.shape[-1]] = t
    return out


def reruns_identical(plan, device, what, inputs, outputs, times=3):
    """Run the plan `times` more times from the same inputs: every output must be bitwise the same as after the first run (fixed-order
    folds; generation-counted barriers and self-resetting counters left behind by a run must not change the next one)."""
    if device != "cuda":
        return
    first = [plan.view(b).clone() for b in outputs]
    for k in range(times - 1):
        for b, t in inputs:
            plan.view(b).copy_(t.reshape(-1).to(plan.view(b).dtype))
        plan.run()
        th.cuda.synchronize()
        for b, f in zip(outputs, first):
            assert th.equal(plan.view(b).view(th.int16 if f.dtype == th.float16 else th.int32), f.view(th.int16 if f.dtype == th.float16 else th.int32)), \
                f"{what}: run {k + 2} differs bitwise from run 1 ({b.name})"


# ---------------------------------------------------------------------------------------------------------------- case tables
# Every signature the cfg2, cfg4, cfg5, default128 and 64x64 plans emit (tests/test_unet_kernel_coverage_cpu.py keeps these complete).
# GN_FWD: (engine, N, HW, C, ldx, ldy, emb, silu); GN_BWD: (engine, N, HW, C, ld_dy, ldx, ld_dx, emb, silu, accumulate), the grid
# backward split into its "ring" and "direct" engines; ATTN: (B, heads, T, d, qkv row stride, out row stride, legacy order, causal);
# POOL2 / UP2: (N, H, W, C, ldx, ldy, scale); ADD: (rows, C, lda, ldb, ldc); COPY: (rows, C, lds, ldd); NCHW_TO_PM: (N, C, HW, ld, flags,
# scale[, shift_0..2, mul_0..2 with flags 4]); PM_TO_NCHW: (N, C, HW, ld, flags, scale[, mul_0..2 with flags 4]).
LPIPS_MUL = tuple(1.0 / s for s in LPIPS_SCALE)  # the per-channel multipliers of the LPIPS ScalingLayer, as lpips.py emits them
GN_FWD_PLAN = [
    ('cluster', 1, 1024, 1024, 1024, 1024, False, 1), ('cluster', 1, 1024, 1024, 1024, 1024, True, 1), ('cluster', 1, 1024, 1280, 1280, 1280, False, 1),
    ('cluster', 1, 1024, 1536, 1536, 1536, False, 1), ('cluster', 1, 1024, 256, 256, 256, True, 1), ('cluster', 1, 1024, 256, 768, 256, False, 1),
    ('cluster', 1, 1024, 512, 1024, 512, False, 1), ('cluster', 1, 1024, 512, 1280, 512, False, 1), ('cluster', 1, 1024, 512, 1536, 512, False, 1),
    ('cluster', 1, 1024, 512, 512, 512, False, 0), ('cluster', 1, 1024, 512, 512, 512, False, 1), ('cluster', 1, 1024, 512, 512, 512, True, 1),
    ('cluster', 1, 1024, 768, 768, 768, False, 1), ('cluster', 1, 1024, 768, 768, 768, True, 1), ('cluster', 1, 256, 1024, 1024, 1024, False, 0),
    ('cluster', 1, 256, 1024, 1024, 1024, False, 1), ('cluster', 1, 256, 1024, 1024, 1024, True, 1), ('cluster', 1, 256, 1024, 2048, 1024, False, 1),
    ('cluster', 1, 256, 1280, 1280, 1280, False, 1), ('cluster', 1, 256, 1536, 1536, 1536, False, 1), ('cluster', 1, 256, 1792, 1792, 1792, False, 1),
    ('cluster', 1, 256, 2048, 2048, 2048, False, 1), ('cluster', 1, 256, 512, 1280, 512, False, 1), ('cluster', 1, 256, 512, 1536, 512, False, 1),
    ('cluster', 1, 256, 512, 512, 512, True, 1), ('cluster', 1, 256, 768, 1536, 768, False, 1), ('cluster', 1, 256, 768, 1792, 768, False, 1),
    ('cluster', 1, 256, 768, 768, 768, False, 0), ('cluster', 1, 256, 768, 768, 768, False, 1), ('cluster', 1, 256, 768, 768, 768, True, 1),
    ('cluster', 1, 4096, 256, 256, 256, False, 1), ('cluster', 1, 4096, 256, 256, 256, True, 1), ('cluster', 1, 4096, 256, 512, 256, False, 1),
    ('cluster', 1, 4096, 256, 768, 256, False, 1), ('cluster', 1, 4096, 512, 1024, 512, False, 1), ('cluster', 1, 4096, 512, 512, 512, False, 1),
    ('cluster', 1, 4096, 512, 512, 512, True, 1), ('cluster', 1, 64, 1024, 1024, 1024, False, 0), ('cluster', 1, 64, 1024, 1024, 1024, False, 1),
    ('cluster', 1, 64, 1024, 1024, 1024, True, 1), ('cluster', 1, 64, 1024, 2048, 1024, False, 1), ('cluster', 1, 64, 1536, 1536, 1536, False, 1),
    ('cluster', 1, 64, 1792, 1792, 1792, False, 1), ('cluster', 1, 64, 2048, 2048, 2048, False, 1), ('cluster', 1, 64, 768, 1536, 768, False, 1),
    ('cluster', 1, 64, 768, 1792, 768, False, 1), ('cluster', 1, 64, 768, 768, 768, False, 0), ('cluster', 1, 64, 768, 768, 768, False, 1),
    ('cluster', 1, 64, 768, 768, 768, True, 1), ('grid', 1, 1024, 192, 192, 192, True, 1), ('grid', 1, 1024, 192, 576, 192, False, 1),
    ('grid', 1, 1024, 384, 384, 384, False, 0), ('grid', 1, 1024, 384, 384, 384, False, 1), ('grid', 1, 1024, 384, 384, 384, True, 1),
    ('grid', 1, 1024, 384, 768, 384, False, 1), ('grid', 1, 1024, 384, 960, 384, False, 1), ('grid', 1, 1024, 576, 576, 576, False, 1),
    ('grid', 1, 1024, 576, 576, 576, True, 1), ('grid', 1, 1024, 960, 960, 960, False, 1), ('grid', 1, 16384, 256, 256, 256, False, 1),
    ('grid', 1, 16384, 256, 256, 256, True, 1), ('grid', 1, 16384, 256, 512, 256, False, 1), ('grid', 1, 16384, 256, 768, 256, False, 1),
    ('grid', 1, 16384, 512, 512, 512, False, 1), ('grid', 1, 16384, 512, 512, 512, True, 1), ('grid', 1, 16384, 768, 768, 768, False, 1),
    ('grid', 1, 256, 1152, 1152, 1152, False, 1), ('grid', 1, 256, 1344, 1344, 1344, False, 1), ('grid', 1, 256, 384, 384, 384, True, 1),
    ('grid', 1, 256, 384, 960, 384, False, 1), ('grid', 1, 256, 576, 1152, 576, False, 1), ('grid', 1, 256, 576, 1344, 576, False, 1),
    ('grid', 1, 256, 576, 576, 576, False, 0), ('grid', 1, 256, 576, 576, 576, False, 1), ('grid', 1, 256, 576, 576, 576, True, 1),
    ('grid', 1, 256, 960, 960, 960, False, 1), ('grid', 1, 262144, 128, 128, 128, False, 1), ('grid', 1, 262144, 128, 128, 128, True, 1),
    ('grid', 1, 262144, 128, 256, 128, False, 1), ('grid', 1, 262144, 128, 384, 128, False, 1), ('grid', 1, 262144, 256, 256, 256, False, 1),
    ('grid', 1, 262144, 256, 256, 256, True, 1), ('grid', 1, 262144, 384, 384, 384, False, 1), ('grid', 1, 4096, 1024, 1024, 1024, False, 1),
    ('grid', 1, 4096, 192, 192, 192, False, 1), ('grid', 1, 4096, 192, 192, 192, True, 1), ('grid', 1, 4096, 192, 384, 192, False, 1),
    ('grid', 1, 4096, 192, 576, 192, False, 1), ('grid', 1, 4096, 384, 384, 384, False, 1), ('grid', 1, 4096, 384, 384, 384, True, 1),
    ('grid', 1, 4096, 576, 576, 576, False, 1), ('grid', 1, 4096, 768, 768, 768, False, 1), ('grid', 1, 64, 1344, 1344, 1344, False, 1),
    ('grid', 1, 64, 576, 1344, 576, False, 1), ('grid', 1, 64, 576, 576, 576, True, 1), ('grid', 1, 65536, 128, 128, 128, True, 1),
    ('grid', 1, 65536, 128, 384, 128, False, 1), ('grid', 1, 65536, 256, 256, 256, False, 1), ('grid', 1, 65536, 256, 256, 256, True, 1),
    ('grid', 1, 65536, 256, 512, 256, False, 1), ('grid', 1, 65536, 384, 384, 384, False, 1), ('grid', 1, 65536, 512, 512, 512, False, 1),
]
GN_BWD_PLAN = [
    ('cluster', 1, 1024, 1024, 1024, 1024, 1024, False, 1, 1), ('cluster', 1, 1024, 1024, 1024, 1024, 1024, True, 1, 0), ('cluster', 1, 1024, 1280, 1280, 1280, 1280, False, 1, 1),
    ('cluster', 1, 1024, 1536, 1536, 1536, 1536, False, 1, 1), ('cluster', 1, 1024, 256, 256, 256, 256, True, 1, 0), ('cluster', 1, 1024, 256, 256, 768, 256, False, 1, 1),
    ('cluster', 1, 1024, 512, 512, 1024, 512, False, 1, 1), ('cluster', 1, 1024, 512, 512, 1280, 512, False, 1, 1), ('cluster', 1, 1024, 512, 512, 1536, 512, False, 1, 1),
    ('cluster', 1, 1024, 512, 512, 512, 512, False, 0, 1), ('cluster', 1, 1024, 512, 512, 512, 512, False, 1, 1), ('cluster', 1, 1024, 512, 512, 512, 512, True, 1, 0),
    ('cluster', 1, 1024, 768, 768, 768, 768, False, 1, 1), ('cluster', 1, 1024, 768, 768, 768, 768, True, 1, 0), ('cluster', 1, 256, 1024, 1024, 1024, 1024, False, 0, 1),
    ('cluster', 1, 256, 1024, 1024, 1024, 1024, False, 1, 1), ('cluster', 1, 256, 1024, 1024, 1024, 1024, True, 1, 0), ('cluster', 1, 256, 1024, 1024, 2048, 1024, False, 1, 1),
    ('cluster', 1, 256, 1280, 1280, 1280, 1280, False, 1, 1), ('cluster', 1, 256, 1536, 1536, 1536, 1536, False, 1, 1), ('cluster', 1, 256, 1792, 1792, 1792, 1792, False, 1, 1),
    ('cluster', 1, 256, 2048, 2048, 2048, 2048, False, 1, 1), ('cluster', 1, 256, 512, 512, 1280, 512, False, 1, 1), ('cluster', 1, 256, 512, 512, 1536, 512, False, 1, 1),
    ('cluster', 1, 256, 512, 512, 512, 512, True, 1, 0), ('cluster', 1, 256, 768, 768, 1536, 768, False, 1, 1), ('cluster', 1, 256, 768, 768, 1792, 768, False, 1, 1),
    ('cluster', 1, 256, 768, 768, 768, 768, False, 0, 1), ('cluster', 1, 256, 768, 768, 768, 768, False, 1, 1), ('cluster', 1, 256, 768, 768, 768, 768, True, 1, 0),
    ('cluster', 1, 4096, 256, 256, 256, 256, False, 1, 1), ('cluster', 1, 4096, 256, 256, 256, 256, True, 1, 0), ('cluster', 1, 4096, 256, 256, 512, 256, False, 1, 1),
    ('cluster', 1, 4096, 256, 256, 768, 256, False, 1, 1), ('cluster', 1, 4096, 512, 512, 1024, 512, False, 1, 1), ('cluster', 1, 4096, 512, 512, 512, 512, False, 1, 1),
    ('cluster', 1, 4096, 512, 512, 512, 512, True, 1, 0), ('cluster', 1, 64, 1024, 1024, 1024, 1024, False, 0, 1), ('cluster', 1, 64, 1024, 1024, 1024, 1024, False, 1, 1),
    ('cluster', 1, 64, 1024, 1024, 1024, 1024, True, 1, 0), ('cluster', 1, 64, 1024, 1024, 2048, 1024, False, 1, 1), ('cluster', 1, 64, 1536, 1536, 1536, 1536, False, 1, 1),
    ('cluster', 1, 64, 1792, 1792, 1792, 1792, False, 1, 1), ('cluster', 1, 64, 2048, 2048, 2048, 2048, False, 1, 1), ('cluster', 1, 64, 768, 768, 1536, 768, False, 1, 1),
    ('cluster', 1, 64, 768, 768, 1792, 768, False, 1, 1), ('cluster', 1, 64, 768, 768, 768, 768, False, 0, 1), ('cluster', 1, 64, 768, 768, 768, 768, False, 1, 1),
    ('cluster', 1, 64, 768, 768, 768, 768, True, 1, 0), ('direct', 1, 16384, 512, 512, 512, 512, False, 1, 1), ('direct', 1, 16384, 512, 512, 512, 512, True, 1, 0),
    ('direct', 1, 16384, 768, 768, 768, 768, False, 1, 1), ('direct', 1, 262144, 256, 256, 256, 256, False, 1, 1), ('direct', 1, 262144, 256, 256, 256, 256, True, 1, 0),
    ('direct', 1, 65536, 256, 256, 256, 256, False, 1, 0), ('direct', 1, 65536, 256, 256, 256, 256, False, 1, 1), ('direct', 1, 65536, 256, 256, 256, 256, True, 1, 0),
    ('direct', 1, 65536, 256, 256, 512, 256, False, 1, 1), ('direct', 1, 65536, 512, 512, 512, 512, False, 1, 1), ('ring', 1, 1024, 192, 192, 192, 192, True, 1, 0),
    ('ring', 1, 1024, 192, 192, 576, 192, False, 1, 1), ('ring', 1, 1024, 384, 384, 384, 384, False, 0, 1), ('ring', 1, 1024, 384, 384, 384, 384, False, 1, 1),
    ('ring', 1, 1024, 384, 384, 384, 384, True, 1, 0), ('ring', 1, 1024, 384, 384, 768, 384, False, 1, 1), ('ring', 1, 1024, 384, 384, 960, 384, False, 1, 1),
    ('ring', 1, 1024, 576, 576, 576, 576, False, 1, 1), ('ring', 1, 1024, 576, 576, 576, 576, True, 1, 0), ('ring', 1, 1024, 960, 960, 960, 960, False, 1, 1),
    ('ring', 1, 16384, 256, 256, 256, 256, False, 1, 0), ('ring', 1, 16384, 256, 256, 256, 256, False, 1, 1), ('ring', 1, 16384, 256, 256, 256, 256, True, 1, 0),
    ('ring', 1, 16384, 256, 256, 512, 256, False, 1, 1), ('ring', 1, 16384, 256, 256, 768, 256, False, 1, 1), ('ring', 1, 256, 1152, 1152, 1152, 1152, False, 1, 1),
    ('ring', 1, 256, 1344, 1344, 1344, 1344, False, 1, 1), ('ring', 1, 256, 384, 384, 384, 384, True, 1, 0), ('ring', 1, 256, 384, 384, 960, 384, False, 1, 1),
    ('ring', 1, 256, 576, 576, 1152, 576, False, 1, 1), ('ring', 1, 256, 576, 576, 1344, 576, False, 1, 1), ('ring', 1, 256, 576, 576, 576, 576, False, 0, 1),
    ('ring', 1, 256, 576, 576, 576, 576, False, 1, 1), ('ring', 1, 256, 576, 576, 576, 576, True, 1, 0), ('ring', 1, 256, 960, 960, 960, 960, False, 1, 1),
    ('ring', 1, 262144, 128, 128, 128, 128, False, 1, 0), ('ring', 1, 262144, 128, 128, 128, 128, True, 1, 0), ('ring', 1, 262144, 128, 128, 256, 128, False, 1, 1),
    ('ring', 1, 262144, 128, 128, 384, 128, False, 1, 1), ('ring', 1, 262144, 384, 384, 384, 384, False, 1, 1), ('ring', 1, 4096, 1024, 1024, 1024, 1024, False, 1, 1),
    ('ring', 1, 4096, 192, 192, 192, 192, False, 1, 0), ('ring', 1, 4096, 192, 192, 192, 192, True, 1, 0), ('ring', 1, 4096, 192, 192, 384, 192, False, 1, 1),
    ('ring', 1, 4096, 192, 192, 576, 192, False, 1, 1), ('ring', 1, 4096, 384, 384, 384, 384, False, 1, 1), ('ring', 1, 4096, 384, 384, 384, 384, True, 1, 0),
    ('ring', 1, 4096, 576, 576, 576, 576, False, 1, 1), ('ring', 1, 4096, 768, 768, 768, 768, False, 1, 1), ('ring', 1, 64, 1344, 1344, 1344, 1344, False, 1, 1),
    ('ring', 1, 64, 576, 576, 1344, 576, False, 1, 1), ('ring', 1, 64, 576, 576, 576, 576, True, 1, 0), ('ring', 1, 65536, 128, 128, 128, 128, True, 1, 0),
    ('ring', 1, 65536, 128, 128, 384, 128, False, 1, 1), ('ring', 1, 65536, 384, 384, 384, 384, False, 1, 1),
]
ATTN_PLAN = [
    (1, 4, 64, 256, 3072, 1024, True, 0), (1, 4, 256, 192, 2304, 768, True, 0),
    (1, 4, 1024, 128, 1536, 512, True, 0), (1, 6, 1024, 64, 1152, 384, False, 0),
    (1, 8, 1024, 64, 1536, 512, True, 0), (1, 9, 256, 64, 1728, 576, False, 0),
    (1, 12, 64, 64, 2304, 768, False, 0), (1, 16, 64, 64, 3072, 1024, True, 0),
    (1, 16, 256, 64, 3072, 1024, True, 0), (16, 12, 50, 64, 2304, 768, False, 0),
    (16, 12, 197, 64, 2304, 768, False, 0), (64, 16, 257, 64, 3072, 1024, False, 0),
]
POOL2_PLAN = [
    (1, 128, 128, 256, 256, 256, 0.25), (1, 128, 128, 256, 256, 256, 1.0), (1, 128, 128, 256, 512, 256, 0.25),
    (1, 128, 128, 256, 512, 256, 1.0), (1, 128, 128, 256, 768, 256, 0.25), (1, 128, 128, 512, 512, 512, 1.0),
    (1, 128, 128, 512, 768, 512, 1.0), (1, 16, 16, 1024, 1024, 1024, 0.25), (1, 16, 16, 1024, 1024, 1024, 1.0),
    (1, 16, 16, 1024, 1792, 1024, 1.0), (1, 16, 16, 1024, 2048, 1024, 0.25), (1, 16, 16, 1024, 2048, 1024, 1.0),
    (1, 16, 16, 576, 1344, 576, 0.25), (1, 16, 16, 576, 576, 576, 0.25), (1, 16, 16, 768, 1344, 768, 1.0),
    (1, 16, 16, 768, 1792, 768, 0.25), (1, 16, 16, 768, 768, 768, 0.25), (1, 16, 16, 768, 768, 768, 1.0),
    (1, 256, 256, 256, 256, 256, 0.25), (1, 256, 256, 256, 256, 256, 1.0), (1, 256, 256, 256, 512, 256, 0.25),
    (1, 256, 256, 256, 512, 256, 1.0), (1, 32, 32, 1024, 1024, 1024, 1.0), (1, 32, 32, 1024, 1536, 1024, 1.0),
    (1, 32, 32, 384, 384, 384, 0.25), (1, 32, 32, 384, 960, 384, 0.25), (1, 32, 32, 512, 1280, 512, 0.25),
    (1, 32, 32, 512, 1536, 512, 0.25), (1, 32, 32, 512, 512, 512, 0.25), (1, 32, 32, 576, 576, 576, 1.0),
    (1, 32, 32, 576, 960, 576, 1.0), (1, 32, 32, 768, 1280, 768, 1.0), (1, 32, 32, 768, 768, 768, 1.0),
    (1, 512, 512, 128, 128, 128, 0.25), (1, 512, 512, 128, 384, 128, 0.25), (1, 512, 512, 256, 256, 256, 1.0),
    (1, 512, 512, 256, 384, 256, 1.0), (1, 64, 64, 192, 192, 192, 0.25), (1, 64, 64, 192, 576, 192, 0.25),
    (1, 64, 64, 256, 256, 256, 0.25), (1, 64, 64, 256, 768, 256, 0.25), (1, 64, 64, 384, 384, 384, 1.0),
    (1, 64, 64, 384, 576, 384, 1.0), (1, 64, 64, 512, 1024, 512, 0.25), (1, 64, 64, 512, 1024, 512, 1.0),
    (1, 64, 64, 512, 512, 512, 0.25), (1, 64, 64, 512, 512, 512, 1.0), (1, 64, 64, 512, 768, 512, 1.0),
]
UP2_PLAN = [
    (1, 128, 128, 256, 256, 256, 0.25), (1, 128, 128, 256, 256, 256, 1.0), (1, 16, 16, 1024, 1024, 1024, 1.0),
    (1, 16, 16, 384, 384, 384, 0.25), (1, 16, 16, 512, 512, 512, 0.25), (1, 16, 16, 576, 576, 576, 1.0),
    (1, 16, 16, 768, 768, 768, 1.0), (1, 256, 256, 128, 128, 128, 0.25), (1, 256, 256, 256, 256, 256, 1.0),
    (1, 32, 32, 192, 192, 192, 0.25), (1, 32, 32, 256, 256, 256, 0.25), (1, 32, 32, 384, 384, 384, 1.0),
    (1, 32, 32, 512, 512, 512, 0.25), (1, 32, 32, 512, 512, 512, 1.0), (1, 64, 64, 256, 256, 256, 0.25),
    (1, 64, 64, 256, 256, 256, 1.0), (1, 64, 64, 512, 512, 512, 1.0), (1, 8, 8, 1024, 1024, 1024, 0.25),
    (1, 8, 8, 1024, 1024, 1024, 1.0), (1, 8, 8, 576, 576, 576, 0.25), (1, 8, 8, 768, 768, 768, 0.25),
    (1, 8, 8, 768, 768, 768, 1.0),
]
ADD_PLAN = [
    (1024, 384, 768, 384, 384), (1024, 384, 960, 384, 384), (1024, 512, 1024, 512, 512), (1024, 512, 1280, 512, 512),
    (1024, 512, 1536, 512, 512), (16384, 256, 256, 256, 256), (16384, 256, 512, 256, 256), (16384, 256, 768, 256, 256),
    (256, 1024, 2048, 1024, 1024), (256, 576, 1152, 576, 576), (256, 576, 1344, 576, 576), (256, 768, 1536, 768, 768),
    (256, 768, 1792, 768, 768), (262144, 128, 256, 128, 128), (262144, 128, 384, 128, 128), (262144, 64, 64, 64, 64),
    (4096, 192, 384, 192, 192), (4096, 192, 576, 192, 192), (4096, 256, 512, 256, 256), (4096, 256, 768, 256, 256),
    (4096, 512, 1024, 512, 512), (4096, 512, 512, 512, 512), (64, 1024, 2048, 1024, 1024), (64, 768, 1536, 768, 768),
    (65536, 128, 128, 128, 128), (65536, 256, 512, 256, 256),
]
COPY_PLAN = [
    (1024, 192, 576, 192), (1024, 256, 768, 256), (1024, 384, 576, 384), (1024, 384, 768, 384),
    (1024, 512, 1024, 512), (1024, 512, 768, 512), (16448, 1024, 1024, 1024), (256, 1024, 1536, 1024),
    (256, 1024, 2048, 1024), (256, 384, 960, 384), (256, 512, 1280, 512), (256, 512, 1536, 512),
    (256, 576, 1152, 576), (256, 576, 960, 576), (256, 768, 1280, 768), (256, 768, 1536, 768),
    (3152, 768, 768, 768), (4096, 256, 768, 256), (64, 1024, 1792, 1024), (64, 1024, 2048, 1024),
    (64, 576, 1344, 576), (64, 768, 1344, 768), (64, 768, 1536, 768), (64, 768, 1792, 768),
    (65536, 128, 384, 128), (800, 768, 768, 768),
]
NCHW_TO_PM_PLAN = [
    (1, 3, 16384, 64, 0, 1.0), (1, 3, 262144, 64, 0, 1.0), (1, 3, 262144, 64, 4, 1.0, *LPIPS_SHIFT, *LPIPS_MUL),
    (1, 3, 4096, 64, 0, 1.0), (1, 3, 65536, 64, 0, 1.0),
]
PM_TO_NCHW_PLAN = [
    (1, 3, 262144, 64, 6, 0.0009765625, *LPIPS_MUL),
]


# ---------------------------------------------------------------------------------------------------------------- GroupNorm
def gn_bwd_grid_engine(HW, C):
    """the engine a GN_BWD_GRID launch runs on: norm_grid.cu's gn_bwd_direct -- the direct-load kernel of norm_grid2.cu where it supports
    the width (gn_grid2_supports: C % 256 == 0 and C <= 2048) and HW * C >= 2^23, the ring kernel otherwise"""
    return "direct" if C % 256 == 0 and C <= 2048 and HW * C >= 1 << 23 else "ring"


def gn_chain(engine, N, HW, C, maxv=16):
    """longest fp32 summation chain behind one group statistic: the serial per-thread sum over the pixels of its lane, then the
    in-CTA fold (PP * cpg / 16 = 8 terms in the ring kernels, fewer in the others), the shuffles and the fold of the CTAs' partials
    (compensated, or in float64): 64 covers the folds"""
    if engine == "cluster":
        cpg = C // 32
        gpc = 16 // cpg if cpg < 16 else 1
        lanes = max(1, gn_fused_cluster(N, HW, C, maxv)) * (512 // (gpc * cpg // 8))
    elif engine in ("grid", "ring", "direct"):
        lanes = max(1, gn_grid_ctas(N, HW, C)) * max(1, 512 // (C // 8))
    else:
        pp = max(1, 256 // (C // 8))
        lanes = int(min(max(1, -(-HW // (pp * 16))), max(1, 296 // N))) * pp
    return -(-HW // lanes) + 64


def emit_gn_fwd(plan, engine, N, HW, C, ldx, ldy, x, gamma, beta, emb, y, stats, silu, eps=1e-5):
    """the ops Plan.group_norm emits for `engine`, on explicit buffers"""
    embp = (emb, 0) if emb is not None else None
    if engine == "cluster":
        cs = gn_fused_cluster(N, HW, C, 16) or 1
        plan.emit("GN_FWD_FUSED", flags=silu, i=[N, HW, C, ldx, ldy, cs], f=[eps], p=[(x, 0), (gamma, 0), (beta, 0), embp, (y, 0), (stats, 0)])
    elif engine == "grid":
        G = gn_grid_ctas(N, HW, C) or 1
        part, bar = plan.new(N * G * 64, "f"), plan.new(2, "u32")
        plan.emit("GN_FWD_GRID", flags=silu, i=[N, HW, C, ldx, ldy, G], f=[eps],
                  p=[(x, 0), (gamma, 0), (beta, 0), embp, (y, 0), (stats, 0), (part, 0), (bar, 0)])
    else:
        pp = max(1, 256 // (C // 8))
        nchunk = int(min(max(1, -(-HW // (pp * 16))), max(1, 296 // N)))
        part, cnt = plan.new(N * nchunk * 64, "f"), plan.new(N, "u32")
        plan.emit("GN_STATS", i=[N, HW, C, ldx, nchunk], f=[eps], p=[(x, 0), (part, 0), (stats, 0), (cnt, 0)])
        plan.emit("GN_APPLY", flags=silu, i=[N, HW, C, ldx, nchunk, ldy], f=[eps], p=[(x, 0), (stats, 0), (gamma, 0), (beta, 0), embp, (y, 0)])


def emit_gn_bwd(plan, engine, N, HW, C, ld_dy, ldx, ld_dx, dy, x, stats, gamma, beta, emb, dx, silu, acc, eps=1e-5):
    common = [(dy, 0), (x, 0), (stats, 0), (gamma, 0), (beta, 0), (emb, 0) if emb is not None else None]
    fl = silu | (2 if acc else 0)
    if engine == "cluster":
        cs = gn_fused_cluster(N, HW, C, 8) or 1
        plan.emit("GN_BWD_FUSED", flags=fl, i=[N, HW, C, ld_dy, ldx, ld_dx, cs], f=[eps], p=common + [(dx, 0)])
    elif engine in ("ring", "direct"):
        G = gn_grid_ctas(N, HW, C) or 1
        part, bar, scratch = plan.new(N * G * 64, "f"), plan.new(2, "u32"), plan.new(N * HW * C, "h")
        plan.emit("GN_BWD_GRID", flags=fl, i=[N, HW, C, ld_dy, ldx, ld_dx, G], f=[eps], p=common + [(dx, 0), (part, 0), (bar, 0), (scratch, 0)])
    else:
        pp = max(1, 256 // (C // 8))
        nchunk = int(min(max(1, -(-HW // (pp * 16))), max(1, 296 // N)))
        part, sums, cnt = plan.new(N * nchunk * 64, "f"), plan.new(N * 64, "f"), plan.new(N, "u32")
        plan.emit("GN_BWD_STATS", flags=silu, i=[N, HW, C, ld_dy, ldx, nchunk], f=[eps], p=common + [(part, 0), (sums, 0), (cnt, 0)])
        plan.emit("GN_BWD_APPLY", flags=fl, i=[N, HW, C, ld_dy, ldx, nchunk, ld_dx], f=[eps], p=common + [(sums, 0), (dx, 0)])


def engine_runs(engine, N, HW, C, fwd):
    """would a plan with this engine forced run it at this shape (the selection rules of Plan.group_norm)?"""
    if engine == "cluster":
        return gn_fused_cluster(N, HW, C, 16 if fwd else 8) > 0
    if engine in ("grid", "ring", "direct"):
        return gn_grid_ctas(N, HW, C) > 0 and (fwd or gn_bwd_grid_engine(HW, C) == engine)
    return True


def gn_inputs(device, N, HW, C, seed, emb):
    """fp16 x [N, HW, C] whose groups have |mean| / std cycling through RATIOS (std itself log-normal), gamma, beta, emb"""
    d, g = dev_of(device), gen(dev_of(device), seed)
    std = th.exp(th.randn(N, 32, device=d, generator=g, dtype=D64) * 0.5)
    ratio = th.tensor(RATIOS, device=d, dtype=D64).repeat(-(-N * 32 // len(RATIOS)))[:N * 32].view(N, 32)
    sign = th.where(th.rand(N, 32, device=d, generator=g) < 0.5, -1.0, 1.0).to(D64)
    z = th.randn(N, HW, 32, C // 32, device=d, generator=g, dtype=D64)
    x = (z * std[:, None, :, None] + (sign * ratio * std)[:, None, :, None]).reshape(N, HW, C).half()
    gamma = (1 + 0.3 * th.randn(C, device=d, generator=g)).float()
    beta = (0.2 * th.randn(C, device=d, generator=g)).float()
    e = (0.3 * th.randn(N, 2 * C, device=d, generator=g)).float() if emb else None
    return x, gamma, beta, e


def gn_ref_stats(x, eps=1e-5):
    """float64 group mean, variance and rstd [N, 32] of fp16 x [N, HW, C]"""
    N, HW, C = x.shape
    xg = x.to(D64).view(N, HW, 32, C // 32)
    mean = xg.mean((1, 3))
    var = (xg - mean[:, None, :, None]).square().mean((1, 3))
    return mean, var, 1 / th.sqrt(var + eps)


def per_channel(t, C):
    """[N, 32] -> [N, 1, C]"""
    return t.repeat_interleave(C // 32, dim=1)[:, None, :]


def gn_affine(gamma, beta, emb, N, C):
    """per-channel scale G = gamma (1 + e0) and shift (beta (1 + e0) + e1) of the normalised value, float64 [N, 1, C]"""
    g, b = gamma.to(D64).view(1, 1, C), beta.to(D64).view(1, 1, C)
    if emb is None:
        return g.expand(N, 1, C), b.expand(N, 1, C)
    e = emb.to(D64).view(N, 1, 2 * C)
    return g * (1 + e[..., :C]), b * (1 + e[..., :C]) + e[..., C:]


GN_FWD_EXTRA = [  # batch 2-3 on the cluster and grid engines; the two-pass fallback engine
    ("cluster", 2, 1024, 512, 512, 512, True, 1), ("cluster", 3, 256, 768, 1536, 768, False, 0), ("grid", 2, 16384, 256, 512, 256, True, 1),
    ("grid", 3, 4096, 384, 384, 384, False, 0), ("twopass", 1, 65536, 256, 768, 256, True, 1), ("twopass", 2, 4096, 192, 576, 192, False, 0),
    ("twopass", 1, 1024, 1024, 1024, 1024, True, 1), ("twopass", 1, 262144, 128, 384, 128, False, 1),
]
GN_BWD_EXTRA = [
    ("cluster", 2, 1024, 512, 512, 512, 512, True, 1, 1), ("cluster", 3, 256, 768, 768, 1536, 768, False, 0, 0),
    ("ring", 2, 16384, 384, 384, 768, 384, True, 1, 0), ("direct", 2, 65536, 256, 256, 512, 256, False, 1, 1),
    ("ring", 3, 4096, 192, 192, 576, 192, False, 0, 1), ("twopass", 1, 65536, 256, 256, 768, 256, True, 1, 1),
    ("twopass", 2, 4096, 192, 192, 576, 192, False, 0, 0), ("twopass", 1, 262144, 128, 128, 384, 128, False, 1, 1),
]
GN_FWD_CPU = [("cluster", 1, 64, 64, 128, 64, True, 1), ("grid", 2, 48, 128, 128, 128, False, 0), ("twopass", 1, 40, 256, 384, 256, True, 1),
              ("grid", 1, 256, 64, 192, 64, False, 1)]
GN_BWD_CPU = [("cluster", 1, 64, 64, 64, 128, 64, True, 1, 1), ("ring", 2, 48, 128, 256, 128, 384, False, 0, 0),
              ("direct", 1, 40, 256, 256, 384, 256, True, 1, 0), ("twopass", 1, 256, 64, 64, 192, 64, False, 1, 1)]


def gn_id(s):
    return "-".join(str(int(v)) if isinstance(v, bool) else str(v) for v in s)


def gn_params(plan_table, extra, cpu):
    gpu = {gn_id(s): s for s in list(plan_table) + extra}
    return cases(gpu, {gn_id(s): s for s in cpu})


@pytest.mark.parametrize("device,case", gn_params(GN_FWD_PLAN, GN_FWD_EXTRA, GN_FWD_CPU))
def test_gn_fwd(device, case):
    """GroupNorm(32) (+SiLU, +scale-shift) forward: y and the (mean, rstd) statistics, over a strided x whose channels C..ldx are NaN and a
    NaN-filled y whose guard channels C..ldy hold a sentinel"""
    engine, N, HW, C, ldx, ldy, has_emb, silu = case
    # the engine forced must be the one the selection rules pick (the interpreter runs every engine's ops alike)
    assert device != "cuda" or engine_runs(engine, N, HW, C, True), f"{engine} does not run {case}"
    x, gamma, beta, emb = gn_inputs(device, N, HW, C, HW + C + N, has_emb)
    plan = Plan()
    bx, bg, bb, by, bst = (plan.new(N * HW * ldx, "h"), plan.new(C, "f"), plan.new(C, "f"), plan.new(N * HW * ldy, "h"),
                           plan.new(N * 64, "f"))
    be = plan.new(N * 2 * C, "f") if has_emb else None
    emit_gn_fwd(plan, engine, N, HW, C, ldx, ldy, bx, bg, bb, be, by, bst, silu)
    y0 = strided(th.full((N, HW, C), float("nan"), device=x.device), ldy, SENTINEL).half()
    inputs = [(bx, strided(x, ldx, float("nan"))), (bg, gamma), (bb, beta), (by, y0)] + ([(be, emb)] if has_emb else [])
    run(plan, device, inputs)
    rd = reader(plan, device)
    what = f"gn_fwd {engine} {case}"

    mean, var, rstd = gn_ref_stats(x)
    L = gn_chain(engine, N, HW, C)
    xg = x.to(D64).view(N, HW, 32, C // 32)
    piv = xg[:, 0, :, 0]  # the grid and two-pass kernels' pivot; the cluster kernel's exact two-pass is within the same bound
    # statistics: the mean is a length-L fp32 sum (of x - pivot in the pivoted engines) and one division; the variance a length-L sum
    # of squares of x - pivot less (mean - pivot)^2, so its error is L u (var + (mean - pivot)^2), halved by the square root, plus a
    # few u for the reciprocal square root and the divisions
    absx = xg.abs().mean((1, 3))
    e_mu = (L + 4) * U * (absx + piv.abs()) + U * mean.abs()
    e_rs = (L + 8) * U * rstd * (var + (mean - piv).square()) / (var + 1e-5) + 4 * U * rstd
    st = rd(bst, (N, 32, 2)).to(D64)
    check(f"{what} mean", st[..., 0], mean, e_mu)
    check(f"{what} rstd", st[..., 1], rstd, e_rs)

    G, B0 = gn_affine(gamma, beta, emb, N, C)
    xd = x.to(D64)
    xhat = (xd - per_channel(mean, C)) * per_channel(rstd, C)
    v = xhat * G + B0
    ref = F.silu(v) if silu else v
    # fp32 floor: v = x A + B with A = rstd G, B = shift - mean A: the statistics' errors times d v / d mean = -A and d v / d rstd =
    # (x - mean) G, and four roundings of |x A| + |B| + |v|.  SiLU's sigmoid is tanh.approx.f32 on the device (absolute error
    # <= 2^-12 in the sigmoid: 2^-12 |v| in silu), and silu' <= 1.1.
    A = per_channel(rstd, C) * G
    Bc = B0 - per_channel(mean, C) * A
    e_v = A.abs() * per_channel(e_mu, C) + (xd - per_channel(mean, C)).abs() * G.abs() * per_channel(e_rs, C) + \
        4 * U * ((xd * A).abs() + Bc.abs() + v.abs())
    floor = (1.1 * e_v + (2.0 ** -12 * v.abs() if device == "cuda" else 4 * U * v.abs())) if silu else e_v
    got = rd(by, (N, HW, ldy))
    check16(what, got[..., :C], ref, floor + 2.0 ** -24)
    if ldy > C:
        assert bool((got[..., C:] == SENTINEL).all()), f"{what}: guard channels of y written"
    if engine != "cluster":
        reruns_identical(plan, device, what, inputs, [by, bst])


def gn_dy(x, mean, rstd, seed):
    """dy = a + b xhat + noise per (image, group): both reduction terms of the backward are many ulps of dx"""
    N, HW, C = x.shape
    g = gen(x.device, seed)
    a = th.randn(N, 32, device=x.device, generator=g, dtype=D64)
    b = th.randn(N, 32, device=x.device, generator=g, dtype=D64)
    xhat = (x.to(D64) - per_channel(mean, C)) * per_channel(rstd, C)
    return (per_channel(a, C) + per_channel(b, C) * xhat + 0.5 * th.randn(N, HW, C, device=x.device, generator=g, dtype=D64)).half()


@pytest.mark.parametrize("device,case", gn_params(GN_BWD_PLAN, GN_BWD_EXTRA, GN_BWD_CPU))
def test_gn_bwd(device, case):
    """GroupNorm(32) (+SiLU, +scale-shift) input gradient, storing (over NaN) and accumulating (flags 2), strided dy / x / dx with NaN
    in the input guard channels and a sentinel in the output's, from float64 statistics rounded to fp32 (the op's input)"""
    engine, N, HW, C, ld_dy, ldx, ld_dx, has_emb, silu, acc = case
    # the engine forced must be the one the selection rules pick (the interpreter runs every engine's ops alike)
    assert device != "cuda" or engine_runs(engine, N, HW, C, False), f"{engine} does not run {case}"
    x, gamma, beta, emb = gn_inputs(device, N, HW, C, HW + C + N + 1, has_emb)
    mean, var, _ = gn_ref_stats(x)
    stats = th.stack([mean, 1 / th.sqrt(var + 1e-5)], -1).float()
    mean, rstd = stats[..., 0].to(D64), stats[..., 1].to(D64)  # the op's statistics
    dy = gn_dy(x, mean, rstd, HW + C + 7)
    old = th.randn(N, HW, C, device=x.device, generator=gen(x.device, 11)).half()
    plan = Plan()
    bdy, bx, bst, bg, bb = (plan.new(N * HW * ld_dy, "h"), plan.new(N * HW * ldx, "h"), plan.new(N * 64, "f"), plan.new(C, "f"),
                            plan.new(C, "f"))
    bdx = plan.new(N * HW * ld_dx, "h")
    be = plan.new(N * 2 * C, "f") if has_emb else None
    emit_gn_bwd(plan, engine, N, HW, C, ld_dy, ldx, ld_dx, bdy, bx, bst, bg, bb, be, bdx, silu, acc)
    dx0 = strided(old if acc else th.full((N, HW, C), float("nan"), device=x.device).half(), ld_dx, SENTINEL).half()
    inputs = [(bdy, strided(dy, ld_dy, float("nan"))), (bx, strided(x, ldx, float("nan"))), (bst, stats), (bg, gamma), (bb, beta),
              (bdx, dx0)] + ([(be, emb)] if has_emb else [])
    run(plan, device, inputs)
    rd = reader(plan, device)
    what = f"gn_bwd {engine} {case}"

    # float64: dx = rstd (dxhat - mean(dxhat) - xhat mean(dxhat xhat)), dxhat = dy silu'(v) G
    G, B0 = gn_affine(gamma, beta, emb, N, C)
    mc, rc = per_channel(mean, C), per_channel(rstd, C)
    xd = x.to(D64)
    xhat = (xd - mc) * rc
    v = xhat * G + B0
    dyd = dy.to(D64)
    if silu:
        s = th.sigmoid(v)
        dsilu = s * (1 + v * (1 - s))
    else:
        dsilu = th.ones_like(v)
    dxh = dyd * dsilu * G
    grp = lambda t: t.view(N, HW, 32, C // 32).mean((1, 3))  # noqa: E731
    m1, m2 = grp(dxh), grp(dxh * xhat)
    t1, t2 = rc * per_channel(m1, C), rc * xhat * per_channel(m2, C)
    ref = rc * dxh - t1 - t2
    if acc:
        ref = ref + old.to(D64)
    # fp32 floor.  dxhat: silu' from tanh.approx.f32 on the device (2^-12 (1 + |v|) absolute) and 4 roundings; the ring kernel stores
    # dxhat in an fp16 scratch and both its statistics and its apply pass read that back (2^-11 |dxhat|).  The two means are length-L
    # sums (L u of the mean of the magnitude) of the per-element errors; xhat is good to 4 u plus u |x| rstd.  The result takes four
    # more roundings of rstd (|dxhat| + |m1| + |xhat m2|), and accumulating one fp32 add of |old|.
    L = gn_chain(engine, N, HW, C, 8)
    e_dxh = (dyd * G).abs() * ((2.0 ** -12 * (1 + v.abs())) if silu and device == "cuda" else 4 * U * dsilu.abs()) + 4 * U * dxh.abs()
    if engine == "ring":
        e_dxh = e_dxh + 2.0 ** -11 * dxh.abs()
    e_xh = 4 * U * xhat.abs() + U * xd.abs() * rc
    e_m1 = L * U * grp(dxh.abs()) + grp(e_dxh)
    e_m2 = L * U * grp((dxh * xhat).abs()) + grp(e_dxh * xhat.abs() + dxh.abs() * e_xh)
    floor = rc * (e_dxh + per_channel(e_m1, C) + xhat.abs() * per_channel(e_m2, C) + e_xh * per_channel(m2, C).abs()) + \
        4 * U * rc * (dxh.abs() + per_channel(m1, C).abs() + (xhat * per_channel(m2, C)).abs()) + (2 * U * old.to(D64).abs() if acc else 0)
    got = rd(bdx, (N, HW, ld_dx))
    check16(what, got[..., :C], ref, floor + 2.0 ** -24)
    # the inputs keep the check sensitive: both reduction terms are >= 50 fp16 ulps of dx somewhere (a kernel dropping either fails)
    u16 = ulp16(ref)
    for name, t in (("mean(dxhat)", t1), ("xhat mean(dxhat xhat)", t2)):
        assert float((t.abs() / (u16 + floor)).max()) >= 50, f"{what}: the {name} term is below 50 ulps of dx everywhere"
    if ld_dx > C:
        assert bool((got[..., C:] == SENTINEL).all()), f"{what}: guard channels of dx written"
    if engine != "cluster":
        reruns_identical(plan, device, what, inputs, [bdx])


# ---------------------------------------------------------------------------------------------------------------- attention
ATTN_EXTRA = [  # the towers the five plans above do not build: ViT-L/14@336px, and the text tower's causal forward
    (8, 16, 577, 64, 3072, 1024, False, 0), (1, 8, 77, 64, 1536, 512, False, 1),
] + [(*s[:6], not s[6], s[7]) for s in ATTN_PLAN if s[0] == 1]  # every UNet (heads, T, d) in the other qkv order as well
ATTN_CPU = [(1, 3, 70, 64, 576, 192, True, 0), (2, 2, 50, 64, 384, 128, False, 0), (1, 2, 67, 128, 768, 256, False, 0)]  # the interpreter has no causal mask


def attn_inputs(device, B, heads, T, d, seed):
    """q, k, v, dO [B, heads, T, d] (fp16).  Query rows cycle through five kinds: 0 plain (logits ~0.5), 1 a logit >= 20 above the rest
    at the last key (in the last, ragged key tile), 2 the same at key 0 (the first tile), 3 all logits equal (q = 0), 4 logits up to
    about +-60.  Keys 0 and T - 1 are the +-1 vectors w0, w1 the peaked rows point at."""
    d_, g = dev_of(device), gen(dev_of(device), seed)
    rn = lambda *s: th.randn(*s, device=d_, generator=g, dtype=D64)  # noqa: E731
    w = th.where(th.rand(B, heads, 1, d, device=d_, generator=g) < 0.5, -1.0, 1.0).to(D64)
    w = th.stack([w * th.where(th.arange(d, device=d_) < d // 2, 1.0, -1.0).to(D64), w])  # w0 . w1 = 0: a peaked row ignores the other peak key
    k = 0.5 * rn(B, heads, T, d)
    k[:, :, T - 1:] = w[1]
    k[:, :, :1] = w[0]
    gam = 30.0 / math.sqrt(d)  # scale * gam * d = 30 at the peak key; the others ~ gam * 0.5 ~ 2 (d = 64)
    kind = th.arange(T, device=d_) % 5
    q = rn(B, heads, T, d)
    q = th.where((kind == 1).view(1, 1, T, 1), gam * w[1] + 0.3 * q, q)
    q = th.where((kind == 2).view(1, 1, T, 1), gam * w[0] + 0.3 * q, q)
    q = th.where((kind == 3).view(1, 1, T, 1), th.zeros_like(q), q)
    q = th.where((kind == 4).view(1, 1, T, 1), 30.0 * q, q)
    return q.half(), k.half(), rn(B, heads, T, d).half(), rn(B, heads, T, d).half(), kind


def qkv_pack(q, k, v, qrs, legacy):
    """[B, heads, T, d] x 3 -> the fused qkv rows [B * T, qrs]: per-head [q|k|v] (legacy) or [q heads | k heads | v heads]"""
    B, H, T, d = q.shape
    t = th.stack([q, k, v], 2 if legacy else 1)  # legacy: [B, H, 3, T, d]; new: [B, 3, H, T, d]
    rows = t.permute(0, 3, 1, 2, 4).reshape(B * T, 3 * H * d)  # [B, T, ...]: the stack axis above already encodes the order
    return strided(rows, qrs, float("nan"))


def qkv_unpack(rows, B, H, T, d, legacy):
    t = rows[:, :3 * H * d].reshape(B, T, *((H, 3) if legacy else (3, H)), d)
    t = t.permute(0, 2, 3, 1, 4) if legacy else t.permute(0, 3, 2, 1, 4)  # [B, H, 3, T, d] either way
    return t[:, :, 0], t[:, :, 1], t[:, :, 2]


def heads_pack(o, ors):
    B, H, T, d = o.shape
    return strided(o.permute(0, 2, 1, 3).reshape(B * T, H * d), ors, float("nan"))


def heads_unpack(rows, B, H, T, d):
    return rows[:, :H * d].reshape(B, T, H, d).permute(0, 2, 1, 3)


def emit_attn(plan, B, heads, T, d, qrs, ors, legacy, bq, bo, blse, scale, causal=False, bwd=None):
    C = heads * d
    hs, qo, ko, vo = (3 * d, 0, d, 2 * d) if legacy else (d, 0, C, 2 * C)
    ii = [B, heads, T, d, T * qrs, qrs, hs, T * ors, ors, d]
    if bwd is None:
        plan.emit("ATTN_FWD", flags=causal, i=ii, f=[scale], p=[(bq, qo), (bq, ko), (bq, vo), (bo, 0), (blse, 0)])
    else:
        bdo, bdq, bdelta = bwd
        plan.emit("ATTN_BWD", i=ii, f=[scale], p=[(bq, qo), (bq, ko), (bq, vo), (bo, 0), (bdo, 0), (blse, 0), (bdq, qo), (bdq, ko), (bdq, vo),
                                                  (bdelta, 0)])


def attn_id(s):
    return "-".join(str(int(v)) if isinstance(v, bool) else str(v) for v in s)


@pytest.mark.parametrize("device,case", cases({attn_id(s): s for s in ATTN_PLAN + ATTN_EXTRA}, {attn_id(s): s for s in ATTN_CPU}))
def test_attention(device, case):
    """ATTN_FWD (out, lse) and ATTN_BWD (dq, dk, dv) against float64, the backward from float64 out / lse rounded to the op's fp16 / fp32
    (a stand-alone op).  lse is stored per (batch, head, query) in fp32 as the natural log of sum_j exp(scale q.k_j): natural-log units of
    the scaled logits."""
    B, heads, T, d, qrs, ors, legacy, causal = case
    q, k, v, do, kind = attn_inputs(device, B, heads, T, d, T * 7 + d + B)
    scale = float(th.tensor(1.0 / math.sqrt(d), dtype=th.float32))
    plan = Plan()
    n = B * T
    bq, bo, blse = plan.new(n * qrs, "h"), plan.new(n * ors, "h"), plan.new(B * heads * T, "f")
    emit_attn(plan, B, heads, T, d, qrs, ors, legacy, bq, bo, blse, scale, causal)
    inputs = [(bq, qkv_pack(q, k, v, qrs, legacy)), (bo, th.full((n * ors,), float("nan"), device=q.device).half()),
              (blse, th.full((B * heads * T,), float("nan"), device=q.device))]
    q64, k64, v64, do64 = (t.to(D64) for t in (q, k, v, do))
    S = q64 @ k64.transpose(-1, -2) * scale
    if causal:
        S = S.masked_fill(th.ones(T, T, dtype=th.bool, device=S.device).triu(1), -math.inf)
    lse = th.logsumexp(S, -1)
    P = th.exp(S - lse[..., None])
    out = P @ v64
    if not causal:
        peaked = S[:, :, kind == 1]
        assert bool((peaked[..., -1] - peaked[..., :-1].amax(-1) >= 20).all()), "the peaked rows are not peaked"
        bo2, blse2, bdo, bdq, bdelta = (plan.new(n * ors, "h"), plan.new(B * heads * T, "f"), plan.new(n * ors, "h"), plan.new(n * qrs, "h"),
                                        plan.new(B * heads * T, "f"))
        emit_attn(plan, B, heads, T, d, qrs, ors, legacy, bq, bo2, blse2, scale, bwd=(bdo, bdq, bdelta))
        o16, lse32 = out.half(), lse.float()
        inputs += [(bo2, heads_pack(o16, ors)), (blse2, lse32), (bdo, heads_pack(do, ors)),
                   (bdq, th.full((n * qrs,), float("nan"), device=q.device).half())]
    run(plan, device, inputs)
    rd = reader(plan, device)
    what = f"attention {case}"

    # forward.  The scaled logits are fp32 MMA sums of d products: E_S = (d + 2) u scale |q|.|k|.  p = exp(S - running max) by ex2.approx
    # (2^-21 relative) of an argument good to E_S + E_S(max) + 4 u (|S| + |max|); P is rounded to fp16 for the P V MMA (2^-11 relative,
    # 2^-25 absolute below 2^-14), the row sum l stays fp32 ((T + 16) u).  Output: ulp16 + sum_j P_ij (2^-11 + 2 eps_ij) |v_j| +
    # 2^-25 sum |v| + |out| ((T + 16) u + max eps).
    qa, ka = q64.abs(), k64.abs()
    E_S = (d + 2) * U * scale * (qa @ ka.transpose(-1, -2))
    m = S.amax(-1, keepdim=True)
    Sf = th.where(th.isfinite(S), S, th.zeros_like(S))
    eps = 2.0 ** -21 + E_S + E_S.amax(-1, keepdim=True) + 4 * U * (Sf.abs() + m.abs())
    va = v64.abs()
    tol_out = (P * (2.0 ** -11 + 2 * eps)) @ va + 2.0 ** -25 * va.sum(-2, keepdim=True) + \
        out.abs() * ((T + 16) * U + (P * eps).sum(-1, keepdim=True) + 2.0 ** -21)
    check16(f"{what} out", heads_unpack(rd(bo, (n, ors)), B, heads, T, d), out, tol_out)
    assert bool(rd(bo, (n, ors))[:, heads * d:].isnan().all()), f"{what}: out guard channels written"
    # lse = max + __logf(l): l good to (T + 16) u + sum_j P eps, __logf to 2^-21 absolute (+ 3 ulps), one add
    tol_lse = (P * eps).sum(-1) + (T + 16) * U + 2.0 ** -21 + 8 * U * (lse.abs() + m[..., 0].abs())
    check(f"{what} lse", rd(blse, (B, heads, T)), lse, tol_lse)
    if causal:
        return

    # backward, from o16 / lse32: P = exp(S - lse) recomputed in fp32 (relative eps_P: E_S, 4 u (|S| + |lse|), ex2.approx; the
    # one-tile kernel renormalises its own softmax: + (T + 16) u); dP = dO V^T: (d + 2) u |dO| |V|^T; delta = rowsum(dO O): d u
    # sum |dO| |O|, plus -- the one-tile kernel takes rowsum(P dP) -- the fp16 rounding of O, sum |dO| ulp16(O), and P's and dP's errors.
    # dS = P (dP - delta) scale is rounded to fp16 (2^-11, 2^-25 below 2^-14) for dQ = dS K and dK = dS^T Q, P to fp16 for dV = P^T dO;
    # those MMAs accumulate T fp32 products ((T + 2) u of the magnitude).
    Pk = th.exp(S - lse32.to(D64)[..., None])
    dP = do64 @ v64.transpose(-1, -2)
    delta = (do64 * o16.to(D64)).sum(-1, keepdim=True)
    dS = Pk * (dP - delta) * scale
    dq, dk, dv = dS @ k64, dS.transpose(-1, -2) @ q64, Pk.transpose(-1, -2) @ do64
    doa = do64.abs()
    eP = 2.0 ** -21 + E_S + 4 * U * (S.abs() + lse32.to(D64).abs()[..., None]) + (T + 16) * U
    eDP = (d + 2) * U * (doa @ va.transpose(-1, -2))
    dPa = dP.abs()
    eDelta = (d + 2) * U * (doa * o16.to(D64).abs()).sum(-1, keepdim=True) + (doa * ulp16(o16.to(D64))).sum(-1, keepdim=True) + \
        (Pk * (eP * dPa + eDP)).sum(-1, keepdim=True) + (T + 16) * U * (Pk * dPa).sum(-1, keepdim=True)
    e_dS = scale * Pk * (eP * (dP - delta).abs() + eDP + eDelta + 3 * U * (dP - delta).abs())
    e_dS16 = e_dS + 2.0 ** -11 * dS.abs() + 2.0 ** -25
    dSa = dS.abs()
    tol_dq = e_dS16 @ ka + (T + 2) * U * (dSa @ ka)
    tol_dk = e_dS16.transpose(-1, -2) @ qa + (T + 2) * U * (dSa.transpose(-1, -2) @ qa)
    tol_dv = (Pk * (eP + 2.0 ** -11) + 2.0 ** -25).transpose(-1, -2) @ doa + (T + 2) * U * (Pk.transpose(-1, -2) @ doa)
    gq, gk, gv = qkv_unpack(rd(bdq, (n, qrs)), B, heads, T, d, legacy)
    check16(f"{what} dq", gq, dq, tol_dq)
    check16(f"{what} dk", gk, dk, tol_dk)
    check16(f"{what} dv", gv, dv, tol_dv)


# ---------------------------------------------------------------------------------------------------------------- glue
def glue_id(name, s):
    return name + "-" + "-".join(str(v) for v in s)


def glue_values(shape, device, seed):
    """fp16 values with |x| in [2^-6, ~5]: two of them add exactly in fp32 (exponents at most 13 apart), four nearly so"""
    g = gen(dev_of(device), seed)
    t = th.randn(*shape, device=dev_of(device), generator=g)
    return (th.sign(t) * (t.abs() + 2.0 ** -6)).half()


POOL2_CPU = [(1, 8, 8, 16, 48, 16, 0.25), (2, 6, 4, 8, 8, 8, 1.0)]
UP2_CPU = [(1, 4, 4, 16, 16, 16, 1.0), (2, 3, 2, 8, 24, 8, 0.25)]
ADD_CPU = [(40, 16, 48, 16, 16), (12, 8, 8, 24, 8)]
COPY_CPU = [(40, 16, 48, 16), (12, 8, 8, 24)]
NCHW_TO_PM_CPU = [(1, 3, 64, 8, 0, 1.0), (2, 3, 20, 16, 4, 0.5, *LPIPS_SHIFT, *LPIPS_MUL)]
PM_TO_NCHW_CPU = [(1, 3, 64, 8, 6, 2.0 ** -10, *LPIPS_MUL), (2, 3, 20, 16, 3, 0.5), (1, 3, 10, 8, 0, 1.0), (1, 3, 10, 8, 5, 1.0, 0.5, 3.0, -2.0)]
# both source dtypes, storing and accumulating, with and without the multiplier, at the plans' shape
PM_TO_NCHW_EXTRA = [(1, 3, 262144, 64, fl, 2.0 ** -10) for fl in (0, 1, 3)] + [(1, 3, 262144, 64, 5, 2.0 ** -10, *LPIPS_MUL)]


@pytest.mark.parametrize("device,case", cases({glue_id("POOL2", s): ("POOL2", s) for s in POOL2_PLAN} | {glue_id("UP2", s): ("UP2", s) for s in UP2_PLAN},
                                              {glue_id("POOL2", s): ("POOL2", s) for s in POOL2_CPU} | {glue_id("UP2", s): ("UP2", s) for s in UP2_CPU}))
def test_pool2_up2(device, case):
    """POOL2 y = scale (sum of the 2x2 block) (Downsample, and the adjoint of Upsample) and UP2 y = scale x repeated 2x2 (Upsample, and the
    adjoint of Downsample) on channel slices: input guard channels NaN, output guard channels a sentinel"""
    name, (N, H, W, C, ldx, ldy, scale) = case
    Ho, Wo = (H // 2, W // 2) if name == "POOL2" else (2 * H, 2 * W)
    x = glue_values((N, H, W, C), device, H * C + ldx)
    plan = Plan()
    bx, by = plan.new(N * H * W * ldx, "h"), plan.new(N * Ho * Wo * ldy, "h")
    plan.emit(name, i=[N, H, W, C, ldx, ldy], f=[scale], p=[(bx, 0), (by, 0)])
    y0 = strided(th.full((N, Ho, Wo, C), float("nan"), device=x.device), ldy, SENTINEL).half()
    run(plan, device, [(bx, strided(x, ldx, float("nan"))), (by, y0)])
    got = reader(plan, device)(by, (N, Ho, Wo, ldy))
    x64 = x.to(D64)
    if name == "POOL2":
        ref = (x64[:, 0::2, 0::2] + x64[:, 0::2, 1::2] + x64[:, 1::2, 0::2] + x64[:, 1::2, 1::2]) * scale
        # three fp32 adds (3 u of the magnitude) and a power-of-two scale, then the fp16 rounding: within one ulp
        mag = (x64[:, 0::2, 0::2].abs() + x64[:, 0::2, 1::2].abs() + x64[:, 1::2, 0::2].abs() + x64[:, 1::2, 1::2].abs()) * scale
        check(f"{name} {case}", got[..., :C], ref, ulp16(ref) + 3 * U * mag)
    else:
        # scale * x is exact in fp32 (scale a power of two): bitwise the float64 value rounded to fp16
        ref = (x64 * scale).repeat_interleave(2, 1).repeat_interleave(2, 2).half()
        assert th.equal(got[..., :C], ref), f"{name} {case}: not bitwise round(scale x)"
    if ldy > C:
        assert bool((got[..., C:] == SENTINEL).all()), f"{name} {case}: guard channels written"


@pytest.mark.parametrize("device,case", cases({glue_id("ADD", s): ("ADD", s) for s in ADD_PLAN} | {glue_id("COPY", s): ("COPY", s) for s in COPY_PLAN},
                                              {glue_id("ADD", s): ("ADD", s) for s in ADD_CPU} | {glue_id("COPY", s): ("COPY", s) for s in COPY_CPU}))
def test_add_copy(device, case):
    """ADD c = a + b (gradient sums, one of them a concatenation's half) and COPY (concatenation, gathers) with their own leading dimensions:
    bitwise the float64 result rounded to fp16 (the fp32 sum of two such fp16 values is exact); NaN in the input guard channels, a
    sentinel in the output's"""
    name, s = case
    rows, C = s[:2]
    lds = s[2:]
    a = glue_values((rows, C), device, rows + C)
    b = glue_values((rows, C), device, rows + C + 1)
    plan = Plan()
    bufs = [plan.new(rows * ld, "h") for ld in lds]
    plan.emit(name, i=list(s), p=[(bf, 0) for bf in bufs])
    srcs = [a, b] if name == "ADD" else [a]
    out0 = strided(th.full((rows, C), float("nan"), device=a.device), lds[-1], SENTINEL).half()
    run(plan, device, [(bf, strided(t, ld, float("nan"))) for bf, t, ld in zip(bufs, srcs, lds)] + [(bufs[-1], out0)])
    got = reader(plan, device)(bufs[-1], (rows, lds[-1]))
    ref = (a.to(D64) + b.to(D64)).half() if name == "ADD" else a
    assert th.equal(got[:, :C], ref), f"{name} {s}: {int((got[:, :C] != ref).sum())} elements differ from the float64 result rounded to fp16"
    if lds[-1] > C:
        assert bool((got[:, C:] == SENTINEL).all()), f"{name} {s}: guard channels written"


@pytest.mark.parametrize("device,case", cases({glue_id("N2P", s): s for s in NCHW_TO_PM_PLAN}, {glue_id("N2P", s): s for s in NCHW_TO_PM_CPU}))
def test_nchw_to_pm(device, case):
    """fp32 NCHW -> fp16 pixel-major [N * HW, ld] (x scale, flags 4: (x - shift_c) * mul_c first): channels C..ld zero-filled over a NaN
    buffer; within one fp16 ulp (the fp32 affine is 3 roundings of the magnitude)"""
    N, C, HW, ld, flags, scale, *aff = case
    g = gen(dev_of(device), HW + ld)
    x = th.randn(N, C, HW, device=dev_of(device), generator=g) * 1.5
    f = [scale, *aff]
    plan = Plan()
    bx, by = plan.new(N * C * HW, "f"), plan.new(N * HW * ld, "h")
    plan.emit("NCHW_TO_PM", flags=flags, i=[N, C, HW, ld], f=f, p=[(bx, 0), (by, 0)])
    run(plan, device, [(bx, x), (by, th.full((N * HW * ld,), float("nan"), device=x.device))])
    got = reader(plan, device)(by, (N, HW, ld))
    x64 = x.to(D64)
    if flags & 4:
        sh = th.tensor(aff[:3], dtype=th.float32, device=x.device).to(D64).view(1, 3, 1)  # the kernel's fp32 operands
        mu = th.tensor(aff[3:], dtype=th.float32, device=x.device).to(D64).view(1, 3, 1)
        ref, mag = (x64 - sh) * mu * scale, (x64.abs() + sh.abs()) * mu.abs() * abs(scale)
    else:
        ref, mag = x64 * scale, x64.abs() * abs(scale)
    check(f"nchw_to_pm {case}", got[..., :C], ref.permute(0, 2, 1), ulp16(ref.permute(0, 2, 1)) + 3 * U * mag.permute(0, 2, 1))
    assert bool((got[..., C:] == 0).all()), f"nchw_to_pm {case}: channels C..ld not zero-filled"


@pytest.mark.parametrize("device,case", cases({glue_id("P2N", s): s for s in PM_TO_NCHW_PLAN + PM_TO_NCHW_EXTRA},
                                              {glue_id("P2N", s): s for s in PM_TO_NCHW_CPU}))
def test_pm_to_nchw(device, case):
    """pixel-major [N * HW, ld] (fp16, flags 1: fp32) -> fp32 NCHW x scale (flags 4: x mul_c too), flags 2 accumulating; the guard
    channels of the source are NaN.  A product by a power of two (exact), one by the multiplier (u of the product) and one fp32 add (u of
    the result)"""
    N, C, HW, ld, flags, scale, *mul = case
    g = gen(dev_of(device), HW + ld + flags)
    src = th.randn(N, HW, C, device=dev_of(device), generator=g) * 3
    src = src if flags & 1 else src.half()
    old = th.randn(N, C, HW, device=src.device, generator=g)
    plan = Plan()
    bs, bd = plan.new(N * HW * ld, "f" if flags & 1 else "h"), plan.new(N * C * HW, "f")
    plan.emit("PM_TO_NCHW", flags=flags, i=[N, C, HW, ld], f=[scale, *mul], p=[(bs, 0), (bd, 0)])
    run(plan, device, [(bs, strided(src, ld, float("nan"))), (bd, old if flags & 2 else th.full_like(old, float("nan")))])
    got = reader(plan, device)(bd, (N, C, HW))
    m = th.tensor(mul, dtype=th.float32, device=src.device).to(D64).view(1, C, 1) if flags & 4 else 1.0
    v = src.to(D64).permute(0, 2, 1) * scale * m
    ref = v + (old.to(D64) if flags & 2 else 0)
    check(f"pm_to_nchw {case}", got, ref, U * (v.abs() + ref.abs()))


# ---------------------------------------------------------------------------------------------------------------- coverage
def covered_signatures() -> set:
    """the op signatures (in tests/test_unet_kernel_coverage_cpu.py's form) the GPU cases above run"""
    out = {("GN_FWD", *s) for s in GN_FWD_PLAN + GN_FWD_EXTRA} | {("GN_BWD", *s) for s in GN_BWD_PLAN + GN_BWD_EXTRA}
    for s in ATTN_PLAN + ATTN_EXTRA:
        out.add(("ATTN_FWD", *s))
        if not s[-1]:
            out.add(("ATTN_BWD", *s))
    out |= {("POOL2", *s) for s in POOL2_PLAN} | {("UP2", *s) for s in UP2_PLAN} | {("ADD", *s) for s in ADD_PLAN}
    out |= {("COPY", *s) for s in COPY_PLAN} | {("NCHW_TO_PM", *s) for s in NCHW_TO_PM_PLAN}
    out |= {("PM_TO_NCHW", *s) for s in PM_TO_NCHW_PLAN + PM_TO_NCHW_EXTRA}
    return out
