"""TEST-ONLY interpreters of the autograd-bridge ops (include/cgd_b200.h CGD_OP_GRAD_SEED / GRAD_UNSCALE / PMV_BWD) on top of
tests/plan_interp.py: fp32 math, one fp16 rounding where the kernels store fp16, the kernels' NaN / inf rules."""
from __future__ import annotations

import torch as th

from clip_guided_diffusion_b200._lib import SC
from tests.plan_interp import Interp


def seed_scale(m: th.Tensor) -> th.Tensor:
    """SEED_QUANT's per-image power of two for maxima `m` (fp32): 2^clamp(floor(log2(4096 / m)), -60, 60), 1 where m == 0"""
    return th.where(m > 0, th.exp2(th.floor(th.log2(4096.0 / m.clamp(min=1e-38))).clamp(-60, 60)), th.ones_like(m))


def image_max(d_out: th.Tensor) -> th.Tensor:
    """per-image max |.| of [B, ...] as GRAD_SEED takes it: NaN dropped, inf saturated at 3e38"""
    a = d_out.abs().reshape(d_out.shape[0], -1)
    return th.where(th.isnan(a), th.zeros_like(a), a).amax(1).clamp(max=3.0e38)


def quantize(v: th.Tensor, scale) -> th.Tensor:
    """fp16(clamp(v * scale, +-60000)) with the kernels' fminf / fmaxf: a NaN becomes -60000"""
    return th.nan_to_num(v * scale, nan=-60000.0).clamp(-60000, 60000).half()


class AgInterp(Interp):
    def op_GRAD_SEED(self, op):
        B, HW, ld = op.i[:3]
        d = self.V(op.p[0], (B, 6, HW), (6 * HW, HW, 1))
        dyn = self.flat(op.p[1], 2 * B)
        dyn[:B] = th.maximum(dyn[:B], image_max(d))
        scale = seed_scale(dyn[:B].clone())
        dyn[B:] = scale
        self.V(op.p[2], (B, HW, 6), (HW * ld, ld, 1)).copy_(quantize(d, scale.view(B, 1, 1)).permute(0, 2, 1))

    def op_GRAD_UNSCALE(self, op):
        B, HW, ld = op.i[:3]
        dyn = self.flat(op.p[2], 2 * B)
        dx = self.V(op.p[0], (B, 3 * HW), (3 * HW, 1)) * (1.0 / dyn[B:]).view(B, 1)
        if op.p[1] is not None:
            dx = dx + self.V(op.p[1], (B, 3 * HW), (3 * HW, 1))
        self.V(op.p[4], (B, 3 * HW), (3 * HW, 1)).copy_(dx)
        dyn[:B] = 0
        self.V(op.p[3], (B, HW, 6), (HW * ld, ld, 1)).zero_()

    def op_PMV_BWD(self, op):
        B, HW = op.i[:2]
        sc = self.flat(op.p[0], SC["COUNT"])
        shp, st = (B, 3, HW), (3 * HW, HW, 1)
        g = [self.V(q, shp, st) if q is not None else th.zeros(shp) for q in op.p[2:6]]
        G = g[0] + sc[SC["POST_COEF1"]] * g[1]
        gl = g[3] + (self.V(op.p[1], shp, st) * g[2] if op.p[4] is not None else 0)
        d = self.V(op.p[6], (B, 6, HW), (6 * HW, HW, 1))
        d[:, :3] = -sc[SC["SQRT_RECIPM1_AC"]] * G
        d[:, 3:] = (sc[SC["MAX_LOG"]] - sc[SC["MIN_LOG"]]) * 0.5 * gl
        self.V(op.p[7], shp, st).copy_(sc[SC["SQRT_RECIP_AC"]] * G + sc[SC["POST_COEF2"]] * g[1])


def interpreted(eng):
    """route the engine's plan launches through the CPU interpreter"""
    it = AgInterp(eng.plan)
    eng.plan.run_range = lambda a, b, stream=None: it.run_range(a, b)
    eng.plan.run = lambda first=0, count=None, stream=None: it.run(first, len(eng.plan.ops) - first if count is None else count)
    return eng
