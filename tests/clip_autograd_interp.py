"""TEST-ONLY interpreters of the CLIP autograd ops (include/cgd_b200.h CGD_OP_CLIP_PATCHIFY / CLIP_SEED / CLIP_UNPATCHIFY) on top of
tests/plan_interp.py: fp32 math, one fp16 rounding where the kernels store fp16, the kernels' NaN / inf rules."""
from __future__ import annotations

import torch as th

from tests.plan_interp import Interp


def clip_seed_scale(d: th.Tensor, band: float) -> th.Tensor:
    """CLIP_SEED's per-row power of two for fp32 rows d [n, D]: m = max |d| (NaN dropped, inf -> 3e38),
    2^clamp(floor(log2(band / m)), -60, 60), 1 where m == 0"""
    a = d.abs()
    m = th.where(th.isnan(a), th.zeros_like(a), a).amax(1).clamp(max=3.0e38)
    return th.where(m > 0, th.exp2(th.floor(th.log2(band / m.clamp(min=1e-38))).clamp(-60, 60)), th.ones_like(m))


class ClipInterp(Interp):
    def _patch_views(self, op, p_rows, p_img):
        n, nb, R, P, kpad = op.i[:5]
        G2 = (R // P) ** 2
        return (self.V(p_rows, (nb, G2, kpad), (G2 * kpad, kpad, 1)), self.V(p_img, (n, 3, R, R), (3 * R * R, R * R, R, 1)), n, P, kpad, R)

    def op_CLIP_PATCHIFY(self, op):
        rows, x, n, P, kpad, _ = self._patch_views(op, op.p[1], op.p[0])
        rows.zero_()
        rows[:n].copy_(Interp._patchify(x.float(), P, kpad).half())

    def op_CLIP_SEED(self, op):
        n, nb, D = op.i[:3]
        d = self.V(op.p[0], (nb, D), (D, 1)).float().clone()
        d[n:] = 0
        scale = clip_seed_scale(d, op.f[0])
        self.V(op.p[1], (nb, D), (D, 1)).copy_(d * scale[:, None])
        self.flat(op.p[2], nb).copy_(scale)

    def op_CLIP_UNPATCHIFY(self, op):
        rows, dx, n, P, _, R = self._patch_views(op, op.p[0], op.p[2])
        scale = self.flat(op.p[1], op.i[1])[:n]
        dx.copy_(Interp._unpatchify(rows[:n].float(), P, R) * (1.0 / scale).view(n, 1, 1, 1))


def interpreted(model):
    """route a ClipModelB200's plan launches through the CPU interpreter"""
    it = ClipInterp(model.plan)
    model.plan.run_range = lambda a, b, stream=None: it.run_range(a, b)
    model.plan.run = lambda first=0, count=None, stream=None: it.run(first, len(model.plan.ops) - first if count is None else count)
    return model
