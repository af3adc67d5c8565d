"""TEST-ONLY interpreters of the LPIPS autograd ops (include/cgd_b200.h CGD_OP_LPIPS_PAIR_FWD / LPIPS_LOSS / LPIPS_SEED / LPIPS_PAIR_BWD and
PM_TO_NCHW flags 8) on top of tests/plan_interp.py: fp32 math, one fp16 rounding where the kernels store fp16, the kernels' NaN / inf
rules and saturation."""
from __future__ import annotations

import torch as th

from tests.plan_interp import Interp


def lpips_seed_scale(d: th.Tensor, n0: int, n1: int, band: float) -> th.Tensor:
    """LPIPS_SEED's powers of two for d_loss [B]: [trunk 0 rows | trunk 1 rows]; m = |d[b]| for a row of its own image, the maximum over
    all images for a broadcast row (NaN dropped, inf -> 3e38); 2^clamp(floor(log2(band / m)), -60, 60), 1 where m == 0"""
    B = d.shape[0]
    a = d.float().abs()
    a = th.where(th.isnan(a), th.zeros_like(a), a).clamp(max=3.0e38)
    ms = [a if n == B else a.amax().expand(1) for n in (n0, n1)]
    m = th.cat(ms)
    return th.where(m > 0, th.exp2(th.floor(th.log2(band / m.clamp(min=1e-38))).clamp(-60, 60)), th.ones_like(m))


def pair_seed(fs: th.Tensor, fo: th.Tensor, w: th.Tensor, a: th.Tensor, eps: float = 1e-10) -> th.Tensor:
    """fp32 d / d fs of sum_b a_b sum_c w_c (fs_c / (||fs|| + 1e-10) - fo_c / (||fo|| + 1e-10))^2 per pixel; fs [Ns, HW, C], fo [No, HW, C],
    a [B] (already times the row's scale / HW), broadcast rows summed over b in order.  Saturated like the kernel."""
    B = a.shape[0]
    rs = fs.pow(2).sum(-1, keepdim=True).sqrt()
    ns = rs + eps
    xo = fo / (fo.pow(2).sum(-1, keepdim=True).sqrt() + eps)
    out = th.zeros_like(fs)
    w = w.to(fs.dtype)
    for b in range(B):
        r = 0 if fs.shape[0] == 1 else b
        f, n, rr = fs[r], ns[r], rs[r]
        g = 2 * w * (f / n - xo[0 if fo.shape[0] == 1 else b])
        gx = (g * f).sum(-1, keepdim=True)
        c2 = th.where(rr > 0, gx / (n * n * rr.clamp(min=1e-38)), th.zeros_like(gx))
        out[r] = out[r] + a[b] * (g / n - f * c2)
    return th.where(th.isfinite(out), out.clamp(-60000, 60000), out)


class LpipsInterp(Interp):
    def op_LPIPS_PAIR_FWD(self, op):
        B, HW, C, n0, n1, nblk = op.i[:6]
        f0 = self.V(op.p[0], (n0, HW, C), (HW * C, C, 1)).float()
        f1 = self.V(op.p[1], (n1, HW, C), (HW * C, C, 1)).float()
        w = self.flat(op.p[2], C)
        x0 = f0 / (f0.pow(2).sum(-1, keepdim=True).sqrt() + 1e-10)
        x1 = f1 / (f1.pow(2).sum(-1, keepdim=True).sqrt() + 1e-10)
        per = ((x0 - x1) ** 2 * w).sum(-1).expand(B, HW)  # [B, HW]
        blk = (th.arange(HW) // 8) % nblk
        self.V(op.p[3], (B, nblk), (nblk, 1)).copy_(th.zeros(B, nblk).index_add_(1, blk, per))

    def op_LPIPS_LOSS(self, op):
        B = op.i[0]
        total = th.zeros(B)
        for k in range(5):
            total = total + self.V(op.p[k], (B, op.i[1 + k]), (op.i[1 + k], 1)).sum(1) * op.f[k]
        self.flat(op.p[5], B).copy_(total)

    def op_LPIPS_SEED(self, op):
        B, n0, n1 = op.i[:3]
        self.flat(op.p[1], n0 + n1).copy_(lpips_seed_scale(self.flat(op.p[0], B), n0, n1, op.f[0]))

    def op_LPIPS_PAIR_BWD(self, op):
        B, HW, C, n0, n1 = op.i[:5]
        f = [self.V(op.p[0], (n0, HW, C), (HW * C, C, 1)).float(), self.V(op.p[1], (n1, HW, C), (HW * C, C, 1)).float()]
        w = self.flat(op.p[2], C)
        d = self.flat(op.p[3], B)
        dyn = self.flat(op.p[4], n0 + n1)
        for s, ns in enumerate((n0, n1)):
            if op.flags & (1 << s):
                srow = dyn[s * n0:s * n0 + ns]
                a = d * (srow if ns == B else srow.expand(B)) * (1.0 / HW)
                self.V(op.p[5 + s], (ns, HW, C), (HW * C, C, 1)).copy_(pair_seed(f[s], f[1 - s], w, a))

    def op_PM_TO_NCHW(self, op):
        if not op.flags & 8:
            return super().op_PM_TO_NCHW(op)
        N, C, HW, ld = op.i[:4]
        src = self.V(op.p[0], (N, HW, C), (HW * ld, ld, 1)).float() * op.f[0]
        if op.flags & 4:
            src = src * th.tensor(op.f[1:4][:C]).view(1, 1, C)
        src = src / self.flat(op.p[2], N).view(N, 1, 1)
        dst = self.V(op.p[1], (N, C, HW), (C * HW, HW, 1))
        dst.copy_(dst + src.permute(0, 2, 1) if op.flags & 2 else src.permute(0, 2, 1))


def interpreted(model):
    """route every plan an LPIPS model builds through the CPU interpreter (the model's device must be the CPU)"""
    build = model.plan_for

    def plan_for(*key):
        fresh = key not in model.plans
        pp = build(*key)
        if fresh:
            it = LpipsInterp(pp.plan)
            pp.ran = []

            def run_range(a, b, stream=None, it=it, pp=pp):
                pp.ran.append(a)
                with th.enable_grad():  # the MAXPOOL2_BWD interpreter differentiates max_pool2d, also inside an autograd backward
                    it.run_range(a, b)
            pp.plan.run_range = run_range
        return pp
    model.plan_for = plan_for
    return model
