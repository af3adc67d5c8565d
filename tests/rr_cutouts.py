"""Test side of the ResizeRight (lanczos3) cutouts on rectangular crops and after the use_augs pipeline: the plan interpreter extended
by the CUTOUTS_RR_* flags 1 (x-axis tables) and 2 (augmented-crop workspace) and CUTOUTS_AUG_* flags 1, and an oracle MakeCutouts that
runs the reference's order -- crop, the torchvision pipeline at crop resolution (oracle.guidance.apply_augs), then
oracle.resize_right.resize_lanczos3 instead of adaptive_avg_pool2d.  Shared by tests/test_rr_cutouts_cpu.py and
tests/test_gpu_rr_cutouts.py."""
import torch as th

from oracle import guidance as og
from oracle.resize_right import resize_lanczos3
from tests.plan_interp import Interp


class AugResizeMakeCutouts(og.MakeCutouts):
    """oracle.guidance.MakeCutouts whose lanczos3 mode also takes the use_augs parameters: every crop goes through apply_augs at its own
    resolution and is then resized to cut_size x cut_size.  The resize runs on the CPU (oracle.resize_right builds its tables there) and
    its result returns to the image's device, so the oracle's networks may live on the GPU."""

    def forward(self, x, use_cache=False, num_cutouts_override=None, coords=None, aug_params=None, aug_noise=None):
        if self.resize != "lanczos3":
            return super().forward(x, use_cache, num_cutouts_override, coords, aug_params, aug_noise)
        outs = []
        for k, (ox, oy, s) in enumerate(coords):
            cut = x[:, :, oy:oy + s, ox:ox + s]
            if aug_params is not None:
                nz = None if aug_noise is None else aug_noise[k][..., :cut.shape[-2], :cut.shape[-1]].to(cut.device)
                cut = og.apply_augs(cut, aug_params[k], nz)
            outs.append(resize_lanczos3(cut.cpu(), (self.cut_size, self.cut_size)).to(x.device))
        return th.cat(outs)


def axis_matrix(left, w, T, S, cs, dtype=th.float32):
    """[cs, S] resampling matrix of one axis' tables: A[o, left[o] + i] = w[o, i] for i < T inside [0, S)"""
    A = th.zeros(cs, S, dtype=dtype)
    for i in range(T):
        idx = left.long() + i
        ok = (idx >= 0) & (idx < S)
        A[th.arange(cs)[ok], idx[ok]] += w[ok, i].to(dtype)
    return A


def crops(coords, H, W):
    """(k, ox, oy, Sy, Sx) of every window: the extents the reference's slicing leaves (clipped at the border, quirk B3)"""
    return [(k, ox, oy, min(s, H - oy), min(s, W - ox)) for k, (ox, oy, s) in enumerate(coords)]


class RRInterp(Interp):
    """the plan interpreter plus the ResizeRight cutouts' per-axis tables and the use_augs crop workspace"""

    def _axis(self, op, axis):
        """the (left, weights, taps | inverse) pointers of axis 0 (y) or 1 (x)"""
        b = 6 if axis == 1 and op.flags & 1 else 3
        return op.p[b], op.p[b + 1], op.p[b + 2]

    def _fwd_matrix(self, op, k, axis, S):
        cutn, cs = op.i[3], op.i[4]
        pl, pw, pt = self._axis(op, axis)
        T = int(self.flat(pt, cutn)[k])
        return axis_matrix(self.V(pl, (cutn, cs), (cs, 1))[k], self.V(pw, (cutn, cs, 16), (cs * 16, 16, 1))[k], T, S, cs)

    def _bwd_matrix(self, op, k, axis, S):
        """[cs, S] from the inverse ranges: M[o, r] = w[o][r - left[o]] for the outputs o in [lo, hi] of input r -- the backward's gather"""
        cutn, cs, Smax = op.i[3], op.i[4], op.i[7]
        pl, pw, pi = self._axis(op, axis)
        left = self.V(pl, (cutn, cs), (cs, 1))[k].long()
        w = self.V(pw, (cutn, cs, 16), (cs * 16, 16, 1))[k]
        inv = self.V(pi, (cutn, Smax, 2), (Smax * 2, 2, 1))[k]
        M = th.zeros(cs, S)
        for r in range(S):
            o = th.arange(int(inv[r, 0]), int(inv[r, 1]) + 1)
            M[o, r] = w[o, r - left[o]]
        return M

    def _ws(self, op, ptr):
        B, cutn, Smax = op.i[0], op.i[3], op.i[7]
        return self.V(ptr, (cutn, B, 3, Smax, Smax), (B * 3 * Smax * Smax, 3 * Smax * Smax, Smax * Smax, Smax, 1))

    def _img(self, op, ptr):
        B, H, W = op.i[:3]
        return self.V(ptr, (B, 3, H, W), (3 * H * W, H * W, W, 1))

    def op_CUTOUTS_RR_FWD(self, op):
        B, H, W, cutn, cs, P, kpad = op.i[:7]
        crop = op.flags & 2
        src = self._ws(op, op.p[0]) if crop else self._img(op, op.p[0])
        mean = th.tensor(op.f[0:3]).view(1, 3, 1, 1)
        std = th.tensor(op.f[3:6]).view(1, 3, 1, 1)
        cuts = []
        for k, ox, oy, sy, sx in crops(self._coords(op), H, W):
            c = src[k, :, :, :sy, :sx] if crop else src[:, :, oy:oy + sy, ox:ox + sx]
            cuts.append(self._fwd_matrix(op, k, 0, sy) @ c @ self._fwd_matrix(op, k, 1, sx).t())
        img = th.cat(cuts)
        img = ((img if crop else (img + 1) * 0.5) - mean) / std
        g2 = (cs // P) ** 2
        self.V(op.p[2], (cutn * B, g2, kpad), (g2 * kpad, kpad, 1)).copy_(self._patchify(img, P, kpad))

    def op_CUTOUTS_RR_BWD(self, op):
        B, H, W, cutn, cs, P, kpad = op.i[:7]
        g2 = (cs // P) ** 2
        dp = self.V(op.p[0], (cutn * B, g2, kpad), (g2 * kpad, kpad, 1)).float()
        dimg = self._unpatchify(dp, P, cs).view(cutn, B, 3, cs, cs)
        std = th.tensor(op.f[3:6]).view(1, 3, 1, 1)
        if op.flags & 2:  # d crop into the workspace, d / d (augmented crop in [0, 1])
            ws = self._ws(op, op.p[2])
            for k, _, _, sy, sx in crops(self._coords(op), H, W):
                ws[k, :, :, :sy, :sx] = self._bwd_matrix(op, k, 0, sy).t() @ dimg[k] @ self._bwd_matrix(op, k, 1, sx) / std * op.f[6]
            return
        gx = th.zeros(B, 3, H, W)
        for k, ox, oy, sy, sx in crops(self._coords(op), H, W):
            gx[:, :, oy:oy + sy, ox:ox + sx] += self._bwd_matrix(op, k, 0, sy).t() @ dimg[k] @ self._bwd_matrix(op, k, 1, sx)
        self._img(op, op.p[2]).copy_(gx * 0.5 / std * op.f[6])

    def _aug_crops(self, op, x01, with_noise):
        """[(k, Sy, Sx, augmented crop [B, 3, Sy, Sx])] of x01 (values in [0, 1]) with the op's parameters (and noise)"""
        B, H, W, cutn = op.i[:4]
        Smax = op.i[7]
        prm = self.V(op.p[3], (cutn, 20), (20, 1))
        nz = None
        if with_noise and op.p[4] is not None:
            nz = self.V(op.p[4], (cutn, 4, B, 3, Smax, Smax), (4 * B * 3 * Smax * Smax, B * 3 * Smax * Smax, 3 * Smax * Smax, Smax * Smax, Smax, 1))
        return [(k, sy, sx, og.apply_augs(x01[:, :, oy:oy + sy, ox:ox + sx], prm[k], None if nz is None else nz[k][..., :sy, :sx]))
                for k, ox, oy, sy, sx in crops(self._coords(op), H, W)]

    def op_CUTOUTS_AUG_FWD(self, op):
        if not op.flags & 1:
            return super().op_CUTOUTS_AUG_FWD(op)
        ws = self._ws(op, op.p[2])
        for k, sy, sx, a in self._aug_crops(op, (self._img(op, op.p[0]) + 1) * 0.5, True):
            ws[k, :, :, :sy, :sx] = a

    def op_CUTOUTS_AUG_BWD(self, op):
        if not op.flags & 1:
            return super().op_CUTOUTS_AUG_BWD(op)
        B, H, W = op.i[:3]
        d = self._ws(op, op.p[0])
        x = th.zeros(B, 3, H, W, requires_grad=True)
        tot = sum((a * d[k, :, :, :sy, :sx]).sum() for k, sy, sx, a in self._aug_crops(op, (x + 1) * 0.5, False))
        (gx,) = th.autograd.grad(tot, x)
        self._img(op, op.p[2]).add_(gx * op.f[6])  # scatter-add into a zeroed buffer (CGD_OP_FILL precedes it)


def interp_runner(eng):
    return RRInterp(eng.plan).run_range
