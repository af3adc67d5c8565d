"""``range_loss`` / ``spherical_dist_loss`` / ``tv_loss`` with the reference's signatures and shapes (cgd/losses.py:5-22), evaluated by
CUDA kernels and differentiable under torch.autograd (csrc/losses.cu: IMG_LOSS_FWD / _BWD, SPH_DIST_FWD / _BWD), so a cond_fn written in
PyTorch gets their gradients.  Values are fp32 and every sum runs in a fixed order: two runs give the same bits.  Gradients come back in
the inputs' dtype; ``create_graph=True`` raises (once_differentiable)."""
from __future__ import annotations

import ctypes
import math

import torch as th

from . import _lib
from ._lib import SC


def _stream():
    return ctypes.c_void_p(th.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _guide(x: th.Tensor):
    """the fused step's tv / range kernel (GUIDE_GRAD through ``cgd_guidance_losses_fwd_bwd``) on one image batch: ([tv, range, sat] per
    image, d(sum tv + sum range) / dx)"""
    if not x.is_cuda:
        raise _lib.CgdError("cgd losses run on the GPU only (no CPU fallback)")
    B, C, H, W = x.shape
    assert C == 3, "losses are defined on RGB images [B,3,H,W]"
    x = x.detach().float().contiguous()
    sc = th.zeros(SC["COUNT"], device=x.device)
    sc[SC["SQRT_RECIP_AC"]] = 1.0
    sc[SC["ONE_MINUS_FAC"]] = 1.0
    seed = th.empty(B * H * W * 8, dtype=th.float16, device=x.device)
    dxd = th.empty_like(x)
    loss = th.zeros(3 * B, device=x.device)
    lib = _lib.load()
    rc = lib.cgd_guidance_losses_fwd_bwd(_p(x), _p(x), None, _p(sc), _p(seed), _p(dxd), _p(loss), ctypes.c_int64(B), ctypes.c_int64(H),
                                         ctypes.c_int64(W), ctypes.c_int64(8), ctypes.c_float(1.0), ctypes.c_float(1.0), ctypes.c_float(0.0),
                                         ctypes.c_float(1.0), _stream())
    _lib.check(rc, "cgd_guidance_losses_fwd_bwd")
    return loss.view(3, B), dxd


def _f32(t: th.Tensor, what: str) -> th.Tensor:
    if not t.is_floating_point():
        raise ValueError(f"{what} takes floating-point tensors, got {t.dtype}")
    return t.detach().float().contiguous()


_TV, _RANGE = 1, 2  # IMG_LOSS_* flags


class _ImgLoss(th.autograd.Function):
    @staticmethod
    def forward(ctx, input, kind):
        what = "tv_loss" if kind == _TV else "range_loss"
        if input.dim() != 4:
            raise ValueError(f"{what} takes [B, C, H, W], got {tuple(input.shape)}")
        x = _f32(input, what)
        B, C, H, W = x.shape
        nblk = max(1, min(math.ceil(C * H * W / 2048), 1024 // B))  # ~8 elements per thread, about a wave of CTAs at most
        partial = th.empty(B * nblk, device=x.device)
        loss = th.empty(B, device=x.device)
        _lib.run_op("IMG_LOSS_FWD", flags=kind, i=[B, C, H, W, nblk], p=[x, partial, loss], what=what)
        ctx.save_for_backward(x)
        ctx.kind, ctx.dtype = kind, input.dtype
        return loss

    @staticmethod
    @th.autograd.function.once_differentiable
    def backward(ctx, d):
        (x,) = ctx.saved_tensors
        dx = th.empty_like(x)
        _lib.run_op("IMG_LOSS_BWD", flags=ctx.kind, i=list(x.shape), p=[x, d.float().contiguous(), dx])
        return dx.to(ctx.dtype), None


def range_loss(input: th.Tensor) -> th.Tensor:
    """mean over C, H, W of (input - input.clamp(-1, 1))^2: fp32 [B]"""
    return _ImgLoss.apply(input, _RANGE)


def tv_loss(input: th.Tensor) -> th.Tensor:
    """L2 total variation with replicate padding, mean over C, H, W: fp32 [B]"""
    return _ImgLoss.apply(input, _TV)


_PAIR_TABLES = {}


def _pair_table(xs: tuple, ys: tuple, device):
    """the broadcast of x rows [*xs] against y rows [*ys] as SPH_DIST's pair list, plus per side the CSR (ptr [N + 1], pair ids [M])
    that the backward gathers over; built on the host once per shape pair"""
    key = (xs, ys, str(device))
    tab = _PAIR_TABLES.get(key)
    if tab is None:
        shape = th.broadcast_shapes(xs, ys)  # raises like torch for shapes it cannot broadcast
        ix = th.arange(math.prod(xs)).view(xs).expand(shape).reshape(-1)
        iy = th.arange(math.prod(ys)).view(ys).expand(shape).reshape(-1)
        csr = []
        for rows, n in ((ix, math.prod(xs)), (iy, math.prod(ys))):
            ptr = th.zeros(n + 1, dtype=th.int64)
            ptr[1:] = th.bincount(rows, minlength=n).cumsum(0)
            csr += [ptr.int().to(device), th.argsort(rows, stable=True).int().to(device)]
        tab = (tuple(shape), th.stack([ix, iy], 1).int().to(device), *csr)
        if len(_PAIR_TABLES) >= 64:
            _PAIR_TABLES.clear()
        _PAIR_TABLES[key] = tab
    return tab


class _SphDist(th.autograd.Function):
    @staticmethod
    def forward(ctx, x, y):
        if x.dim() == 0 or y.dim() == 0 or x.shape[-1] != y.shape[-1]:
            raise ValueError(f"spherical_dist_loss needs x [..., D] and y [..., D] with the same D, got {tuple(x.shape)} and {tuple(y.shape)}")
        if x.device != y.device:
            raise ValueError(f"spherical_dist_loss: x is on {x.device}, y on {y.device}")
        D = x.shape[-1]
        shape, pairs, xptr, xidx, yptr, yidx = _pair_table(tuple(x.shape[:-1]), tuple(y.shape[:-1]), x.device)
        xs, ys = _f32(x, "spherical_dist_loss").view(-1, D), _f32(y, "spherical_dist_loss").view(-1, D)
        M = pairs.shape[0]
        out = th.empty(M, device=x.device)
        if M:
            _lib.run_op("SPH_DIST_FWD", i=[M, D, xs.shape[0], ys.shape[0]], p=[xs, ys, pairs, out], what="spherical_dist_loss")
        ctx.save_for_backward(xs, ys, pairs, xptr, xidx, yptr, yidx)
        ctx.meta = (x.shape, x.dtype, y.shape, y.dtype)
        return out.view(shape)

    @staticmethod
    @th.autograd.function.once_differentiable
    def backward(ctx, d):
        xs, ys, pairs, xptr, xidx, yptr, yidx = ctx.saved_tensors
        xshape, xdtype, yshape, ydtype = ctx.meta
        want = ctx.needs_input_grad[:2]
        dx = th.empty_like(xs) if want[0] else None
        dy = th.empty_like(ys) if want[1] else None
        M = pairs.shape[0]
        if M:
            _lib.run_op("SPH_DIST_BWD", flags=int(want[0]) | 2 * int(want[1]), i=[M, xs.shape[1], xs.shape[0], ys.shape[0]],
                        p=[xs, ys, pairs, d.float().contiguous().view(-1), dx, dy] + ([xptr, xidx] if want[0] else [None, None]) +
                        ([yptr, yidx] if want[1] else [None, None]))
        else:
            dx, dy = (None if t is None else t.zero_() for t in (dx, dy))
        return (None if dx is None else dx.view(xshape).to(xdtype)), (None if dy is None else dy.view(yshape).to(ydtype))


def spherical_dist_loss(x: th.Tensor, y: th.Tensor) -> th.Tensor:
    """2 asin(|x^ - y^| / 2)^2 of F.normalize'd rows, x [..., D] and y [..., D] broadcast like torch (the reference's call site passes
    [1, cutn, B, D] against [1, P, D], cgd/cgd.py:196-197): fp32 of the broadcast batch shape"""
    return _SphDist.apply(x, y)
