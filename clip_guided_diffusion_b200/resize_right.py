"""Host side of the ResizeRight resampler: per-(input size, output size) 1-D resampling tables for the CUDA cutout kernels (at most
``T_MAX`` taps) and for the ``RESIZE_AXIS`` op of image prompts (``t_max=None``: any tap count).

``north_star`` names "MakeCutouts' random-crop + ResizeRight downsample"; the reference's MakeCutouts actually pools
(cgd/modules.py:63) and only ``encode_image_prompt`` calls the vendored resampler (cgd/clip_util.py:95-97, lanczos3, antialiasing).
This mode resizes every crop Sy x Sx (S x S inside the image, clipped at its border like the reference's slicing) -> cut_size x
cut_size exactly like
``cgd/ResizeRight/resize_right.py:31-122`` (tensor path, pad_mode='constant', by_convs=False): for one dimension

    projected grid   g[o] = o / s + (S - 1) / 2 - (O - 1) / (2 s)                      (resize_right.py:126-137), s = O / S
    antialiasing     s < 1: support = 6 / s, kernel(x) = s * lanczos3(s * x)             (resize_right.py:341-353)
    field of view    left[o] = ceil(g[o] - support / 2 - eps), T = ceil(support - eps)   (resize_right.py:140-150)
    weights          kernel(g[o] - (left[o] + i)), normalised to sum 1 per output        (resize_right.py:202-213)
    out[o] = sum_i w[o, i] * in[left[o] + i], samples outside [0, S) are zero            (resize_right.py:216-247)

The same float32 torch arithmetic in the same order as the reference decides the ceil() boundaries; the tables are cached per
crop extent (MakeCutouts draws S in [min(cut_size, side), side]).  Each axis takes the table of its own extent; both axes of a square
crop share one.
"""
from __future__ import annotations

from math import ceil, pi

import numpy as np
import torch as th

T_MAX = 16  # taps per output of the device tables (lanczos3 at s >= 0.4: 6 / 0.4 = 15)
_EPS = float(th.finfo(th.float32).eps)
_cache: dict = {}


def _lanczos3(x: th.Tensor) -> th.Tensor:  # cgd/ResizeRight/interp_methods.py:51-55
    return ((th.sin(pi * x) * th.sin(pi * x / 3) + _EPS) / ((pi ** 2 * x ** 2 / 3) + _EPS)) * (abs(x) < 3).to(x.dtype)


def tables(S: int, O: int, t_max: "int | None" = T_MAX):
    """-> (left int32 [O] relative to the crop, weights float32 [O, t_max] zero-padded, taps T).
    ``t_max=None``: no cap, the weights are [O, T] (the RESIZE_AXIS op of image prompts, any scale factor)."""
    key = (int(S), int(O), t_max)
    if key in _cache:
        return _cache[key]
    if S == O:  # scale factor 1: the reference leaves the dimension untouched (resize_right.py:58-62)
        wt = th.zeros(O, t_max or 1)
        wt[:, 0] = 1.0
        res = (th.arange(O, dtype=th.int32), wt, 1)
        _cache[key] = res
        return res
    s = float(O / S)
    o = th.arange(O)
    grid = o / s + (S - 1) / 2 - (O - 1) / (2 * s)  # float32, like the reference's tensor expression
    if s < 1.0:
        support = 6 / s
        kern = lambda a: s * _lanczos3(s * a)  # noqa: E731
    else:
        support = 6
        kern = _lanczos3
    left = (grid - support / 2 - _EPS).ceil().long()
    T = ceil(support - _EPS)
    if t_max is not None and T > t_max:
        raise ValueError(f"resize {S} -> {O}: {T} taps exceed the device tables ({t_max}); scale factors below 0.4 are unsupported")
    fov = left[:, None] + th.arange(T)
    pad = -int(fov[0, 0])  # the reference shifts grid and field of view by the left padding before evaluating the kernel
    w = kern((grid + pad)[:, None] - (fov + pad))
    sw = w.sum(1, keepdim=True)
    sw[sw == 0] = 1
    w = w / sw
    wt = th.zeros(O, t_max or T)
    wt[:, :T] = w
    res = (left.to(th.int32).contiguous(), wt.contiguous(), T)
    _cache[key] = res
    return res


def inverse_ranges(left: th.Tensor, T: int, S: int):
    """For every input index r in [0, S): the contiguous range [lo, hi] of outputs whose field of view contains r
    (left is non-decreasing); lo > hi when no output touches r.  -> int32 [S, 2]"""
    l = left.numpy().astype(np.int64)
    r = np.arange(S)
    lo = np.searchsorted(l + T - 1, r, side="left")   # first o with left[o] + T - 1 >= r
    hi = np.searchsorted(l, r, side="right") - 1      # last o with left[o] <= r
    return th.from_numpy(np.stack([lo, hi], 1).astype(np.int32))
