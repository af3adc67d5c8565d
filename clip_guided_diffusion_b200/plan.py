"""Plan builder: turns a network description into the flat op list of include/cgd_b200.h.

A *plan* is built once per (network, batch shape): every activation, saved tensor, gradient and workspace gets a
fixed offset in one arena (a single device allocation, 180 GB HBM makes reuse unnecessary at these sizes), weights
are packed into the kernel layouts and uploaded into the same arena, and the forward and input-gradient backward
op lists are emitted.  Per timestep the host only replays the list (``Plan.run``; normally inside a CUDA graph).

The backward list is produced by a tape at plan-build time (hand-scheduled reverse mode, dgrad only -- no weight
gradients exist on this path, cgd/cgd.py:228, cgd/script_util.py:318); nothing is traced at run time.
"""
from __future__ import annotations

import ctypes
import math
import os
from dataclasses import dataclass, field
from typing import Callable, Optional

import torch as th

from . import _lib
from ._lib import OP, CgdOp

_DT = {"h": (2, th.float16), "f": (4, th.float32), "i32": (4, th.int32), "i64": (8, th.int64), "u32": (4, th.int32)}


@dataclass
class Buf:
    """A typed region of the arena."""
    off: int  # byte offset
    numel: int
    dt: str
    name: str = ""

    @property
    def nbytes(self):
        return self.numel * _DT[self.dt][0]


@dataclass
class Act:
    """Pixel-major fp16 activation view: [N, H, W, C] with row stride ld (elements), image stride H*W*ld."""
    buf: Buf
    eoff: int  # element offset into buf
    N: int
    H: int
    W: int
    C: int
    ld: int
    frozen: bool = False  # never accumulate into this storage in place

    @property
    def HW(self):
        return self.H * self.W

    @property
    def rows(self):
        return self.N * self.H * self.W

    def cslice(self, c0, c1):
        return Act(self.buf, self.eoff + c0, self.N, self.H, self.W, c1 - c0, self.ld, self.frozen)

    def key(self):
        return (self.buf.off, self.eoff, self.C, self.ld)


@dataclass
class PlanOp:
    code: int
    flags: int = 0
    i: list = field(default_factory=list)
    f: list = field(default_factory=list)
    p: list = field(default_factory=list)  # entries: None | (Buf, element offset)
    tag: str = ""


def _round_up(a, b):
    return (a + b - 1) // b * b


def pick_bn(npad: int, m_tiles: int, kblocks: int = 1 << 30) -> int:
    """Output-channel tile width.  The conv kernel runs one 128-pixel x BN tile per CTA and one CTA per SM (its operand ring
    takes most of the shared memory), so a layer takes ceil(tiles / N_SMS) rounds; wide tiles amortise the A-operand traffic
    and the per-tile epilogue (a wgmma of N = 256 reads the same 64-row A slice as one of N = 64), narrow ones fill the
    machine: maximise utilisation x a per-width efficiency prior (256 > 192 > 128 > 64).
    Short-K GEMMs (<= 16 K-blocks: 1x1 convs, the ViT's K = 768 Linears) that fit one round are latency-bound, not
    tensor-bound: the narrowest tile that still fits one round wins and split-K (a second launch) does not pay."""
    cands = [b for b in (256, 192, 128, 64, 32, 16) if npad % b == 0]
    big = [b for b in cands if b >= 64]
    if not big:
        return cands[0]
    if kblocks <= 16:
        one_round = [b for b in big if m_tiles * (npad // b) <= N_SMS]
        if one_round:
            return min(one_round)
    eff = {256: 1.0, 192: 0.95, 128: 0.85, 64: 0.6}
    best, best_score = big[0], -1.0
    for b in big:
        tiles = m_tiles * (npad // b)
        rounds = -(-tiles // N_SMS)
        util = tiles / (rounds * float(N_SMS))
        if tiles < N_SMS:  # split-K will add parallelism; do not punish wide tiles too hard
            util = max(util, 0.6)
        score = util * eff[b]
        if score > best_score + 1e-9:
            best, best_score = b, score
    return best


def conv_tile_count(NB, H, W):
    tw = 1
    while tw < W and tw < 128:
        tw <<= 1
    hceil = 1
    while hceil < H:
        hceil <<= 1
    t_h = min(128 // tw, hceil)
    tn = 128 // (tw * t_h)
    return -(-W // tw) * -(-H // t_h) * -(-NB // tn)


def pick_splits(m_tiles, n_tiles, kblocks, npad, ws_cap_bytes=16 << 20) -> int:
    """split-K factor for layers whose output tiles cannot fill the SMs: aim at one full round, keep at least
    6 K-blocks (of 64) per tile so the TMA/MMA pipeline amortises its fill, bound the fp32 partial workspace."""
    tiles = m_tiles * n_tiles
    if tiles * 2 > N_SMS or kblocks <= 16:
        return 1
    s = min(kblocks // 6, N_SMS // tiles, 32)
    cap = ws_cap_bytes // (m_tiles * 128 * npad * 4)
    s = max(1, min(s, cap))
    per = -(-kblocks // s)
    return -(-kblocks // per)


_CLUSTER_CAP = {}
# co-resident clusters of S CTAs of the conv kernel (one CTA per SM; the same for every tile width), cudaOccupancyMaxActiveClusters on
# an H100 80GB HBM3 (132 SMs): the answers CPU plan builds use, so that they make the same choices as the device
_H100_CLUSTER_CAP = {1: 132, 2: 66, 4: 30, 8: 15}


def cluster_capacity(bn: int, S: int) -> int:
    """co-resident clusters of S CTAs for tile width bn: asked from the library on a CUDA box (cudaOccupancyMaxActiveClusters),
    the H100 answers when there is no device (CPU plan builds: interpreter tests, op_report)"""
    key = (bn, S)
    if key not in _CLUSTER_CAP:
        cap = -1
        try:
            import torch as _th
            if _th.cuda.is_available():
                from . import _lib
                cap = int(_lib.load().cgd_conv_cluster_capacity(bn, S))
        except Exception:
            cap = -1
        _CLUSTER_CAP[key] = cap if cap >= 0 else _H100_CLUSTER_CAP[S]
    return _CLUSTER_CAP[key]


def pick_cluster_split(m_tiles: int, npad: int, kblocks: int, cout: int):
    """(BN, S, K-blocks per CTA) for the in-cluster split-K path of the conv kernel (csrc/conv_tc.cu, CONV i23), or None.  One
    cluster of S CTAs per output tile of 128 pixels x BN channels; the whole launch must fit one wave of clusters
    (`cluster_capacity`); each CTA gets >= 3 K-blocks and BN / S (the columns a CTA reduces and stores) is a multiple of 16.
    The shortest K loop per CTA wins; ties go to the smaller cluster (less distributed-shared-memory traffic), then the wider tile."""
    if cout % 8:
        return None
    best = None
    for bn in (256, 192, 128, 64):
        if npad % bn:
            continue
        tiles = m_tiles * (npad // bn)
        for S in (2, 4, 8):
            if bn % S or (bn // S) % 16 or tiles > cluster_capacity(bn, S):
                continue
            kps = -(-kblocks // S)
            if kps < 3 or (S - 1) * kps >= kblocks:
                continue
            if best is None or kps < best[2]:
                best = (bn, S, kps)
    return best


def gn_fused_cluster(N: int, HW: int, C: int, maxv: int) -> int:
    """Cluster size (CTAs along the pixel dimension) of the single-launch GroupNorm kernels (csrc/norm_fused.cu), or 0 when the
    two-pass kernels are the better choice.  512 threads, 16-byte vectors, at most `maxv` vectors per thread (16 forward,
    8 backward), clusters of at most 4 CTAs.  A CTA reads only its groups'
    channels of every pixel (32-128 contiguous bytes), so beyond ~4 MB per image the partial-line traffic loses against the
    full-row two-pass kernels; below, the single launch wins by 2-4x."""
    if C % 256 != 0 or C > 4096 or HW * C > (2 << 20):
        return 0
    cpg = C // 32
    gpc = 16 // cpg if cpg < 16 else 1
    vpp = gpc * cpg // 8
    pp = 512 // vpp
    cs = 1
    while cs <= 4 and -(-HW // cs) > maxv * pp:
        cs *= 2
    if cs > 4:
        return 0
    while cs < 4 and (32 // gpc) * cs * N < 128 and -(-HW // (2 * cs)) >= pp:
        cs *= 2
    return cs


N_SMS = 132  # H100 SXM


def gn_grid_ctas(N: int, HW: int, C: int) -> int:
    """CTAs per image of the persistent GroupNorm kernels (csrc/norm_grid.cu): one resident CTA per SM, every CTA at least
    one pass of its pixel lanes; 0 when the batch alone exceeds the SM count (two-pass kernels then)."""
    if C % 64 != 0 or C > 2048 or N > N_SMS:
        return 0
    pp = 512 // (C // 8)
    return max(1, min(N_SMS // N, HW // pp))


class Plan:
    def __init__(self, conv_impl: int = 0):
        self._gn_scratch = None
        self.grid_gn = True  # single persistent launch with a grid barrier for the large GroupNorms (csrc/norm_grid.cu)
        self.fused_gn = True  # single-launch GroupNorm where the slab fits a cluster (csrc/norm_fused.cu)
        self.ops: list[PlanOp] = []
        self._size = 0
        self._consts: list[tuple[Buf, th.Tensor]] = []
        self._tape: list[Callable[[], None]] = []
        self._grads: dict = {}
        self.conv_impl = conv_impl
        # split-K reduced inside a thread-block cluster through DSMEM (csrc/conv_tc.cu) instead of partials + a reduce launch
        self.cluster_splitk = os.environ.get("CGD_CONV_CLUSTER", "1") == "1"
        # ... also for one-wave layers that did not need split-K to fill the machine but have long K loops (the 64 x 64 level's
        # 512 -> 512 and 1024 -> 512 3x3s): a wider tile split along K inside a cluster shortens the K loop per SM.
        # CGD_CLUSTER_WIDE=0 switches it off for A/B runs.
        self.cluster_wide = os.environ.get("CGD_CLUSTER_WIDE", "1") == "1"
        # (Quick)GELU output Act key -> (its pre-activation Act, exact GELU?) (dgrad-epilogue fusion, CONV flags 4 / 8)
        self._gelu_src = {}
        self.arena: Optional[th.Tensor] = None
        self.handle = None
        self._c_ops = None
        self.marks: dict[str, int] = {}
        self.bufs: list[Buf] = []

    # ------------------------------------------------------------------ memory
    def new(self, numel: int, dt: str, name: str = "") -> Buf:
        off = _round_up(self._size, 256)
        b = Buf(off, int(numel), dt, name)
        self._size = off + b.nbytes
        self.bufs.append(b)
        return b

    def const(self, t: th.Tensor, dt: str, name: str = "") -> Buf:
        t = t.detach().to(_DT[dt][1]).contiguous().cpu()
        b = self.new(t.numel(), dt, name)
        self._consts.append((b, t))
        return b

    def act(self, N, H, W, C, name="", ld=None) -> Act:
        ld = ld or C
        return Act(self.new(N * H * W * ld, "h", name), 0, N, H, W, C, ld)

    # ------------------------------------------------------------------ low-level emit
    def emit(self, code, *, flags=0, i=(), f=(), p=(), tag=""):
        self.ops.append(PlanOp(OP[code] if isinstance(code, str) else code, flags, list(i), list(f), list(p), tag))

    def mark(self, name):
        self.marks[name] = len(self.ops)

    @staticmethod
    def _ap(a: Optional[Act]):
        return None if a is None else (a.buf, a.eoff)

    @staticmethod
    def _bp(b: Optional[Buf], eoff: int = 0):
        return None if b is None else (b, eoff)

    # ------------------------------------------------------------------ gradient bookkeeping (build time only)
    def grad_of(self, a: Act) -> Optional[Act]:
        return self._grads.get(a.key())

    def add_grad(self, a: Act, g: Act):
        """Accumulate gradient view g into the gradient of activation a (alias when first, in-place ADD otherwise)."""
        cur = self._grads.get(a.key())
        if cur is None:
            self._grads[a.key()] = g
            return
        if cur.frozen:
            dst = self.act(a.N, a.H, a.W, a.C, "gsum")
        else:
            dst = cur
        self.emit("ADD", i=[a.rows, a.C, cur.ld, g.ld, dst.ld], p=[self._ap(cur), self._ap(g), self._ap(dst)], tag="grad+=")
        self._grads[a.key()] = dst

    def writable_grad(self, a: Act) -> tuple[Optional[Act], bool]:
        """Gradient storage of `a` that a kernel may accumulate into in place: (act, exists)."""
        cur = self._grads.get(a.key())
        if cur is None:
            return None, False
        if cur.frozen:
            dst = self.act(a.N, a.H, a.W, a.C, "gcopy")
            self.emit("COPY", i=[a.rows, a.C, cur.ld, dst.ld], p=[self._ap(cur), self._ap(dst)], tag="grad copy")
            self._grads[a.key()] = dst
            return dst, True
        return cur, True

    def backward(self):
        """Emit the backward op list (reverse tape)."""
        for fn in reversed(self._tape):
            fn()
        self._tape = []

    # ------------------------------------------------------------------ conv / GEMM
    def _emit_conv(self, x_ptr, x_strides, NB, H, W, Cin, wbuf, npad, Cout, taps, bias, res_ptr, res_strides, out_ptr, out_strides,
                   out_f32=False, out_sc=1, tag="", res_gelu=False, exact_gelu=False):
        m_tiles = conv_tile_count(NB, H, W)
        kblocks = taps * Cin // 64
        bn = pick_bn(npad, m_tiles, kblocks)
        splits = pick_splits(m_tiles, npad // bn, kblocks, npad)
        if exact_gelu:
            # the exact GELU has no stand-alone backward: its dgrad always takes the CONV flags 8 epilogue, which needs one K loop per
            # tile (no split-K) and tiles of >= 64 columns -- forced here instead of picked (small batches would pick split-K)
            assert self.exact_gelu_epilogue_ok(npad, Cout), tag
            bn, splits = max(bn, 64), 1
        cluster = 0
        if splits > 1 and self.cluster_splitk and self.conv_impl in (0, 3) and not out_f32 and out_sc == 1:
            # one launch and no fp32 partial tensor, unless the workspace split would give each CTA a shorter K loop
            pick = pick_cluster_split(m_tiles, npad, kblocks, Cout)
            if pick is not None and pick[2] <= -(-kblocks // splits):
                bn, splits = pick[:2]
                cluster = 1
        elif (splits == 1 and self.cluster_wide and self.cluster_splitk and self.conv_impl in (0, 3) and not out_f32 and out_sc == 1
              and not res_gelu  # the QuickGELU' epilogue needs splits == 1 (conv_gelu_epilogue_ok)
              and m_tiles >= 2 and kblocks >= 32):
            # one wave of narrow tiles with a long K loop (the 64 x 64 level: 64 BN-128 tiles x 72 K-blocks = 33 us at 0.46 us per K-block):
            # wider tiles split along K inside a cluster can be shorter even though no split-K was "needed" to fill the machine
            pick = pick_cluster_split(m_tiles, npad, kblocks, Cout)
            rounds = -(-(m_tiles * (npad // bn)) // N_SMS)
            if pick is not None and 2 * pick[2] <= rounds * kblocks:  # at least halves the K loop per SM
                bn, splits = pick[:2]
                cluster = 1
        ws = None
        if splits > 1 and not cluster:
            ws = self.new(splits * m_tiles * 128 * npad, "f", "splitk_ws")
        i = [NB, H, W, Cin, Cout, npad, taps, *x_strides, *out_strides, *(res_strides or (0, 0, 0)), bn, splits, self.conv_impl, out_sc,
             0, 0, 0, cluster]  # i20..i22 reserved
        if res_gelu and not exact_gelu:
            assert self.conv_gelu_epilogue_ok(NB, H, W, Cin, npad, Cout, taps), tag
        self.emit("CONV", flags=(1 if out_f32 else 0) | ((8 if exact_gelu else 4) if res_gelu else 0), i=i,
                  p=[x_ptr, self._bp(wbuf), self._bp(bias), res_ptr, out_ptr, self._bp(ws), None], tag=tag)

    def conv_gelu_epilogue_ok(self, NB, H, W, Cin, npad, Cout, taps) -> bool:
        """would this conv run with the epilogue that implements CONV flags 4?  Mirrors the choices of `_emit_conv` /
        conv_tc_prepare: wgmma path, >= 2 pixel tiles, no split-K, BN >= 64, whole 64-channel chunks."""
        if self.conv_impl not in (0, 3) or os.environ.get("CGD_QGELU_EPI", "1") == "0":
            return False
        m_tiles = conv_tile_count(NB, H, W)
        kblocks = taps * Cin // 64
        bn = pick_bn(npad, m_tiles, kblocks)
        return (m_tiles >= 2 or self.conv_impl == 3) and pick_splits(m_tiles, npad // bn, kblocks, npad) == 1 and bn >= 64 and Cout % 64 == 0

    def exact_gelu_epilogue_ok(self, npad, Cout) -> bool:
        """can a dgrad take the exact-GELU' epilogue (CONV flags 8)?  Any shape on the wgmma kernels (`_emit_conv` forces BN >= 64 and no
        split-K for it, and CGD_QGELU_EPI does not apply: there is no other backward); not on the SIMT verification kernel (conv_impl 1)"""
        return self.conv_impl != 1 and npad % 64 == 0 and Cout % 64 == 0

    @staticmethod
    def _strides(a: Act):
        return (a.H * a.W * a.ld, a.W * a.ld, a.ld)

    def conv(self, x: Act, w: "ConvW", res: Optional[Act] = None, out: Optional[Act] = None, name="conv") -> Act:
        """y = conv(x) + bias (+ res).  Registers the dgrad on the tape."""
        assert x.C == w.cin_pad, (x.C, w.cin_pad, name)
        y = out if out is not None else self.act(x.N, x.H, x.W, w.cout, name)
        assert y.C == w.cout and (y.N, y.H, y.W) == (x.N, x.H, x.W)
        self._emit_conv(self._ap(x), self._strides(x), x.N, x.H, x.W, x.C, w.fwd, w.fwd_npad, w.cout, w.taps, w.bias,
                        self._ap(res), self._strides(res) if res is not None else None, self._ap(y), self._strides(y), tag=name)

        def bwd():
            dy = self.grad_of(y)
            if dy is None:
                return
            if res is not None:
                self.add_grad(res, dy)
            if w.bwd is None:
                return
            u, exact = self._gelu_src.get(x.key(), (None, False))
            fusable = (self.exact_gelu_epilogue_ok(w.bwd_npad, x.C) if exact
                       else self.conv_gelu_epilogue_ok(x.N, x.H, x.W, dy.C, w.bwd_npad, x.C, w.taps))
            if u is not None and self.grad_of(x) is None and u.ld == u.C and fusable:
                # x = QuickGELU(u) feeds only this conv: its dgrad epilogue multiplies by QuickGELU'(u) (CONV flags 4; GELU'(u), flags 8,
                # for an exact GELU) and writes d u directly -- no d a tensor, no QGELU_BWD launch (quick_gelu's own backward then finds
                # no gradient and emits nothing)
                du = self.act(u.N, u.H, u.W, u.C, "d_" + name + ".gelu")
                self._emit_conv(self._ap(dy), self._strides(dy), x.N, x.H, x.W, dy.C, w.bwd, w.bwd_npad, x.C, w.taps, None,
                                self._ap(u), self._strides(u), self._ap(du), self._strides(du), tag="d_" + name + "*gelu'", res_gelu=True,
                                exact_gelu=exact)
                self.add_grad(u, du)
                return
            cur, has = self.writable_grad(x)
            dx = cur if has else self.act(x.N, x.H, x.W, x.C, "d_" + name)
            # dgrad: same kernel over dy with tap-flipped, transposed weights; existing dx folded in as the residual
            self._emit_conv(self._ap(dy), self._strides(dy), x.N, x.H, x.W, dy.C, w.bwd, w.bwd_npad, x.C, w.taps, None,
                            self._ap(cur) if has else None, self._strides(cur) if has else None, self._ap(dx), self._strides(dx),
                            tag="d_" + name)
            self._grads[x.key()] = dx

        self._tape.append(bwd)
        return y

    # ------------------------------------------------------------------ GroupNorm (+SiLU, +scale/shift)
    def group_norm(self, x: Act, gamma: Buf, beta: Buf, emb: Optional[tuple] = None, silu=True, eps=1e-5, name="gn") -> Act:
        N, HW, C = x.N, x.HW, x.C
        y = self.act(N, x.H, x.W, C, name)
        stats = self.new(N * 64, "f", name + "_stats")
        embp = self._bp(emb[0], emb[1]) if emb is not None else None
        cs_f = gn_fused_cluster(N, HW, C, 16) if self.fused_gn else 0
        gn_g = gn_grid_ctas(N, HW, C) if self.grid_gn else 0
        if cs_f:
            self.emit("GN_FWD_FUSED", flags=1 if silu else 0, i=[N, HW, C, x.ld, y.ld, cs_f], f=[eps],
                      p=[self._ap(x), self._bp(gamma), self._bp(beta), embp, self._ap(y), self._bp(stats)], tag=name)
        elif gn_g:
            partials = self.new(N * gn_g * 64, "f", name + "_part")
            bar = self.new(2, "u32", name + "_bar")
            self.emit("GN_FWD_GRID", flags=1 if silu else 0, i=[N, HW, C, x.ld, y.ld, gn_g], f=[eps],
                      p=[self._ap(x), self._bp(gamma), self._bp(beta), embp, self._ap(y), self._bp(stats), self._bp(partials), self._bp(bar)], tag=name)
        else:
            pp = max(1, 256 // (C // 8))
            nchunk = int(min(max(1, -(-HW // (pp * 16))), max(1, 296 // N)))
            partials = self.new(N * nchunk * 64, "f", name + "_part")
            counters = self.new(N, "u32", name + "_cnt")
            self.emit("GN_STATS", i=[N, HW, C, x.ld, nchunk], f=[eps], p=[self._ap(x), self._bp(partials), self._bp(stats), self._bp(counters)], tag=name)
            self.emit("GN_APPLY", flags=1 if silu else 0, i=[N, HW, C, x.ld, nchunk, y.ld], f=[eps],
                      p=[self._ap(x), self._bp(stats), self._bp(gamma), self._bp(beta), embp, self._ap(y)], tag=name)

        def bwd():
            dy = self.grad_of(y)
            if dy is None:
                return
            common = [self._ap(dy), self._ap(x), self._bp(stats), self._bp(gamma), self._bp(beta), embp]
            cs_b = gn_fused_cluster(N, HW, C, 8) if self.fused_gn else 0
            cur, has = self.writable_grad(x)
            dx = cur if has else self.act(N, x.H, x.W, C, "d_" + name)
            fl = (1 if silu else 0) | (2 if has else 0)
            if cs_b:
                self.emit("GN_BWD_FUSED", flags=fl, i=[N, HW, C, dy.ld, x.ld, dx.ld, cs_b], f=[eps], p=common + [self._ap(dx)], tag="d_" + name)
            elif gn_g:
                bpart = self.new(N * gn_g * 64, "f", name + "_bpart")
                bbar = self.new(2, "u32", name + "_bbar")
                # one scratch tensor shared by every GroupNorm backward of the plan (they run one after the other)
                if self._gn_scratch is None or self._gn_scratch.numel < N * HW * C:
                    self._gn_scratch = self.new(N * HW * C, "h", "gn_bwd_dxhat")
                self.emit("GN_BWD_GRID", flags=fl, i=[N, HW, C, dy.ld, x.ld, dx.ld, gn_g], f=[eps],
                          p=common + [self._ap(dx), self._bp(bpart), self._bp(bbar), self._bp(self._gn_scratch)], tag="d_" + name)
            else:
                pp = max(1, 256 // (C // 8))
                nchunk = int(min(max(1, -(-HW // (pp * 16))), max(1, 296 // N)))
                bpart = self.new(N * nchunk * 64, "f", name + "_bpart")
                sums = self.new(N * 64, "f", name + "_bsums")
                bcnt = self.new(N, "u32", name + "_bcnt")
                self.emit("GN_BWD_STATS", flags=1 if silu else 0, i=[N, HW, C, dy.ld, x.ld, nchunk], f=[eps],
                          p=common + [self._bp(bpart), self._bp(sums), self._bp(bcnt)], tag="d_" + name)
                self.emit("GN_BWD_APPLY", flags=fl, i=[N, HW, C, dy.ld, x.ld, nchunk, dx.ld], f=[eps],
                          p=common + [self._bp(sums), self._ap(dx)], tag="d_" + name)
            self._grads[x.key()] = dx

        self._tape.append(bwd)
        return y

    # ------------------------------------------------------------------ resampling
    def pool2(self, x: Act, name="down") -> Act:
        y = self.act(x.N, x.H // 2, x.W // 2, x.C, name)
        self.emit("POOL2", i=[x.N, x.H, x.W, x.C, x.ld, y.ld], f=[0.25], p=[self._ap(x), self._ap(y)], tag=name)

        def bwd():
            dy = self.grad_of(y)
            if dy is None:
                return
            dx = self.act(x.N, x.H, x.W, x.C, "d_" + name)
            self.emit("UP2", i=[y.N, y.H, y.W, y.C, dy.ld, dx.ld], f=[0.25], p=[self._ap(dy), self._ap(dx)], tag="d_" + name)
            self.add_grad(x, dx)

        self._tape.append(bwd)
        return y

    def up2(self, x: Act, name="up") -> Act:
        y = self.act(x.N, x.H * 2, x.W * 2, x.C, name)
        self.emit("UP2", i=[x.N, x.H, x.W, x.C, x.ld, y.ld], f=[1.0], p=[self._ap(x), self._ap(y)], tag=name)

        def bwd():
            dy = self.grad_of(y)
            if dy is None:
                return
            dx = self.act(x.N, x.H, x.W, x.C, "d_" + name)
            self.emit("POOL2", i=[y.N, y.H, y.W, y.C, dy.ld, dx.ld], f=[1.0], p=[self._ap(dy), self._ap(dx)], tag="d_" + name)
            self.add_grad(x, dx)

        self._tape.append(bwd)
        return y

    def concat(self, a: Act, b: Act, name="cat") -> Act:
        """channel concat [a | b]; `a`/`b` are copied (callers may instead produce `a` directly into the slice)."""
        y = self.act(a.N, a.H, a.W, a.C + b.C, name)
        ya, yb = y.cslice(0, a.C), y.cslice(a.C, a.C + b.C)
        self.emit("COPY", i=[a.rows, a.C, a.ld, ya.ld], p=[self._ap(a), self._ap(ya)], tag=name)
        self.emit("COPY", i=[b.rows, b.C, b.ld, yb.ld], p=[self._ap(b), self._ap(yb)], tag=name)

        def bwd():
            dy = self.grad_of(y)
            if dy is None:
                return
            # slices of a gradient buffer alias storage that later in-place accumulation must not touch
            ga, gb = dy.cslice(0, a.C), dy.cslice(a.C, a.C + b.C)
            ga.frozen = gb.frozen = True
            self.add_grad(a, ga)
            self.add_grad(b, gb)

        self._tape.append(bwd)
        return y

    # ------------------------------------------------------------------ VGG pieces of the LPIPS loss (csrc/lpips.cu)
    def relu(self, x: Act, name="relu") -> Act:
        assert x.ld == x.C
        y = self.act(x.N, x.H, x.W, x.C, name)
        self.emit("RELU_FWD", i=[x.rows * x.C], p=[self._ap(x), self._ap(y)], tag=name)

        def bwd():
            dy = self.grad_of(y)
            if dy is None:
                return
            assert dy.ld == dy.C
            cur, has = self.writable_grad(x)
            dx = cur if has else self.act(x.N, x.H, x.W, x.C, "d_" + name)
            self.emit("RELU_BWD", flags=2 if has else 0, i=[x.rows * x.C], p=[self._ap(dy), self._ap(y), self._ap(dx)], tag="d_" + name)
            self._grads[x.key()] = dx

        self._tape.append(bwd)
        return y

    def maxpool2(self, x: Act, name="maxpool") -> Act:
        assert x.ld == x.C and x.H % 2 == 0 and x.W % 2 == 0
        y = self.act(x.N, x.H // 2, x.W // 2, x.C, name)
        self.emit("MAXPOOL2_FWD", i=[x.N, x.H, x.W, x.C], p=[self._ap(x), self._ap(y)], tag=name)

        def bwd():
            dy = self.grad_of(y)
            if dy is None:
                return
            assert dy.ld == dy.C
            dx = self.act(x.N, x.H, x.W, x.C, "d_" + name)
            self.emit("MAXPOOL2_BWD", i=[x.N, x.H, x.W, x.C], p=[self._ap(dy), self._ap(x), self._ap(dx)], tag="d_" + name)
            self.add_grad(x, dx)

        self._tape.append(bwd)
        return y

    def concat_view(self, y: Act, a: Act, b: Act):
        """`y` = [a | b] where a and b are channel slices of y's own storage, already written there by their producers:
        no forward op; the backward hands the matching slices of dy to a and b."""
        assert a.buf is y.buf and b.buf is y.buf and a.eoff == y.eoff and b.eoff == y.eoff + a.C and a.C + b.C == y.C

        def bwd():
            dy = self.grad_of(y)
            if dy is None:
                return
            ga, gb = dy.cslice(0, a.C), dy.cslice(a.C, a.C + b.C)
            ga.frozen = gb.frozen = True
            self.add_grad(a, ga)
            self.add_grad(b, gb)

        self._tape.append(bwd)
        return y

    # ------------------------------------------------------------------ attention (head dim 64; 128 / 192 / 256 for the 128^2 checkpoint)
    def attention(self, qkv: Act, heads: int, T: int, nbatch: int, legacy_order: bool, causal: bool = False, name="attn",
                  scale: Optional[float] = None) -> Act:
        """qkv: [nbatch*T rows, 3C].  legacy_order: per-head [q|k|v] interleave (UNet QKVAttentionLegacy);
        otherwise [q heads | k heads | v heads] (QKVAttention, nn.MultiheadAttention).  causal: query i attends to keys <= i
        (ATTN_FWD flags 1, the CLIP text tower); forward only.  scale: the softmax scale, 1 / sqrt(head dim) by default (a tower whose
        heads are zero-padded to a wider kernel head dim passes its own, vit.py)."""
        C = qkv.C // 3
        d = C // heads
        assert d in (64, 128, 192, 256), f"attention kernels support head dims 64 / 128 / 192 / 256, got {d}"
        out = Act(self.new(nbatch * T * C, "h", name), 0, qkv.N, qkv.H, qkv.W, C, C)
        lse = self.new(nbatch * heads * T, "f", name + "_lse")
        if legacy_order:
            hs, qo, ko, vo = 3 * d, 0, d, 2 * d
        else:
            hs, qo, ko, vo = d, 0, C, 2 * C
        ii = [nbatch, heads, T, d, T * qkv.ld, qkv.ld, hs, T * out.ld, out.ld, d]
        scale = 1.0 / math.sqrt(d) if scale is None else float(scale)
        q = (qkv.buf, qkv.eoff + qo)
        k = (qkv.buf, qkv.eoff + ko)
        v = (qkv.buf, qkv.eoff + vo)
        self.emit("ATTN_FWD", flags=1 if causal else 0, i=ii, f=[scale], p=[q, k, v, self._ap(out), self._bp(lse)], tag=name)

        def bwd():
            do = self.grad_of(out)
            if do is None:
                return
            if causal:
                raise NotImplementedError(f"{name}: a causal attention has no backward (ATTN_BWD takes no flags)")
            assert do.ld == out.ld
            dqkv = Act(self.new(nbatch * T * qkv.ld, "h", "d_" + name), 0, qkv.N, qkv.H, qkv.W, qkv.C, qkv.ld)
            delta = self.new(nbatch * heads * T, "f", name + "_delta")
            self.emit("ATTN_BWD", i=ii, f=[scale],
                      p=[q, k, v, self._ap(out), self._ap(do), self._bp(lse), (dqkv.buf, qo), (dqkv.buf, ko), (dqkv.buf, vo), self._bp(delta)],
                      tag="d_" + name)
            self.add_grad(qkv, dqkv)

        self._tape.append(bwd)
        return out

    # ------------------------------------------------------------------ LayerNorm / QuickGELU (ViT)
    def layer_norm(self, x: Act, gamma: Buf, beta: Buf, eps=1e-5, rows=None, ldx=None, name="ln") -> Act:
        rows = rows if rows is not None else x.rows
        ldx = ldx if ldx is not None else x.ld
        y = Act(self.new(rows * x.C, "h", name), 0, 1, 1, rows, x.C, x.C)
        stats = self.new(rows * 2, "f", name + "_stats")
        self.emit("LN_FWD", i=[rows, x.C, ldx, y.ld], f=[eps], p=[self._ap(x), self._bp(gamma), self._bp(beta), self._ap(y), self._bp(stats)], tag=name)

        def bwd():
            dy = self.grad_of(y)
            if dy is None:
                return
            if rows == x.rows and ldx == x.ld:
                cur, has = self.writable_grad(x)
                dx = cur if has else self.act(x.N, x.H, x.W, x.C, "d_" + name)
                self.emit("LN_BWD", flags=2 if has else 0, i=[rows, x.C, dy.ld, ldx, dx.ld],
                          p=[self._ap(dy), self._ap(x), self._bp(gamma), self._bp(stats), self._ap(dx)], tag="d_" + name)
                self._grads[x.key()] = dx
            else:
                # strided row subset (cls token of every image): scatter into a zero gradient of the full tensor.  The arena
                # is zero-initialised and only these rows are ever written, so the other rows stay zero across replays.
                assert self.grad_of(x) is None
                dx = self.act(x.N, x.H, x.W, x.C, "d_" + name)
                dx.frozen = True
                self.emit("LN_BWD", i=[rows, x.C, dy.ld, ldx, ldx], p=[self._ap(dy), self._ap(x), self._bp(gamma), self._bp(stats), self._ap(dx)],
                          tag="d_" + name)
                self._grads[x.key()] = dx

        self._tape.append(bwd)
        return y

    def attnpool_embed(self, x: Act, pos: Buf, name="attnpool.embed") -> Act:
        """[3P] CLIP AttentionPool2d token assembly: [n, HW, C] -> [n*(HW+1) rows, C] = [mean; x] + positional_embedding"""
        n, HW, C = x.N, x.HW, x.C
        y = Act(self.new(n * (HW + 1) * C, "h", name), 0, 1, 1, n * (HW + 1), C, C)
        self.emit("ATTNPOOL_EMBED_FWD", i=[n, HW, C, x.ld], p=[self._ap(x), self._bp(pos), self._ap(y)], tag=name)

        def bwd():
            dy = self.grad_of(y)
            if dy is None:
                return
            assert dy.ld == C
            cur, has = self.writable_grad(x)
            dx = cur if has else self.act(x.N, x.H, x.W, x.C, "d_" + name)
            self.emit("ATTNPOOL_EMBED_BWD", flags=2 if has else 0, i=[n, HW, C, dx.ld], p=[self._ap(dy), self._ap(dx)], tag="d_" + name)
            self._grads[x.key()] = dx

        self._tape.append(bwd)
        return y

    def gather_rows(self, x: Act, rows: int, ldx: int, name="rows") -> Act:
        """y[r, :] = x[row r * (ldx / x.ld), :]: every (ldx / x.ld)-th row of x as a dense [rows, C] matrix (first token of every image).
        Backward scatters into a zero gradient of the full tensor: the arena is zero-initialised and only these rows are ever
        written, so the others stay zero across replays (same scheme as the strided layer_norm)."""
        y = Act(self.new(rows * x.C, "h", name), 0, 1, 1, rows, x.C, x.C)
        self.emit("COPY", i=[rows, x.C, ldx, y.ld], p=[self._ap(x), self._ap(y)], tag=name)

        def bwd():
            dy = self.grad_of(y)
            if dy is None:
                return
            assert self.grad_of(x) is None
            dx = self.act(x.N, x.H, x.W, x.C, "d_" + name)
            dx.frozen = True
            self.emit("COPY", i=[rows, x.C, dy.ld, ldx], p=[self._ap(dy), self._ap(dx)], tag="d_" + name)
            self._grads[x.key()] = dx

        self._tape.append(bwd)
        return y

    def quick_gelu(self, u: Act, name="gelu", exact=False) -> Act:
        """QuickGELU, or with `exact` the erf GELU (QGELU_FWD flags 1).  The backward of either is normally fused into the consuming
        conv's dgrad epilogue (CONV flags 4 / 8); only QuickGELU has a stand-alone backward op."""
        assert u.ld == u.C
        a = self.act(u.N, u.H, u.W, u.C, name)
        self.emit("QGELU_FWD", flags=1 if exact else 0, i=[u.rows * u.C], p=[self._ap(u), self._ap(a)], tag=name)
        self._gelu_src[a.key()] = (u, exact)

        def bwd():
            da = self.grad_of(a)
            if da is None:
                return
            if exact:
                raise NotImplementedError(f"{name}: the exact GELU's backward runs only in the dgrad epilogue (CONV flags 8) of a single "
                                          "consuming conv on the wgmma kernels; the SIMT verification kernel (conv_impl=1) has none")
            assert da.ld == da.C
            du = self.act(u.N, u.H, u.W, u.C, "d_" + name)
            self.emit("QGELU_BWD", i=[u.rows * u.C], p=[self._ap(da), self._ap(u), self._ap(du)], tag="d_" + name)
            self.add_grad(u, du)

        self._tape.append(bwd)
        return a

    # ------------------------------------------------------------------ finalize / run
    def lower(self, base: int):
        """the op list as the C structs of include/cgd_b200.h, pointers = base + arena offsets"""
        assert base % 256 == 0
        arr = (CgdOp * len(self.ops))()
        for k, op in enumerate(self.ops):
            c = arr[k]
            c.code, c.flags = op.code, op.flags
            assert len(op.i) <= _lib.CGD_OP_NI and len(op.f) <= _lib.CGD_OP_NF and len(op.p) <= _lib.CGD_OP_NP, op.tag
            for j, v in enumerate(op.i):
                c.i[j] = int(v)
            for j, v in enumerate(op.f):
                c.f[j] = float(v)
            for j, v in enumerate(op.p):
                c.p[j] = None if v is None else base + v[0].off + v[1] * _DT[v[0].dt][0]
        return arr

    def finalize(self, device):
        """Allocate the arena on `device`, upload constants, lower ops.  On a CUDA device this also creates the
        native plan (TMA descriptors); on CPU the arena exists only so tests can interpret the op list."""
        device = th.device(device)
        nbytes = _round_up(self._size, 256) + 256
        self.arena = th.zeros(nbytes, dtype=th.uint8, device=device)
        for b, t in self._consts:
            self.arena[b.off:b.off + b.nbytes].copy_(t.view(-1).view(th.uint8))
        # the host copies (2.3 GB for the 256x256 UNet) are not kept: the index is what `reload_consts` needs to re-pack a checkpoint
        self.const_index = [(b.name, b.off, b.nbytes) for b, _ in self._consts]
        self._consts = []
        self._consts_done = True
        if device.type != "cuda":
            return self
        lib = _lib.load()
        arr = self.lower(self.arena.data_ptr())
        h = ctypes.c_void_p()
        _lib.check(lib.cgd_plan_create(arr, len(self.ops), ctypes.byref(h)), "cgd_plan_create")
        self.handle, self._c_ops = h, arr
        return self

    def reload_consts(self, shadow: "Plan", first: int = 0) -> int:
        """Overwrite this (finalized) plan's packed constants with those of `shadow` -- a plan built by the same constructor calls
        from another state_dict and never finalized -- starting at constant number `first`.  Names, offsets and sizes must agree
        one by one (same network, same shapes, same packing decisions); nothing else of the arena is touched, op lists, TMA
        descriptors and captured CUDA graphs stay valid (they hold addresses, not values).  Returns the number re-loaded."""
        if self.arena is None:
            raise RuntimeError("reload_consts: the plan is not finalized")
        new = shadow._consts
        if first + len(new) > len(self.const_index):
            raise ValueError(f"reload_consts: {len(new)} constants from #{first} exceed the plan's {len(self.const_index)}")
        base = shadow_off = None
        for j, (b, t) in enumerate(new):
            name, off, nbytes = self.const_index[first + j]
            if base is None:
                base, shadow_off = off, b.off
            if (b.name, b.nbytes, b.off - shadow_off) != (name, nbytes, off - base):
                raise ValueError(f"reload_consts: constant #{first + j} is {name!r} ({nbytes} B at +{off - base}) in the plan but "
                                 f"{b.name!r} ({b.nbytes} B at +{b.off - shadow_off}) in the new pack: different architecture or flags")
        for j, (b, t) in enumerate(new):
            _, off, nbytes = self.const_index[first + j]
            self.arena[off:off + nbytes].copy_(t.view(-1).view(th.uint8), non_blocking=False)
        return len(new)

    def view(self, b: Buf, shape=None) -> th.Tensor:
        t = self.arena[b.off:b.off + b.nbytes].view(_DT[b.dt][1])
        return t.view(shape) if shape is not None else t

    def run(self, first: int = 0, count: Optional[int] = None, stream=None):
        if self.handle is None:
            raise _lib.CgdError("plan has no native handle: it was finalized on a CPU device; the sampling step has no CPU path "
                                "(tests interpret op lists with tests/plan_interp.py)")
        count = len(self.ops) - first if count is None else count
        st = th.cuda.current_stream().cuda_stream if stream is None else stream
        _lib.check(_lib.load().cgd_plan_run(self.handle, first, count, ctypes.c_void_p(st)), "cgd_plan_run")

    def run_range(self, a: str, b: str, stream=None):
        self.run(self.marks[a], self.marks[b] - self.marks[a], stream)

    def conv_flops(self, k: int) -> float:
        """2 * MACs of CONV op k from its executed dims (image channels padded 3 -> 64 count as executed: +1 % on a UNet)"""
        op = self.ops[k]
        assert op.code == OP["CONV"]
        NB, H, W, Cin, Cout, _npad_, taps = op.i[:7]
        return 2.0 * NB * H * W * Cin * Cout * taps

    def num_launches(self, first=0, count=None) -> int:
        count = len(self.ops) - first if count is None else count
        return int(_lib.load().cgd_plan_num_launches(self.handle, first, count))

    def __del__(self):
        try:
            if self.handle is not None:
                _lib.load().cgd_plan_destroy(self.handle)
        except Exception:
            pass


# ---------------------------------------------------------------------- weight packing
@dataclass
class ConvW:
    """Packed weights of one conv / linear layer (forward and dgrad orientations)."""
    fwd: Buf
    fwd_npad: int
    bwd: Optional[Buf]
    bwd_npad: int
    bias: Optional[Buf]
    cin_pad: int
    cout: int
    taps: int


def _npad(n):
    return _round_up(n, 16) if n < 64 else _round_up(n, 64)


def pack_conv(plan: Plan, w: th.Tensor, bias: Optional[th.Tensor], *, need_bwd=True, cin_pad=None, name="w") -> ConvW:
    """w: [Cout, Cin, kh, kw] (kh=kw in {1,3}) or [Cout, Cin] / [Cout, Cin, 1].  Input channels are zero-padded to a
    multiple of 64 (TMA K-slices are 64 channels), output rows to the tile width."""
    w = w.detach().float()
    if w.dim() == 3:
        w = w[..., None]
    if w.dim() == 2:
        w = w[..., None, None]
    cout, cin, kh, kw = w.shape
    taps = kh * kw
    assert taps in (1, 9)
    cin_p = cin_pad or _round_up(cin, 64)
    cout_p64 = _round_up(cout, 64)
    # forward: Wp[co, tap*cin_p + ci]
    wf = th.zeros(_npad(cout), taps, cin_p)
    wf[:cout, :, :cin] = w.permute(0, 2, 3, 1).reshape(cout, taps, cin)
    fwd = plan.const(wf.reshape(_npad(cout), taps * cin_p), "h", name + ".fwd")
    bwd, bnp = None, 0
    if need_bwd:
        # dgrad: Wd[ci, tap'*cout_p + co] = w[co, ci, 2-ky', 2-kx'] (taps flipped), K = taps * cout_p
        bnp = _npad(cin)
        wb = th.zeros(bnp, taps, cout_p64)
        wflip = th.flip(w, dims=(2, 3)) if taps == 9 else w
        wb[:cin, :, :cout] = wflip.permute(1, 2, 3, 0).reshape(cin, taps, cout)
        bwd = plan.const(wb.reshape(bnp, taps * cout_p64), "h", name + ".bwd")
    b = plan.const(bias.float(), "f", name + ".bias") if bias is not None else None
    return ConvW(fwd, _npad(cout), bwd, bnp, b, cin_p, cout, taps)
