"""The LPIPS trunk's ReLU, 2x2 max-pool and fused tap kernels, the ResizeRight (lanczos3) cutout kernels and FILL, one launch at a time,
at every signature the shipped plans make (tests/op_plan_table.py) plus hand-written edge cases, against float64 references; and the
towers' and encoders' attention / glue launches that no other table lists, through tests/test_gpu_unet_kernels.py's harness.

As in tests/test_gpu_kernels_fullshape.py: `gpu` cases run the native kernels at production shapes; `cpu-*` cases run reduced shapes
through tests/plan_interp.py, which checks the references on a machine without a GPU.  The references never call interpreter code.
Outputs are poisoned (NaN or a sentinel) before the launch, so an element a kernel does not write fails."""
import math

import numpy as np
import pytest
import torch as th
import torch.nn.functional as F

from clip_guided_diffusion_b200 import resize_right as rr
from clip_guided_diffusion_b200.guidance import CLIP_MEAN, CLIP_STD
from clip_guided_diffusion_b200.plan import Plan
from tests.kernel_check import D64, U, cases, check, run, ulp16
from tests.op_plan_table import UNET_OTHER_PLAN, rows


def _id(sig):
    return "-".join(str(int(v)) for v in sig)


def specials16(n, g, scale=1.0):
    """fp16 values: randn * scale, led by +-0, subnormals, +-65504 and +-inf"""
    x = th.randn(n, generator=g) * scale
    sp = th.tensor([0.0, -0.0, 2.0 ** -24, -2.0 ** -24, 2.0 ** -20, -2.0 ** -15, 65504.0, -65504.0, math.inf, -math.inf, 6e-5, -6e-5])
    k = min(n, sp.numel())
    x[:k] = sp[:k]
    return x.half()


# ---------------------------------------------------------------------------------------------------------------- ReLU
RELU_GPU = {_id(s): s[0] for s in sorted({(r[0],) for r in rows("RELU_FWD") + rows("RELU_BWD")})}
RELU_GPU.update({"hand-8": 8, "hand-1048584": 1048584})
RELU_CPU = {"8": 8, "4104": 4104}


@pytest.mark.parametrize("device,n", cases(RELU_GPU, RELU_CPU))
def test_relu(device, n):
    """forward y = max(x, 0): bitwise.  Backward (ATen's threshold_backward on the output): dx = dy where y > 0, else 0 -- bitwise when
    storing; with flags 2, fp16(fp32(old) + that), the kernel's one IEEE fp32 add and one rounding."""
    g = th.Generator().manual_seed(n)
    x = specials16(n, g)
    dy = specials16(n, g, 100.0).flip(0)
    old = (th.randn(n, generator=g) * 1000).half()
    plan = Plan()
    bx, by, bdy, bdx, bdx2 = (plan.new(n, "h") for _ in range(5))
    plan.emit("RELU_FWD", i=[n], p=[(bx, 0), (by, 0)])
    plan.emit("RELU_BWD", i=[n], p=[(bdy, 0), (by, 0), (bdx, 0)])
    plan.emit("RELU_BWD", flags=2, i=[n], p=[(bdy, 0), (by, 0), (bdx2, 0)])
    rd = run(plan, device, [(bx, x), (by, th.full((n,), math.nan).half()), (bdy, dy), (bdx, th.full((n,), math.nan).half()), (bdx2, old)])
    x64 = x.to(D64)
    y = rd(by)
    assert th.equal(y.to(D64), th.where(x64 > 0, x64, th.zeros(()))), "relu_fwd"
    r = th.where(y.to(D64) > 0, dy.to(D64), th.zeros((), dtype=D64))
    assert th.equal(rd(bdx).to(D64), r), "relu_bwd"
    assert th.equal(rd(bdx2), (old.float() + r.float()).half()), "relu_bwd accumulate"


# ---------------------------------------------------------------------------------------------------------------- max-pool
MP_GPU = {_id(s): s for s in sorted(set(rows("MAXPOOL2_FWD")) | set(rows("MAXPOOL2_BWD")))}
MP_GPU.update({"hand-3-6-10-8": (3, 6, 10, 8)})
MP_CPU = {"1-8-8-16": (1, 8, 8, 16), "2-4-6-8": (2, 4, 6, 8)}


def first_max_rule(x, dy):
    """[N, H, W, C] -> (max, dx): dy goes to the first position in row-major window order holding the maximum, 0 to the others"""
    N, H, W, C = x.shape
    win = x.view(N, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(N, H // 2, W // 2, 4, C)
    m = win.amax(3)
    first = (win == m[:, :, :, None]).int().argmax(3)  # argmax of a 0/1 mask returns its first 1
    dx = th.zeros_like(win)
    dx.scatter_(3, first[:, :, :, None], dy[:, :, :, None])
    return m, dx.view(N, H // 2, W // 2, 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(N, H, W, C)


@pytest.mark.parametrize("device,case", cases(MP_GPU, MP_CPU))
def test_maxpool2(device, case):
    """2x2 / stride 2 max-pool on pixel-major fp16: forward bitwise; backward bitwise against ATen's rule (first maximum in row-major
    window order gets dy, the other three positions are written with 0).  Half the windows hold exact ties at positive values, as
    post-ReLU fp16 activations often do."""
    N, H, W, C = case
    g = th.Generator().manual_seed(N * H * C)
    tied = (th.randint(0, 3, (N, H, W, C), generator=g).float() * 0.5)  # 0, 0.5, 1: ties at 0 and at positive values
    x = th.where(th.rand(N, H, W, C, generator=g) < 0.5, tied, th.relu(th.randn(N, H, W, C, generator=g))).half()
    x.view(-1)[:4] = th.tensor([-1.0, -2.0, -1.0, -3.0]).half()  # a negative maximum
    dy = (th.randn(N, H // 2, W // 2, C, generator=g) + 0.25).half()
    plan = Plan()
    bx, by, bdy, bdx = plan.new(x.numel(), "h"), plan.new(dy.numel(), "h"), plan.new(dy.numel(), "h"), plan.new(x.numel(), "h")
    plan.emit("MAXPOOL2_FWD", i=[N, H, W, C], p=[(bx, 0), (by, 0)])
    plan.emit("MAXPOOL2_BWD", i=[N, H, W, C], p=[(bdy, 0), (bx, 0), (bdx, 0)])
    rd = run(plan, device, [(bx, x), (by, th.full((dy.numel(),), math.nan).half()), (bdy, dy), (bdx, th.full((x.numel(),), math.nan).half())])
    m, dx = first_max_rule(x.float(), dy.float())  # fp16 values are exact in fp32; max and the routing are exact
    assert th.equal(rd(by, dy.shape).float(), m), "maxpool2_fwd"
    got = rd(bdx, x.shape).float()
    bad = got != dx
    assert not bool(bad.any()), f"maxpool2_bwd: {int(bad.sum())} of {bad.numel()} elements differ from the first-maximum rule"
    if device == "cpu":  # the rule is ATen's: float64 autograd of max_pool2d routes the same way
        x64 = x.to(D64).permute(0, 3, 1, 2).requires_grad_()
        (ga,) = th.autograd.grad(F.max_pool2d(x64, 2, 2), x64, dy.to(D64).permute(0, 3, 1, 2))
        assert th.equal(ga.permute(0, 2, 3, 1), dx.to(D64))


# ---------------------------------------------------------------------------------------------------------------- LPIPS tap
TAP_GPU = {_id(s): s for s in rows("LPIPS_TAP")}
TAP_GPU.update({f"hand-{B}-{HW}-{C}-{Bt}": (B, HW, C, Bt) for B, HW, C, Bt in (
    (2, 65536, 128, 1), (2, 65536, 128, 2), (4, 16384, 256, 4), (4, 4096, 512, 1), (2, 262144, 64, 2), (4, 1024, 512, 4), (1, 37, 64, 1))})
TAP_CPU = {f"{B}-{HW}-{C}-{Bt}": (B, HW, C, Bt) for B, HW, C, Bt in ((1, 64, 64, 1), (2, 48, 128, 2), (4, 16, 512, 1), (2, 9, 256, 2))}


def ref_tap(f, tn, w):
    """per image sum_p sum_c w_c (f_c / (||f|| + 1e-10) - tn_c)^2 / HW and its float64 autograd gradient (vector_norm's backward is 0 at
    a zero vector, so an all-zero pixel gets the limit g / 1e-10 instead of 0 * inf)"""
    f = f.to(D64).requires_grad_()
    xh = f / (th.linalg.vector_norm(f, dim=-1, keepdim=True) + 1e-10)
    per = ((xh - tn.to(D64)) ** 2 * w.to(D64)).sum(-1).mean(-1)
    (gf,) = th.autograd.grad(per.sum(), f)
    return per.detach(), gf


@pytest.mark.parametrize("device,case", cases(TAP_GPU, TAP_CPU))
def test_lpips_tap(device, case):
    """fused LPIPS tap: df = gscale * d loss / d f, fp16, saturated at +-60000 where the float64 value exceeds it (an all-zero pixel),
    loss_part += per-image loss, fp32 with atomics"""
    B, HW, C, Bt = case
    g = th.Generator().manual_seed(B * HW + C)
    f = th.relu(th.randn(B, HW, C, generator=g) * 2).half()
    zero = [(0, 0), (B - 1, HW - 1), (B // 2, HW // 2)]  # pixels whose channels are all zero after ReLU
    for b, p in zero:
        f[b, p] = 0
    t = th.relu(th.randn(Bt, HW, C, generator=g))
    tn = (t / (t.norm(dim=-1, keepdim=True) + 1e-10)).half()
    w = th.rand(C, generator=g) * 0.2
    gscale = 64.0 * HW  # gscale / HW = 64: df of order 1 .. 100
    plan = Plan()
    bf, bt, bw, bd, bl = plan.new(f.numel(), "h"), plan.new(tn.numel(), "h"), plan.new(C, "f"), plan.new(f.numel(), "h"), plan.new(B, "f")
    plan.emit("LPIPS_TAP", i=[B, HW, C, Bt], f=[gscale], p=[(bf, 0), (bt, 0), (bw, 0), (bd, 0), (bl, 0)])
    rd = run(plan, device, [(bf, f), (bt, tn), (bw, w), (bd, th.full((f.numel(),), math.nan).half()), (bl, th.full((B,), 5.0))])
    per, gf = ref_tap(f, tn.expand(B, HW, C), w)
    ref = gf * gscale
    got = rd(bd, (B, HW, C)).to(D64)
    # saturated where |float64| > 60000: exactly +-60000 with the float64 sign (only the all-zero pixels get there)
    sat = ref.abs() > 60000
    assert th.equal(got[sat], 60000 * th.sign(ref[sat])), "lpips_tap: unsaturated or wrong-signed value at an all-zero pixel"
    assert all(bool(sat[b, p].any()) for b, p in zero) and int(sat.sum()) <= sum(int((tn.expand(B, HW, C)[b, p] != 0).sum()) for b, p in zero)
    # elsewhere: one fp16 ulp plus an fp32 floor.  ss = sum f^2 and gx = sum_c g_c f_c are warp reductions -- <= 16 serial fmas per lane
    # and a 5-level butterfly: 21 roundings -- then sqrt, the reciprocal, the differences and products: 32 u of the magnitude
    # sc (|g| / n + |f| sum_c |g_c f_c| / (n^2 r)) with |g| = 2 w (|xh| + |tn|) the magnitude of g.
    f64, tn64, w64 = f.to(D64), tn.expand(B, HW, C).to(D64), w.to(D64)
    r = f64.norm(dim=-1, keepdim=True)
    n = r + 1e-10
    gm = 2 * w64 * (f64 / n + tn64.abs())
    mag = 64.0 * (gm / n + f64 * (gm * f64).sum(-1, keepdim=True) / (n * n * r.clamp(min=1e-30)))
    tol = ulp16(ref) + 32 * U * mag
    check("lpips_tap df", got.masked_fill(sat, 0), ref.masked_fill(sat, 0), tol.masked_fill(sat, 0))
    # loss: per pixel <= 16 serial fmas and a butterfly; per warp serial over its pixels; the warps' partials in any order (atomics):
    # depth 21 + pixels per warp + warps per image, times the sum of the (non-negative) terms, plus the old value 5.0
    warps = min(-(-B * HW // 8), 132 * 8) * 8
    depth = 24 + -(-B * HW // warps) + min(warps, HW)
    d = f64 / n - tn64
    lmag = (w64 * 2 * d.abs() * (f64 / n) * 16).sum(-1).mean(-1)  # d's own rounding error, 16 u of |xh|, through d^2
    check("lpips_tap loss", rd(bl), 5.0 + per, depth * U * (5.0 + per) + U * lmag)


def test_tap_reference_matches_oracle_lpips():
    """ref_tap on one tap equals oracle/lpips.py's per-layer term (normalize_tensor, squared difference, 1x1 lin conv, spatial mean)"""
    from oracle.lpips import normalize_tensor
    g = th.Generator().manual_seed(0)
    B, H, W, C = 2, 5, 7, 64
    f0 = th.relu(th.randn(B, C, H, W, generator=g, dtype=D64))
    f1 = th.relu(th.randn(B, C, H, W, generator=g, dtype=D64))
    lin = th.rand(1, C, 1, 1, generator=g, dtype=D64)
    want = F.conv2d((normalize_tensor(f0) - normalize_tensor(f1)) ** 2, lin).mean([2, 3]).view(B)
    tn = normalize_tensor(f1).permute(0, 2, 3, 1).reshape(B, H * W, C)
    per, _ = ref_tap(f0.permute(0, 2, 3, 1).reshape(B, H * W, C), tn, lin.view(C))
    assert th.allclose(per, want, rtol=1e-12, atol=0)


# ---------------------------------------------------------------------------------------------------------------- ResizeRight cutouts
RR_GPU = {_id(s): s[:7] for s in rows("CUTOUTS_RR_FWD")}
RR_GPU.update({  # (B, H, W, cutn, cs, P, Kpad): P 14 / 2 with padded columns, B = 2, S up to 576 at cs 224 (T 16)
    "hand-B2-576-P16": (2, 576, 576, 8, 224, 16, 768), "hand-B2-300-P14-kpad": (2, 300, 300, 6, 224, 14, 640),
    "hand-B2-100-P2-kpad": (2, 100, 100, 6, 64, 2, 16), "hand-up-48-P32": (1, 48, 48, 5, 224, 32, 3072)})
RR_CPU = {"B1-40-P4-kpad": (1, 40, 40, 5, 16, 4, 64), "B2-12-up-P4": (2, 12, 12, 4, 16, 4, 48), "B2-30-P2-kpad": (2, 30, 30, 4, 12, 2, 16)}


def rr_windows(side, cs, cutn, seed):
    """square crops inside the image: the largest at the origin and at the bottom-right border, one at S == cs when it fits (T = 1),
    the rest of seeded sizes in [min(cs, side), side] -- different S (so different T) in one launch"""
    g = np.random.default_rng(seed)
    mn = min(cs, side)
    out = [(0, 0, side), (side - mn, side - mn, mn), (side - (side + mn) // 2, side - (side + mn) // 2, (side + mn) // 2)]
    while len(out) < cutn:
        s = int(g.integers(mn, side + 1))
        out.append((int(g.integers(0, side - s + 1)), int(g.integers(0, side - s + 1)), s))
    return out[:cutn]


def rr_matrix(S, cs):
    """float64 [cs, S] resampling matrix of the host tables: A[o, left[o] + i] = w[o, i] for i < T inside the crop"""
    left, wt, T = rr.tables(S, cs)
    A = th.zeros(cs, S, dtype=D64)
    for i in range(T):
        idx = left.long() + i
        ok = (idx >= 0) & (idx < S)
        A[th.arange(cs)[ok], idx[ok]] += wt[ok, i].to(D64)
    return A


def ref_rr(x, coords, cs, A):
    """[cutn * B, 3, cs, cs] float64: every crop resampled by A_k . crop . A_k^T"""
    return th.cat([A[k] @ x[:, :, oy:oy + s, ox:ox + s] @ A[k].t() for k, (ox, oy, s) in enumerate(coords)])


@pytest.mark.parametrize("device,case", cases(RR_GPU, RR_CPU))
def test_cutouts_rr(device, case):
    """CUTOUTS_RR_FWD against ((resize(crop) + 1) / 2 - mean) / std rounded once to fp16, zero in the padded columns; CUTOUTS_RR_BWD
    against the exact transpose (float64 autograd of that forward) times scale.  Weight slots at index >= T are NaN and the inverse
    ranges of rows past S are empty: a kernel that reads outside a field of view, or an inverse range that is not exact, fails."""
    from tests.test_gpu_kernels_fullshape import clip_normalize, from_patches, to_patches
    B, H, W, cutn, cs, P, kpad = case
    coords = rr_windows(H, cs, cutn, seed=H + cs)
    g = th.Generator().manual_seed(H * cutn)
    x = (th.randn(B, 3, H, W, generator=g) * 0.7).float()
    G2 = (cs // P) ** 2
    dpatch = (th.randn(cutn * B, G2, kpad, generator=g) * 0.01).half()
    left, wt = th.zeros(cutn, cs, dtype=th.int32), th.full((cutn, cs, rr.T_MAX), math.nan)
    taps, inv = th.zeros(cutn, dtype=th.int32), th.tensor([1, 0], dtype=th.int32).repeat(cutn, H, 1)
    for k, (_, _, S) in enumerate(coords):
        l, w, T = rr.tables(S, cs)
        left[k], taps[k] = l, T
        wt[k, :, :T] = w[:, :T]
        inv[k, :S] = rr.inverse_ranges(l, T, S)
    assert H <= cs or len(set(taps.tolist())) > 1  # crops larger than cs: per-cutout tap counts differ in one launch
    scale = 0.25
    plan = Plan()
    bx, bc, bo, bd, bg = plan.new(x.numel(), "f"), plan.new(cutn * 3, "i32"), plan.new(cutn * B * G2 * kpad, "h"), plan.new(dpatch.numel(), "h"), \
        plan.new(x.numel(), "f")
    bl, bw, bt, bi = plan.new(left.numel(), "i32"), plan.new(wt.numel(), "f"), plan.new(cutn, "i32"), plan.new(inv.numel(), "i32")
    geo = [B, H, W, cutn, cs, P, kpad]
    plan.emit("CUTOUTS_RR_FWD", i=geo, f=[*CLIP_MEAN, *CLIP_STD], p=[(bx, 0), (bc, 0), (bo, 0), (bl, 0), (bw, 0), (bt, 0)])
    plan.emit("CUTOUTS_RR_BWD", i=geo + [H], f=[0, 0, 0, *CLIP_STD, scale], p=[(bd, 0), (bc, 0), (bg, 0), (bl, 0), (bw, 0), (bi, 0)])
    rd = run(plan, device, [(bx, x), (bc, th.tensor(coords, dtype=th.int32)), (bo, th.full((cutn * B * G2 * kpad,), 7.0).half()), (bd, dpatch),
                            (bg, th.full((x.numel(),), math.nan)), (bl, left), (bw, wt), (bt, taps), (bi, inv)])
    A = [rr_matrix(S, cs) for _, _, S in coords]
    Tmax = int(taps.max())
    # forward: a row pass of T fmas and a column pass of T fmas, then (acc + 1) * 0.5 - mean and / std: (2 T + 8) u of the magnitude
    x64 = x.to(D64)
    ref = to_patches(clip_normalize((ref_rr(x64, coords, cs, A) + 1) / 2), P, kpad)
    Aabs = [a.abs() for a in A]
    sd = th.tensor(CLIP_STD, dtype=D64).view(1, 3, 1, 1)
    mag = to_patches(((ref_rr(x64.abs(), coords, cs, Aabs) + 1) / 2 + th.tensor(CLIP_MEAN, dtype=D64).view(1, 3, 1, 1)) / sd, P, kpad)
    got = rd(bo, (cutn * B, G2, kpad))
    check("cutouts_rr_fwd", got, ref, ulp16(ref) + (2 * Tmax + 8) * U * mag)
    assert bool((got[:, :, 3 * P * P:] == 0).all()), "patch-vector padding not zeroed"
    # backward: per pixel a gather over the outputs of every crop holding it (<= T per axis per crop), two fmas deep each, then two
    # products: (2 T cutn_at_pixel + 6) u of the same sum on absolute values
    xr = th.zeros(B, 3, H, W, dtype=D64, requires_grad=True)
    dimg = from_patches(dpatch.to(D64), P, cs)
    (gref,) = th.autograd.grad((clip_normalize((ref_rr(xr, coords, cs, A) + 1) / 2) * dimg).sum(), xr)
    (gmag,) = th.autograd.grad((clip_normalize((ref_rr(xr, coords, cs, Aabs) + 1) / 2) * dimg.abs()).sum(), xr)
    gmag = gmag.abs()
    check("cutouts_rr_bwd", rd(bg, x.shape), gref * scale, (2 * Tmax * cutn + 6) * U * gmag * scale + 1e-30)


RR_GOLDEN = ("down_237_224", "down_64_56", "down_60_32", "down_73_32", "same_32", "up_16_56", "up_20_32")


@pytest.mark.parametrize("name", RR_GOLDEN)
def test_rr_reference_matches_the_reference_golden(name):
    """rr_matrix's resampling and its transpose against tests/golden/resize_right_golden.npz, written by the reference's own
    ResizeRight (fp32): forward y and the autograd gradient g of sum(y * w), down, same and up"""
    import os
    d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resize_right_golden.npz"))
    S, O, _ = (int(v) for v in d[name + "_shape"])
    A = rr_matrix(S, O)
    x = th.from_numpy(d[name + "_x"]).to(D64).requires_grad_()
    y = A @ x @ A.t()
    assert th.allclose(y.detach(), th.from_numpy(d[name + "_y"]).to(D64), rtol=1e-5, atol=2e-6)
    (gx,) = th.autograd.grad((y * th.from_numpy(d[name + "_w"]).to(D64)).sum(), x)
    assert th.allclose(gx, th.from_numpy(d[name + "_g"]).to(D64), rtol=1e-5, atol=2e-6)


# ---------------------------------------------------------------------------------------------------------------- FILL
FILL_GPU = {_id(s): s[0] for s in rows("FILL")}
FILL_GPU.update({"hand-1000003": 1000003})
FILL_CPU = {"1": 1, "77": 77}


@pytest.mark.parametrize("device,n", cases(FILL_GPU, FILL_CPU))
def test_fill(device, n):
    """n fp32 elements set to the value, bitwise; the element after them keeps its sentinel"""
    plan = Plan()
    b = plan.new(n + 1, "f")
    plan.emit("FILL", i=[n], f=[-0.375], p=[(b, 0)])
    rd = run(plan, device, [(b, th.full((n + 1,), math.nan).index_fill_(0, th.tensor([n]), 9.0))])
    got = rd(b)
    assert th.equal(got[:n], th.full((n,), -0.375)) and float(got[n]) == 9.0


# ---------------------------------------------------------------------------------------------------------------- towers' UNet-kernel launches
@pytest.mark.gpu
@pytest.mark.parametrize("sig", UNET_OTHER_PLAN, ids=[repr(s) for s in UNET_OTHER_PLAN])
def test_tower_unet_kernel_launches(sig, monkeypatch):
    """attention, POOL2 / UP2, ADD / COPY launches of the RN / ViT / text towers and image-prompt encoders at their batch sizes, on the
    bit-exact / float64 harness of tests/test_gpu_unet_kernels.py (dispatched as the load_clip table's rows are)"""
    from tests.test_gpu_clip_autograd import test_tower_other_launches
    test_tower_other_launches(sig, monkeypatch)
