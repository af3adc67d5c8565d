"""GPU: GroupNorm(32) + SiLU + scale/shift forward and input-gradient -- the single-launch cluster kernels
(csrc/norm_fused.cu), the persistent grid kernels (csrc/norm_grid.cu, csrc/norm_grid2.cu) and the two-pass kernels (csrc/norm.cu) --
against a plain PyTorch fp32 reference of the same op ([3P] GroupNorm32 -> SiLU -> conv input, ResBlock out_layers with
use_scale_shift_norm; SURVEY.md K5, K6) and against each other, over every (HW, C) the 256x256 / 512x512 UNets produce at the levels
the fused kernel covers.  In `grid` mode the cases lie on both sides of the HW * C = 2^23 threshold of the backward (for example
65536 x 512 and 16384 x 512 against 4096 x 512), so both persistent engines run: the ring kernels for every forward and the smaller
backward passes, the direct-load kernel for the larger backward passes."""
import pytest
import torch as th
import torch.nn.functional as F

from clip_guided_diffusion_b200.plan import Plan, gn_fused_cluster

pytestmark = pytest.mark.gpu

CASES = [
    # N, HW, C, emb, silu
    (1, 64, 1024, True, True),
    (1, 64, 2048, False, True),
    (2, 256, 1024, True, True),
    (1, 256, 1536, False, False),
    (1, 1024, 512, True, True),
    (3, 1024, 1024, False, True),
    (1, 4096, 512, True, True),
    (1, 4096, 256, False, True),
    (1, 4096, 768, True, True),
    (1, 16384, 256, True, True),
    (1, 16384, 512, False, True),
    (1, 16384, 768, False, True),   # backward slab too large -> two-pass backward, fused forward
    (1, 900, 256, True, True),      # ragged pixel count
    (1, 65536, 256, True, True),    # persistent grid kernel (or two-pass)
    (1, 65536, 512, False, True),   # 33 M elements: the direct-load backward engine (norm_grid2.cu)
    (2, 4096, 192, True, True),     # C = 192: groups straddle the 8-channel vectors (64x64 checkpoint widths)
    (3, 1024, 64, False, True),
    # widths of the 128x128 checkpoint: 24 / 40 / 56 channels per group = 3 / 5 / 7 16-byte vectors per pixel per CTA in the fused kernels
    (1, 256, 768, True, True),
    (1, 64, 768, False, False),
    (1, 1024, 1280, True, True),
    (1, 256, 1792, True, True),
    (1, 64, 1792, False, True),
]


def _ref(x, gamma, beta, emb, silu, eps=1e-5):
    N, HW, C = x.shape
    h = F.group_norm(x.permute(0, 2, 1).float(), 32, gamma, beta, eps).permute(0, 2, 1)
    if emb is not None:
        h = h * (1 + emb[:, None, :C]) + emb[:, None, C:]
    return F.silu(h) if silu else h


@pytest.mark.parametrize("fused", ["auto", "grid", "twopass"])
@pytest.mark.parametrize("case", CASES, ids=[f"n{c[0]}_hw{c[1]}_c{c[2]}{'_emb' if c[3] else ''}{'' if c[4] else '_nosilu'}" for c in CASES])
def test_group_norm_fwd_bwd(case, fused):
    N, HW, C, has_emb, silu = case
    th.manual_seed(0)
    plan = Plan()
    plan.fused_gn = fused == "auto"      # cluster kernel where the slab fits, else the persistent grid kernel
    plan.grid_gn = fused != "twopass"
    gamma = 1 + 0.2 * th.randn(C)
    beta = 0.1 * th.randn(C)
    emb = 0.3 * th.randn(N, 2 * C) if has_emb else None
    gb, bb = plan.const(gamma, "f", "gamma"), plan.const(beta, "f", "beta")
    eb = plan.const(emb, "f", "emb") if has_emb else None
    x = plan.act(N, 1, HW, C, "x")
    y1 = plan.group_norm(x, gb, bb, emb=(eb, 0) if has_emb else None, silu=silu, name="gn1")
    y2 = plan.group_norm(x, gb, bb, emb=None, silu=True, name="gn2")  # second consumer: its backward accumulates into dx
    dy1, dy2 = plan.act(N, 1, HW, C, "dy1"), plan.act(N, 1, HW, C, "dy2")
    plan._grads[y1.key()] = dy1
    plan._grads[y2.key()] = dy2
    plan.mark("bwd")
    plan.backward()
    plan.finalize("cuda")
    codes = [op.tag for op in plan.ops]
    n_fused = sum(1 for op in plan.ops if op.code in (33, 34))
    n_grid = sum(1 for op in plan.ops if op.code in (35, 36))
    if fused == "auto" and gn_fused_cluster(N, HW, C, 16):
        assert n_fused >= 2, codes
    if fused == "grid":
        assert n_fused == 0 and n_grid == 4, codes
    if fused == "twopass":
        assert n_fused == 0 and n_grid == 0
    xv = plan.view(x.buf, (N, HW, C))
    xv.copy_(th.randn(N, HW, C) * 1.5 + 0.3 * th.randn(N, 1, C))
    d1 = plan.view(dy1.buf, (N, HW, C)).normal_()
    d2 = plan.view(dy2.buf, (N, HW, C)).normal_()
    plan.run()
    th.cuda.synchronize()
    xg = xv.float().clone().requires_grad_()
    ge, be = gamma.cuda(), beta.cuda()
    r1 = _ref(xg, ge, be, emb.cuda() if has_emb else None, silu)
    r2 = _ref(xg, ge, be, None, True)
    (gref,) = th.autograd.grad((r1 * d1.float()).sum() + (r2 * d2.float()).sum(), xg)
    for yy, rr, nm in ((y1, r1, "y1"), (y2, r2, "y2")):
        got = plan.view(yy.buf, (N, HW, C)).float()
        err = float((got - rr.detach()).abs().max() / rr.detach().abs().max())
        # tolerance: fp16 output rounding (2^-11 relative) of values up to ~6 -> 1.5e-3 of max
        assert th.isfinite(got).all() and err < 2e-3, f"{nm} fused={fused}: rel-to-max {err:.3e}"
    dx = plan.view(plan.grad_of(x).buf, (N, HW, C)).float()
    err = float((dx - gref).abs().max() / gref.abs().max())
    # two fp16 roundings (first dx, accumulated dx)
    assert th.isfinite(dx).all() and err < 3e-3, f"dx fused={fused}: rel-to-max {err:.3e}"


def test_all_paths_agree_on_statistics():
    """Cluster, grid and two-pass kernels must hand the same (mean, rstd) to the backward."""
    N, HW, C = 2, 1024, 512
    outs = []
    for mode in ("fused", "grid", "twopass"):
        th.manual_seed(1)
        plan = Plan()
        plan.fused_gn = mode == "fused"
        plan.grid_gn = mode == "grid"
        gb, bb = plan.const(th.ones(C), "f", "g"), plan.const(th.zeros(C), "f", "b")
        x = plan.act(N, 1, HW, C, "x")
        plan.group_norm(x, gb, bb, silu=False, name="gn")
        plan.finalize("cuda")
        plan.view(x.buf, (N, HW, C)).copy_(th.randn(N, HW, C) * 2 + 1)
        plan.run()
        th.cuda.synchronize()
        st = [b for b in plan.bufs if b.name == "gn_stats"][0]
        outs.append(plan.view(st, (N, 32, 2)).clone())
    assert th.allclose(outs[0], outs[2], rtol=2e-5, atol=2e-6), float((outs[0] - outs[2]).abs().max())
    assert th.allclose(outs[1], outs[2], rtol=2e-5, atol=2e-6), float((outs[1] - outs[2]).abs().max())
