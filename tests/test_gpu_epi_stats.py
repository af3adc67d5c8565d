"""GPU: GroupNorm forward from conv-epilogue statistics (CONV flags 2 -> GN_APPLY_EPI; plan.gn_epi_stats / CGD_GN_EPI_STATS=1).
Interpreter-verified (tests/test_plan_cpu.py) and device-validated (round 2); the path itself stays opt-in because it measured no net
gain (DESIGN.md)."""
import os

import pytest
import torch as th
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("shape", [(1, 128, 128, 256, 256, True), (2, 64, 64, 128, 512, False), (1, 256, 256, 256, 256, True)],
                         ids=["128x128_c256_res", "b2_64x64_c512", "256x256_c256_res"])
def test_epilogue_statistics_groupnorm(shape):
    from clip_guided_diffusion_b200 import plan as P
    N, H, W, Cin, C, use_res = shape
    th.manual_seed(0)
    w = th.randn(C, Cin, 3, 3) * (9 * Cin) ** -0.5
    b = th.randn(C) * 0.1
    gamma_t, beta_t, emb_t = 1 + 0.1 * th.randn(C), 0.1 * th.randn(C), 0.2 * th.randn(N * 2 * C)
    outs = {}
    for epi in (False, True):
        plan = P.Plan()
        plan.gn_epi_stats, plan.fused_gn, plan.grid_gn = epi, False, True
        cw = P.pack_conv(plan, w, b, need_bwd=True, name="w")
        x = plan.act(N, H, W, Cin, "x")
        res = plan.act(N, H, W, C, "res") if use_res else None
        h = plan.conv(x, cw, res=res, name="c")
        gamma, beta, emb = plan.const(gamma_t, "f", "g"), plan.const(beta_t, "f", "b"), plan.const(emb_t, "f", "e")
        y = plan.group_norm(h, gamma, beta, emb=(emb, 0), silu=True, name="gn")
        dy = plan.act(N, H, W, C, "dy")
        plan._grads[y.key()] = dy
        plan.backward()
        plan.finalize("cuda")
        assert (P.OP["GN_APPLY_EPI"] in [o.code for o in plan.ops]) == epi
        g = th.Generator().manual_seed(1)
        plan.view(x.buf, (N, H, W, Cin)).copy_(th.randn(N, H, W, Cin, generator=g))
        if use_res:
            plan.view(res.buf, (N, H, W, C)).copy_(th.randn(N, H, W, C, generator=g))
        plan.view(dy.buf, (N, H, W, C)).copy_(th.randn(N, H, W, C, generator=g))
        plan.run()
        th.cuda.synchronize()
        outs[epi] = (plan.view(y.buf, (N, H, W, C)).float().cpu(), plan.view(plan.grad_of(x).buf, (N, H, W, Cin)).float().cpu(),
                     plan.view(h.buf, (N, H, W, C)).float().cpu())
    (y0, dx0, h0), (y1, dx1, h1) = outs[False], outs[True]
    assert th.equal(h0, h1)  # the STATS instantiation stores the same tile
    assert float((y1 - y0).abs().max()) < 4e-3 * float(y0.abs().max())
    assert float((dx1 - dx0).norm() / dx0.norm()) < 3e-3
    e = emb_t.view(N, 2 * C)
    ref = F.silu(F.group_norm(h1.permute(0, 3, 1, 2), 32, gamma_t, beta_t, eps=1e-5) * (1 + e[:, :C, None, None]) + e[:, C:, None, None]).permute(0, 2, 3, 1)
    assert float((y1 - ref).abs().max()) < 4e-3 * float(ref.abs().max())
