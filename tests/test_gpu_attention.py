"""GPU: softmax attention (head dim 64; 128 / 192 / 256 for the 128x128 checkpoint's four heads: csrc/attention_wide.cu) forward and
input-gradient -- the single-tile tensor-core kernels (T <= 64: csrc/attention_small.cu), the flash kernels (csrc/attention_mma.cu)
and the batched-GEMM path (T % 256 == 0) -- against a plain PyTorch
fp32 reference of [3P] QKVAttentionLegacy / QKVAttention / nn.MultiheadAttention's core (SURVEY.md K4, K14)."""
import math

import pytest
import torch as th

from clip_guided_diffusion_b200.plan import Act, Plan

pytestmark = pytest.mark.gpu

CASES = [  # nbatch, heads, T, legacy
    (16, 12, 50, False),   # ViT-B/32 over 16 cutouts
    (1, 16, 64, True),     # UNet 8x8 level
    (2, 2, 5, False),      # tiny ViT of the step tests
    (3, 4, 33, True),
    (2, 3, 64, False),
    (2, 4, 100, True),     # > 64: flash kernels
    (1, 2, 197, False),    # ViT-B/16 token count
    (1, 4, 256, True),     # UNet 16x16 level
    (1, 8, 1024, True),    # UNet 32x32 level
    (1, 2, 300, False),    # ragged last tile
    (2, 16, 577, False),   # ViT-L/14@336px token count (24 x 24 patches + class token): nine full tiles and one row
    # head dims of the 128x128 checkpoint (num_heads = 4): 32x32 level 512 / 4, 16x16 level 768 / 4, 8x8 level 1024 / 4
    (1, 4, 1024, True, 128),
    (1, 4, 256, True, 192),
    (1, 4, 64, True, 256),
    (2, 2, 100, True, 128),    # ragged last tile, two images
    (2, 3, 37, False, 192),    # single ragged tile, [q.. | k.. | v..] order
    (1, 2, 130, False, 256),   # three tiles, the last with 2 rows
]


def _case_id(c):
    return f"b{c[0]}_h{c[1]}_t{c[2]}_{'legacy' if c[3] else 'new'}" + (f"_d{c[4]}" if len(c) > 4 else "")


def _split(qkv, heads, legacy):
    B, T, C3 = qkv.shape
    C = C3 // 3
    d = C // heads
    if legacy:  # per head [q | k | v]
        x = qkv.view(B, T, heads, 3, d)
        return x[:, :, :, 0], x[:, :, :, 1], x[:, :, :, 2]
    x = qkv.view(B, T, 3, heads, d)
    return x[:, :, 0], x[:, :, 1], x[:, :, 2]


def _ref(qkv, heads, legacy):
    q, k, v = _split(qkv, heads, legacy)  # [B, T, h, d]
    w = th.einsum("bthd,bshd->bhts", q, k) / math.sqrt(q.shape[-1])
    p = th.softmax(w, dim=-1)
    o = th.einsum("bhts,bshd->bthd", p, v)
    return o.reshape(qkv.shape[0], qkv.shape[1], -1)


# id "tcgen05_gemms" kept stable across the port: the batched-GEMM formulation, now on the wgmma conv kernel
@pytest.mark.parametrize("tc", [False, True], ids=["flash", "tcgen05_gemms"])
@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_attention_fwd_bwd(case, tc):
    B, heads, T, legacy = case[:4]
    d = case[4] if len(case) > 4 else 64
    if tc and (T % 256 != 0 or d != 64):
        pytest.skip("the batched-GEMM path needs T % 256 == 0 and head dim 64")
    C = heads * d
    th.manual_seed(0)
    plan = Plan()
    plan.tc_attention = tc  # False: flash kernels (attention_small.cu / attention_mma.cu); True: batched wgmma GEMMs
    qkv = Act(plan.new(B * T * 3 * C, "h", "qkv"), 0, 1, 1, B * T, 3 * C, 3 * C)
    out = plan.attention(qkv, heads, T, B, legacy_order=legacy, name="attn")
    do = Act(plan.new(B * T * C, "h", "do"), 0, 1, 1, B * T, C, C)
    plan._grads[out.key()] = do
    plan.mark("bwd")
    plan.backward()
    plan.finalize("cuda")
    qv = plan.view(qkv.buf, (B, T, 3 * C))
    qv.copy_(th.randn(B, T, 3 * C) * 1.2)
    dv = plan.view(do.buf, (B, T, C)).normal_()
    plan.run()
    th.cuda.synchronize()
    xg = qv.float().clone().requires_grad_()
    ref = _ref(xg, heads, legacy)
    (gref,) = th.autograd.grad((ref * dv.float()).sum(), xg)
    got = plan.view(out.buf, (B, T, C)).float()
    err = float((got - ref.detach()).abs().max() / ref.detach().abs().max())
    # fp16 operands / fp16 P (like the reference's fp16 attention weights), fp32 accumulate and softmax
    assert th.isfinite(got).all() and err < 4e-3, f"fwd rel-to-max {err:.3e}"
    dq = plan.view(plan.grad_of(qkv).buf, (B, T, 3 * C)).float()
    err = float((dq - gref).abs().max() / gref.abs().max())
    assert th.isfinite(dq).all() and err < 6e-3, f"bwd rel-to-max {err:.3e}"
