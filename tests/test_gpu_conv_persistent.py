"""GPU: the persistent one-CTA conv kernel (csrc/conv_tc.cu `conv_tc_persistent_kernel`: min(tiles, SMs) CTAs, each walking its
tiles with the operand ring carried from tile to tile, epilogue through per-warp fp16 sub-tiles) against F.conv2d in fp32, at
geometries that stress what the persistent walk adds: CTAs with different tile counts (a ragged last round), partial edge tiles,
outputs and residuals that are channel slices of wider tensors, column tiles beyond the first, no bias."""
import pytest
import torch as th
import torch.nn.functional as F

from clip_guided_diffusion_b200.plan import Plan, pack_conv, conv_tile_count, pick_bn, pick_splits

pytestmark = pytest.mark.gpu

CASES = [
    # name, NB, H, W, Cin, Cout, taps, bias, res, out_ld (0: contiguous), res_ld
    # 2 x 100 rows of 128-pixel row segments: 200 tiles over 132 CTAs (68 CTAs take two), 28 of 128 pixels outside the image
    ("ragged_edge_3x3", 2, 100, 100, 128, 256, 9, True, False, 0, 0),
    ("ragged_edge_3x3_res_nobias", 2, 100, 100, 128, 256, 9, False, True, 0, 0),
    # output written as channels [0, 256) of a 512-wide concatenation, residual read from channels [128, 384) of a 384-wide tensor
    ("concat_out_res_slice", 1, 64, 96, 256, 256, 9, True, True, 512, 384),
    # 1x1 with three column tiles: the tile walk crosses column tiles inside one CTA
    ("conv1x1_three_col_tiles", 3, 48, 48, 192, 768, 1, True, True, 0, 0),
    # the dominant 256 x 256 layer: 512 tiles, 3.9 rounds
    ("dominant_256x256_res", 1, 256, 256, 256, 256, 9, True, True, 0, 0),
    # Cout not a multiple of 64: the last column tile is partly padding
    ("cout_200_partial_col_tile", 1, 80, 80, 128, 200, 9, True, True, 0, 0),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_persistent_conv_vs_fp32(case):
    name, NB, H, W, Cin, Cout, taps, has_b, has_r, out_ld, res_ld = case
    m_tiles, kblocks = conv_tile_count(NB, H, W), taps * Cin // 64
    npad = -(-Cout // 64) * 64
    assert pick_splits(m_tiles, npad // pick_bn(npad, m_tiles, kblocks), kblocks, npad) == 1, "case must take the one-CTA path"
    th.manual_seed(0)
    k = 3 if taps == 9 else 1
    w = th.randn(Cout, Cin, k, k) * (taps * Cin) ** -0.5
    b = th.randn(Cout) * 0.1 if has_b else None
    plan = Plan()
    cw = pack_conv(plan, w, b, need_bwd=False, name=name)
    x = plan.act(NB, H, W, Cin, "x")
    res_full = plan.act(NB, H, W, res_ld or Cout, "res") if has_r else None
    r0 = (res_ld - Cout) // 2 if res_ld else 0
    res = res_full.cslice(r0, r0 + Cout) if has_r else None
    out_full = plan.act(NB, H, W, out_ld or Cout, "out")
    out = out_full.cslice(0, Cout)
    plan.conv(x, cw, res=res, out=out, name=name)
    plan.finalize("cuda")
    xv = plan.view(x.buf, (NB, H, W, Cin)).normal_()
    rfull = plan.view(res_full.buf, (NB, H, W, res_full.ld)).normal_() if has_r else None
    ofull = plan.view(out_full.buf, (NB, H, W, out_full.ld))
    ofull.fill_(7.0)
    plan.run()
    th.cuda.synchronize()
    ref = F.conv2d(xv.float().permute(0, 3, 1, 2), w.cuda(), b.cuda() if has_b else None, padding=1 if taps == 9 else 0).permute(0, 2, 3, 1)
    if has_r:
        ref = ref + rfull[..., r0:r0 + Cout].float()
    got = ofull[..., :Cout].float()
    err = float((got - ref).abs().max() / ref.abs().max())
    assert th.isfinite(got).all() and err < 3e-3, f"{name}: rel-to-max err {err:.3e}"
    if out_ld:
        assert bool((ofull[..., Cout:] == 7.0).all()), f"{name}: channels beyond the output slice were written"
