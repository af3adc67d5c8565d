"""GPU: the TMA epilogue of the persistent conv kernel (csrc/conv_tc.cu `conv_tc_persistent_kernel`): the residual is TMA-loaded
into a swizzled fp16 staging tile during the K loop, the output is TMA-stored from it, and the TMA unit clips rows outside the
image and columns >= Cout.  Each case runs one CONV op with an explicit tile width BN and compares it with F.conv2d in fp32:
residual and QuickGELU' (CONV flags 4) at every BN >= 64, outputs and residuals that are channel slices (a non-zero channel
offset), guard channels around the output slice that must keep their sentinel, multi-image tiles clipped in N, a partial last
column box, column tiles wholly beyond Cout, BN 32 / 16 (narrower boxes and swizzles), fewer tiles than SMs, and more than 8
rounds of tiles per CTA."""
import pytest
import torch as th
import torch.nn.functional as F

from clip_guided_diffusion_b200 import _lib

pytestmark = pytest.mark.gpu

SENTINEL = 7.0

CASES = [
    # name, NB, H, W, Cin, Cout, taps, BN, bias, res ("add" / "gelu" / None), out (ld, c0), res (ld, c0)
    ("bn64_res", 1, 64, 64, 128, 256, 9, 64, True, "add", None, None),
    ("bn128_res", 1, 64, 64, 128, 256, 9, 128, True, "add", None, None),
    ("bn192_res", 1, 64, 64, 128, 384, 9, 192, True, "add", None, None),
    ("bn256_res", 1, 64, 64, 128, 256, 9, 256, True, "add", None, None),
    ("bn64_gelu", 1, 64, 64, 128, 256, 9, 64, False, "gelu", None, None),
    ("bn128_gelu", 1, 64, 64, 128, 256, 9, 128, False, "gelu", None, None),
    ("bn192_gelu", 1, 64, 64, 128, 384, 9, 192, False, "gelu", None, None),
    ("bn256_gelu", 2, 48, 40, 64, 256, 1, 256, False, "gelu", None, None),
    # output into the second half of a concatenation, with guard channels on both sides; residual from a channel slice
    ("concat_second_half", 1, 64, 96, 256, 256, 9, 256, True, "add", (576, 256), (384, 64)),
    ("concat_second_half_bn128", 2, 40, 40, 128, 128, 9, 128, False, "add", (264, 128), (200, 8)),
    # multi-image tiles: 8x8 images (TN = 2), 4x4 (TN = 8), the last pixel tile clipped in N; 16x16 with NB > 1
    ("img8x8_tn2", 5, 8, 8, 128, 256, 9, 256, True, "add", (320, 32), None),
    ("img4x4_tn8", 11, 4, 4, 64, 128, 9, 64, True, "add", None, (136, 8)),
    ("img16x16_nb3", 3, 16, 16, 192, 192, 9, 192, False, "gelu", None, None),
    # Cout = 200: the last 64-channel box of the last column tile is partly beyond Cout
    ("cout200_bn256", 1, 80, 80, 128, 200, 9, 256, True, "add", (208, 0), None),
    ("cout200_bn128", 2, 30, 50, 64, 200, 1, 128, True, "add", None, None),
    # 8 tiles on 132 SMs; 512 pixel tiles x 3 column tiles = 12 rounds of one K-block each
    ("few_tiles", 1, 32, 32, 64, 64, 9, 64, True, "add", None, None),
    ("rounds_12_kblock_1", 1, 256, 256, 64, 192, 1, 64, True, "add", (200, 8), (192, 0)),
    ("rounds_12_no_res", 1, 256, 256, 64, 192, 1, 64, True, None, None, None),
    # narrow tiles: a 32-channel box with the 64-byte swizzle, a 16-channel box with the 32-byte swizzle
    ("bn32_res", 2, 40, 40, 128, 32, 9, 32, True, "add", (48, 8), (40, 8)),
    ("bn16_res", 2, 40, 40, 128, 16, 9, 16, True, "add", (32, 16), None),
    # Npad = 256 for Cout = 64 at BN 64: three column tiles lie wholly beyond Cout and store nothing
    ("col_tiles_beyond_cout", 1, 64, 64, 128, 64, 9, 64, True, "add", (72, 8), None),
]
NPAD = {"col_tiles_beyond_cout": 256}  # padded weight rows when not the next multiple of BN


def _conv_op(x, wp, bias, res, out, NB, H, W, Cin, Cout, npad, taps, bn, flags):
    rs = res.stride()[:3] if res is not None else (0, 0, 0)
    _lib.run_op("CONV", flags=flags, i=[NB, H, W, Cin, Cout, npad, taps, *x.stride()[:3], *out.stride()[:3], *rs, bn, 1, 0, 1, 0, 0, 0, 0],
                p=[x, wp, bias, res, out], what="conv")


def _qgelu_grad(u):
    s = th.sigmoid(1.702 * u)
    return s * (1 + 1.702 * u * (1 - s))


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_tma_epilogue_vs_fp32(case):
    name, NB, H, W, Cin, Cout, taps, bn, has_b, mode, out_sl, res_sl = case
    assert not (has_b and mode == "gelu"), "CONV flags 4 takes no bias"
    th.manual_seed(0)
    dev = "cuda"
    k = 3 if taps == 9 else 1
    npad = NPAD.get(name, -(-Cout // bn) * bn)
    w = th.randn(Cout, Cin, k, k) * (taps * Cin) ** -0.5
    wp = th.zeros(npad, taps, Cin)
    wp[:Cout] = w.permute(0, 2, 3, 1).reshape(Cout, taps, Cin)
    wp = wp.reshape(npad, taps * Cin).half().to(dev)
    b = (th.randn(Cout) * 0.1).to(dev) if has_b else None
    x = th.randn(NB, H, W, Cin, device=dev).half()
    old, oc0 = out_sl or (Cout, 0)
    out_full = th.full((NB, H, W, old), SENTINEL, device=dev, dtype=th.half)
    out = out_full[..., oc0:oc0 + Cout]
    res_full, res, rc0 = None, None, 0
    if mode is not None:
        rld, rc0 = res_sl or (Cout, 0)
        res_full = th.randn(NB, H, W, rld, device=dev).half()
        res = res_full[..., rc0:rc0 + Cout]
    _conv_op(x, wp, b, res, out, NB, H, W, Cin, Cout, npad, taps, bn, 4 if mode == "gelu" else 0)
    th.cuda.synchronize()

    wr = wp.float().reshape(npad, taps, Cin)[:Cout].reshape(Cout, k, k, Cin).permute(0, 3, 1, 2)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wr, b, padding=k // 2).permute(0, 2, 3, 1)
    if mode == "add":
        ref = ref + res.float()
    elif mode == "gelu":
        ref = ref * _qgelu_grad(res.float())
    got = out.float()
    err = float((got - ref).abs().max() / ref.abs().max())
    assert th.isfinite(got).all() and err < 3e-3, f"{name}: rel-to-max err {err:.3e}"
    guard = th.ones(old, dtype=th.bool, device=dev)
    guard[oc0:oc0 + Cout] = False
    assert bool((out_full[..., guard] == SENTINEL).all()), f"{name}: channels outside the output slice were written"
