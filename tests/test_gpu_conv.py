"""GPU: the wgmma implicit-GEMM conv / GEMM kernel (and its SIMT verification twin) against a plain PyTorch fp32
reference of the same op, across tile geometries, paddings, split-K, epilogues and output layouts."""
import pytest
import torch as th
import torch.nn.functional as F

from clip_guided_diffusion_b200.plan import Plan, pack_conv, Act

pytestmark = pytest.mark.gpu

CASES = [
    # name, NB, H, W, Cin, Cout, taps, bias, res
    ("conv3x3_64x64_c128", 1, 64, 64, 128, 128, 9, True, False),
    ("conv3x3_32x32_c256_res", 2, 32, 32, 256, 256, 9, True, True),
    ("conv3x3_16x16_c512_splitk", 1, 16, 16, 512, 512, 9, True, True),
    ("conv3x3_8x8_c1024_tn2", 2, 8, 8, 1024, 1024, 9, True, False),
    ("conv3x3_8x8_b1", 1, 8, 8, 512, 1024, 9, False, False),
    ("conv3x3_256w_c64", 1, 4, 256, 64, 64, 9, True, False),
    ("conv1x1_skip", 1, 32, 32, 512, 256, 1, True, False),
    ("conv3x3_c192", 1, 32, 32, 192, 384, 9, True, False),
    ("conv3x3_c576_bn192", 1, 16, 16, 384, 576, 9, True, True),
    ("conv3x3_rowseg_128w_c128_res", 1, 8, 128, 128, 256, 9, True, True),     # tile = one 128-pixel row segment (TW = 128, TH = 1)
    ("conv3x3_rowseg_256w_c256_b2", 2, 6, 256, 256, 256, 9, True, True),
    ("conv3x3_rowseg_192w_ragged", 1, 5, 192, 128, 128, 9, True, False),      # second tile of each row is half out of the image
    ("conv3x3_rowseg_c192_bn192", 1, 3, 128, 192, 192, 9, False, True),
    ("linear_m800_qkv", 1, 1, 800, 768, 2304, 1, True, False),
    ("linear_m50", 1, 1, 50, 768, 768, 1, True, True),
    ("linear_k3072", 1, 1, 800, 3072, 768, 1, True, True),
    ("conv3x3_32x32_c512_cluster8", 1, 32, 32, 512, 512, 9, True, True),      # in-cluster split-K: 16 CTAs per tile (BN 256, S = 8)
    ("conv1x1_16x16_k3072", 1, 16, 16, 3072, 1024, 1, True, False),
    ("linear_k2304_m800", 1, 1, 800, 2304, 768, 1, False, True),              # BN 192, S = 4, ragged last pixel tile
    # the dominant layer of the benchmarked configuration: 31 % of the 256x256 UNet's FLOPs (M = 65536, N = 256, K = 2304), the
    # shape bench.py's `roofline` line times -- 512 tiles of 128 pixels, with and without the ResBlock residual
    ("conv3x3_256x256_c256_dominant", 1, 256, 256, 256, 256, 9, True, False),
    ("conv3x3_256x256_c256_dominant_res", 1, 256, 256, 256, 256, 9, True, True),
    ("conv3x3_256x256_c512_to_256", 1, 256, 256, 512, 256, 9, True, False),      # output blocks at 256x256: K = 4608
    ("conv3x3_128x128_c256", 1, 128, 128, 256, 256, 9, True, True),
    # 8 x 8 images: the weight-streaming kernel (csrc/conv_narrow.cu, conv_small_kernel: 8 output channels per CTA, no split-K) -- the
    # deepest UNet level's 3x3 convs and attention 1x1s, forward and dgrad, with / without residual, two images
    ("conv3x3_8x8_c1024_res", 1, 8, 8, 1024, 1024, 9, True, True),
    ("conv1x1_8x8_qkv", 1, 8, 8, 1024, 3072, 1, True, False),
    ("conv1x1_8x8_proj_res_b2", 2, 8, 8, 1024, 1024, 1, True, True),
    ("conv1x1_8x8_k3072", 1, 8, 8, 3072, 1024, 1, True, False),
    ("conv3x3_8x8_c2048_to_1024", 1, 8, 8, 2048, 1024, 9, True, False),   # K too large for the slab: stays on the wgmma split-K path
    # widths of the 128x128 checkpoint (channel_mult 1, 1, 2, 3, 4: a 768-wide 16x16 level, 1280 / 1792-wide concatenations)
    ("conv3x3_16x16_c768_res", 1, 16, 16, 768, 768, 9, True, True),
    ("conv3x3_16x16_c1792_to_768", 1, 16, 16, 1792, 768, 9, True, False),
    ("conv3x3_32x32_c1280_to_512", 1, 32, 32, 1280, 512, 9, True, False),
    ("conv1x1_16x16_c768_qkv", 1, 16, 16, 768, 2304, 1, True, False),
    ("conv3x3_8x8_c1792_to_1024", 1, 8, 8, 1792, 1024, 9, True, False),
    # CLIP RN50x4 (288 px, width 80 zero-padded to 128; 320 / 640 / 2560-wide stages) and RN50x16 (384 px) shapes
    ("conv1x1_72x72_c128_to_320_res", 1, 72, 72, 128, 320, 1, True, True),
    ("conv3x3_144x144_c64_to_128", 1, 144, 144, 64, 128, 9, True, False),
    ("conv3x3_36x36_c192", 2, 36, 36, 192, 192, 9, True, False),
    ("conv1x1_9x9_c2560_to_640", 1, 9, 9, 2560, 640, 1, True, True),
    ("linear_m82_k2560_qkv", 1, 1, 82, 2560, 7680, 1, True, False),
]


def _ref_conv(x, w, b, res, taps):
    xf = x.float().permute(0, 3, 1, 2)
    y = F.conv2d(xf, w.float(), b.float() if b is not None else None, padding=1 if taps == 9 else 0)
    y = y.permute(0, 2, 3, 1)
    return y + res.float() if res is not None else y


# ids (kept stable across the port): tc1 = impl 2, the wgmma tile kernel for every layer with workspace split-K; tc2pair = impl 3, the
# same kernel for every layer with in-cluster split-K; tc2pair_ws_splitk = impl 3 with the in-cluster reduction switched off
@pytest.mark.parametrize("impl", [0, 1, 2, 3, 13], ids=["auto", "simt", "tc1", "tc2pair", "tc2pair_ws_splitk"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv_fwd_and_dgrad(case, impl):
    name, NB, H, W, Cin, Cout, taps, has_b, has_r = case
    cluster = impl != 13  # 13: impl 3 with the workspace split-K + reduce launch instead of the in-cluster reduction
    impl = 3 if impl == 13 else impl
    if impl == 1 and NB * H * W * Cout * taps * Cin > 3e10:
        pytest.skip("SIMT twin only on small cases")
    th.manual_seed(0)
    k = 3 if taps == 9 else 1
    w = th.randn(Cout, Cin, k, k) * (taps * Cin) ** -0.5
    b = th.randn(Cout) * 0.1 if has_b else None
    plan = Plan(conv_impl=impl)
    plan.cluster_splitk = cluster
    cw = pack_conv(plan, w, b, need_bwd=True, name=name)
    x = plan.act(NB, H, W, Cin, "x")
    res = plan.act(NB, H, W, Cout, "res") if has_r else None
    y = plan.conv(x, cw, res=res, name=name)
    dy = plan.act(NB, H, W, Cout, "dy")
    plan._grads[y.key()] = dy
    plan.mark("bwd")
    plan.backward()
    plan.mark("end")
    plan.finalize("cuda")
    xv = plan.view(x.buf, (NB, H, W, Cin)).normal_()
    rv = plan.view(res.buf, (NB, H, W, Cout)).normal_() if has_r else None
    dyv = plan.view(dy.buf, (NB, H, W, Cout)).normal_()
    plan.run(0, plan.marks["bwd"])
    th.cuda.synchronize()
    ref = _ref_conv(xv, w.cuda(), b.cuda() if has_b else None, rv, taps)
    got = plan.view(y.buf, (NB, H, W, Cout)).float()
    err = float((got - ref).abs().max() / ref.abs().max())
    assert th.isfinite(got).all() and err < 3e-3, f"{name} fwd impl={impl}: rel-to-max err {err:.3e}, got_max {float(got.abs().max()):.3e} ref_max {float(ref.abs().max()):.3e}"
    # dgrad vs autograd of the reference
    plan.run(plan.marks["bwd"], plan.marks["end"] - plan.marks["bwd"])
    th.cuda.synchronize()
    xg = xv.float().clone().requires_grad_()
    yr = _ref_conv(xg, w.cuda(), None, None, taps)
    (gref,) = th.autograd.grad((yr * dyv.float()).sum(), xg)
    dx = plan.grad_of(x)
    gg = plan.view(dx.buf, (NB, H, W, Cin)).float()
    err = float((gg - gref).abs().max() / gref.abs().max())
    assert th.isfinite(gg).all() and err < 3e-3, f"{name} dgrad impl={impl}: rel-to-max err {err:.3e}"


@pytest.mark.parametrize("impl", [0, 1, 2, 3], ids=["auto", "simt", "tc1", "tc2pair"])
def test_conv_special_layouts(impl):
    """UNet head (fp32 NCHW out, 6 of 16 padded channels), stem dgrad (3 channels) and the ViT patch-embed geometry
    (49 tokens per image written at a row offset with a batch stride)."""
    th.manual_seed(1)
    plan = Plan(conv_impl=impl)
    B, H, W, C = 2, 16, 16, 128
    w = th.randn(6, C, 3, 3) * (9 * C) ** -0.5
    b = th.randn(6) * 0.1
    cw = pack_conv(plan, w, b, need_bwd=False, name="head")
    x = plan.act(B, H, W, C, "x")
    out = plan.new(B * 6 * H * W, "f", "out")
    plan._emit_conv(plan._ap(x), plan._strides(x), B, H, W, C, cw.fwd, cw.fwd_npad, 6, 9, cw.bias, None, None, (out, 0), (6 * H * W, W, 1),
                    out_f32=True, out_sc=H * W, tag="head")
    # patch-embed like: n images x 49 tokens, K=192, written to rows 1.. of a [n, 50, w] tensor
    n, G2, T, K, wd = 5, 49, 50, 192, 128
    wp = th.randn(wd, K) * K ** -0.5
    cp = pack_conv(plan, wp, None, need_bwd=False, name="patch")
    patches = plan.new(n * G2 * K, "h", "patches")
    tok = plan.new(n * T * wd, "h", "tok")
    plan._emit_conv((patches, 0), (G2 * K, G2 * K, K), n, 1, G2, K, cp.fwd, cp.fwd_npad, wd, 1, None, None, None, (tok, wd), (T * wd, T * wd, wd),
                    tag="patch")
    plan.finalize("cuda")
    xv = plan.view(x.buf, (B, H, W, C)).normal_()
    pvw = plan.view(patches, (n, G2, K)).normal_()
    plan.run()
    th.cuda.synchronize()
    ref = F.conv2d(xv.float().permute(0, 3, 1, 2), w.cuda(), b.cuda(), padding=1)
    got = plan.view(out, (B, 6, H, W))
    assert float((got - ref).abs().max() / ref.abs().max()) < 3e-3
    reft = pvw.float() @ wp.cuda().t()
    gott = plan.view(tok, (n, T, wd)).float()
    assert float((gott[:, 1:] - reft).abs().max() / reft.abs().max()) < 3e-3
    assert float(gott[:, 0].abs().max()) == 0.0  # cls rows untouched


@pytest.mark.parametrize("rows", [800, 200])
def test_quick_gelu_backward_fused_into_dgrad_epilogue(rows):
    """CLIP MLP: a = QuickGELU(u), y = c_proj(a).  The dgrad of c_proj multiplies its accumulator by QuickGELU'(u) in the epilogue
    (CONV flags 4: u arrives through the residual TMA path) and writes d u directly -- no d a tensor, no QGELU_BWD launch."""
    from clip_guided_diffusion_b200._lib import OP
    th.manual_seed(0)
    Cin, Cout = 3072, 768
    w = th.randn(Cout, Cin) * Cin ** -0.5
    plan = Plan()
    cw = pack_conv(plan, w, th.zeros(Cout), need_bwd=True, name="c_proj")
    u = plan.act(1, 1, rows, Cin, "u")
    a = plan.quick_gelu(u, "gelu")
    y = plan.conv(a, cw, name="c_proj")
    dy = plan.act(1, 1, rows, Cout, "dy")
    plan._grads[y.key()] = dy
    plan.backward()
    plan.finalize("cuda")
    codes = [op.code for op in plan.ops]
    assert OP["QGELU_BWD"] not in codes and any(op.code == OP["CONV"] and op.flags & 4 for op in plan.ops)
    uv = plan.view(u.buf, (rows, Cin)).normal_()
    dv = plan.view(dy.buf, (rows, Cout)).normal_()
    plan.run()
    th.cuda.synchronize()
    ug = uv.float().clone().requires_grad_()
    yr = (ug * th.sigmoid(1.702 * ug)) @ w.cuda().t()
    (gref,) = th.autograd.grad((yr * dv.float()).sum(), ug)
    got = plan.view(plan.grad_of(u).buf, (rows, Cin)).float()
    err = float((got - gref).abs().max() / gref.abs().max())
    assert th.isfinite(got).all() and err < 3e-3, err


@pytest.mark.parametrize("shape", [(1, 256, 256, 256, 6), (1, 256, 256, 256, 3), (2, 37, 45, 128, 6), (1, 64, 64, 192, 6)],
                         ids=["head_256x256", "stem_dgrad_256x256", "ragged_b2", "64px_c192"])
def test_narrow_conv_halo_kernel(shape):
    """3x3 conv with <= 8 output channels and an fp32 NCHW output (UNet head 256 -> 6, stem dgrad 256 -> 3): the halo-tile
    mma.sync kernel (csrc/conv_narrow.cu) against F.conv2d, including image borders that cut the 4 x 32 tiles."""
    NB, H, W, C, Cout = shape
    th.manual_seed(2)
    plan = Plan(conv_impl=0)
    w = th.randn(Cout, C, 3, 3) * (9 * C) ** -0.5
    b = th.randn(Cout) * 0.1
    cw = pack_conv(plan, w, b, need_bwd=False, name="head")
    x = plan.act(NB, H, W, C, "x")
    out = plan.new(NB * Cout * H * W, "f", "out")
    plan._emit_conv(plan._ap(x), plan._strides(x), NB, H, W, C, cw.fwd, cw.fwd_npad, Cout, 9, cw.bias, None, None, (out, 0), (Cout * H * W, W, 1),
                    out_f32=True, out_sc=H * W, tag="head")
    plan.finalize("cuda")
    xv = plan.view(x.buf, (NB, H, W, C)).normal_()
    plan.run()
    th.cuda.synchronize()
    ref = F.conv2d(xv.float().permute(0, 3, 1, 2), w.cuda().half().float(), b.cuda(), padding=1)
    got = plan.view(out, (NB, Cout, H, W))
    err = float((got - ref).abs().max() / ref.abs().max())
    assert th.isfinite(got).all() and err < 2e-3, err


def test_small_image_weight_streaming_kernel():
    """CGD_CONV_SMALL=1: 8 x 8 images take conv_small_kernel (csrc/conv_narrow.cu: a CTA per 8 output channels streaming its whole
    weight slab, TMA box per activation slice, mma.sync) instead of split-K wgmma tiles.  Opt-in (measured break-even); the switch
    is read once per process, so the 8 x 8 cases are re-run in a child process with it on."""
    import os, subprocess, sys
    env = dict(os.environ, CGD_CONV_SMALL="1")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_conv.py", "-q", "-x", "-m", "gpu", "-k", "8x8 and (auto or tc2pair) and not small_image",
                        "-p", "no:cacheprovider"], cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
