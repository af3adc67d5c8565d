"""CPU tests of the host-side plan builder: the UNet / ViT op lists (graph walk, weight packing, strides,
hand-scheduled backward) are executed with the test-only PyTorch interpreter and compared with the oracle's
forward and autograd input gradients.  No CUDA involved; the same op lists run through libcgd_b200 on the GPU."""
import numpy as np
import pytest
import torch as th

from clip_guided_diffusion_b200 import unet as pu
from clip_guided_diffusion_b200 import vit as pv
from oracle.unet import UNetModel, tiny_config, seeded_init_
from oracle.clip_vit import CLIPVisualOnly, ViTConfig as OViTConfig
from tests.plan_interp import Interp


def rel(a, b):
    return float((a - b).norm() / (b.norm() + 1e-12))


def cos(a, b):
    return float(th.nn.functional.cosine_similarity(a.flatten(), b.flatten(), dim=0))


def _prod_cfg(ocfg):
    return pu.UNetConfig(image_size=ocfg.image_size, model_channels=ocfg.model_channels, num_res_blocks=ocfg.num_res_blocks,
                         channel_mult=ocfg.channel_mult, attention_resolutions=ocfg.attention_resolutions,
                         num_heads=ocfg.num_heads, num_head_channels=ocfg.num_head_channels, class_cond=ocfg.class_cond,
                         num_classes=ocfg.num_classes, use_new_attention_order=ocfg.use_new_attention_order)


@pytest.mark.parametrize("new_order,cond", [(False, True), (True, False)])
def test_unet_plan_matches_oracle(new_order, cond):
    th.manual_seed(0)
    ocfg = tiny_config(image_size=32, model_channels=64, channel_mult=(1, 2), num_res_blocks=1, attention_resolutions=(16,),
                       class_cond=cond, use_new_attention_order=new_order)
    oracle = seeded_init_(UNetModel(ocfg)).eval()
    B = 2
    net = pu.UNetB200(_prod_cfg(ocfg), oracle.state_dict(), batch=B, device="cpu", seed_scale=64.0)
    it = Interp(net.plan)
    x = th.randn(B, 3, 32, 32)
    t = th.tensor([7.0, 431.0])
    y = th.tensor([3, 8]) if cond else None
    net.set_inputs(x, t, y)
    it.run_range("unet_emb", "unet_bwd")
    xo = x.clone().requires_grad_()
    ref = oracle(xo, t, y)
    out = net.out_view.clone()
    assert rel(out, ref.detach()) < 2e-2, rel(out, ref.detach())
    d_out = th.randn(B, 6, 32, 32) * 0.1
    (gref,) = th.autograd.grad((ref * d_out).sum(), xo)
    sv = net.seed_view
    sv[:, :, :6] = (d_out * net.seed_scale).reshape(B, 6, -1).permute(0, 2, 1).half()
    it.run_range("unet_bwd", "unet_end")
    g = net.dx_view / net.seed_scale
    assert cos(g, gref) > 0.999 and rel(g, gref) < 4e-2, (cos(g, gref), rel(g, gref))


@pytest.mark.parametrize("heads,mult", [(1, (1, 2)), (1, (1, 2, 3))])
def test_unet_plan_with_num_heads_wide_head_dims(heads, mult):
    """the 128x128 checkpoint's attention (data/diffusion_model_flags.py: num_heads = 4, num_head_channels unset -> head dim =
    channels / num_heads = 128 / 192 / 256; csrc/attention_wide.cu): here 128 and 192 channels in one head, legacy qkv order"""
    import dataclasses
    th.manual_seed(0)
    size = 16 * 2 ** (len(mult) - 1)
    ocfg = tiny_config(image_size=size, model_channels=64, channel_mult=mult, num_res_blocks=1, attention_resolutions=(size // 2, size // 4))
    ocfg = dataclasses.replace(ocfg, num_heads=heads, num_head_channels=-1)
    oracle = seeded_init_(UNetModel(ocfg)).eval()
    B = 1
    net = pu.UNetB200(_prod_cfg(ocfg), oracle.state_dict(), batch=B, device="cpu", seed_scale=64.0)
    from clip_guided_diffusion_b200._lib import OP
    dims = sorted({op.i[3] for op in net.plan.ops if op.code == OP["ATTN_FWD"]})
    assert dims == [64 * m for m in mult[1:]], dims
    it = Interp(net.plan)
    x = th.randn(B, 3, size, size)
    t = th.tensor([431.0])
    y = th.tensor([3])
    net.set_inputs(x, t, y)
    it.run_range("unet_emb", "unet_bwd")
    xo = x.clone().requires_grad_()
    ref = oracle(xo, t, y)
    assert rel(net.out_view.clone(), ref.detach()) < 2e-2
    d_out = th.randn(B, 6, size, size) * 0.1
    (gref,) = th.autograd.grad((ref * d_out).sum(), xo)
    net.seed_view[:, :, :6] = (d_out * net.seed_scale).reshape(B, 6, -1).permute(0, 2, 1).half()
    it.run_range("unet_bwd", "unet_end")
    g = net.dx_view / net.seed_scale
    assert cos(g, gref) > 0.999 and rel(g, gref) < 4e-2, (cos(g, gref), rel(g, gref))


def test_vit_plan_matches_oracle():
    th.manual_seed(0)
    ocfg = OViTConfig(64, 32, 128, 2, 64)
    oracle = seeded_init_(CLIPVisualOnly(ocfg), seed=5).eval()
    n = 3
    cfg = pv.ViTConfig(64, 32, 128, 2, 64)
    assert pv.vit_config_from_state_dict(oracle.state_dict()) == cfg
    net = pv.ViTB200(cfg, oracle.state_dict(), n_images=n, device="cpu")
    it = Interp(net.plan)
    img = th.randn(n, 3, 64, 64, requires_grad=True)
    ref = oracle.encode_image(img)
    net.plan.view(net.patches, (n, 4, cfg.kpad)).copy_(Interp._patchify(img.detach(), 32, cfg.kpad))
    it.run_range("vit_fwd", "vit_bwd")
    emb = net.plan.view(net.embeds, (n, 64)).clone()
    assert rel(emb, ref.detach()) < 2e-2, rel(emb, ref.detach())
    d_emb = th.randn(n, 64)
    (gref,) = th.autograd.grad((ref * d_emb).sum(), img)
    net.plan.view(net.d_embeds, (n, 64)).copy_(d_emb)
    it.run_range("vit_bwd", "vit_end")
    g = Interp._unpatchify(net.plan.view(net.d_patches, (n, 4, cfg.kpad)).float(), 32, 64)
    assert cos(g, gref) > 0.999 and rel(g, gref) < 4e-2, (cos(g, gref), rel(g, gref))


def test_param_inventories_match_oracle():
    from clip_guided_diffusion_b200 import weights as pw
    from oracle.unet import config_for as oconfig_for
    from oracle.clip_vit import VIT_CONFIGS as OV
    for size, cond in [(64, True), (128, True), (256, True), (256, False), (512, True)]:
        with th.device("meta"):
            m = UNetModel(oconfig_for(size, cond))
        ref = {k: tuple(v.shape) for k, v in m.state_dict().items()}
        assert pw.unet_param_shapes(pu.config_for(size, cond)) == ref
    for name in ("ViT-B/32", "ViT-B/16", "ViT-L/14", "ViT-L/14@336px"):
        with th.device("meta"):
            m = CLIPVisualOnly(OV[name])
        ref = {k: tuple(v.shape) for k, v in m.state_dict().items()}
        assert pw.vit_param_shapes(pv.VIT_CONFIGS[name]) == ref


def test_cluster_split_picks_are_eligible():
    """plan.pick_cluster_split only returns configurations the C side accepts (csrc/conv_tc.cu: the CONV i23 check of conv_tc_prepare)
    and that fit one wave of clusters (one cluster of S CTAs per 128-pixel x BN tile); every K split is non-empty."""
    from clip_guided_diffusion_b200 import plan as P
    seen = 0
    for (NB, H, W) in [(1, 8, 8), (2, 8, 8), (1, 16, 16), (1, 32, 32), (1, 64, 64), (1, 1, 800), (1, 1, 3152), (4, 16, 16),
                       (1, 72, 72), (1, 36, 36), (2, 18, 18), (1, 9, 9), (1, 1, 82), (1, 12, 12), (1, 1, 145)]:
        m_tiles = P.conv_tile_count(NB, H, W)
        for cin in (128, 192, 256, 320, 512, 640, 768, 1024, 1280, 1536, 1792, 2048, 2304, 2560, 3072):
            for cout in (128, 192, 256, 320, 512, 640, 768, 1024, 1280, 1536, 1792, 2048, 2560, 3072, 7680):
                for taps in (1, 9):
                    kb = taps * cin // 64
                    npad = P._npad(cout)
                    pick = P.pick_cluster_split(m_tiles, npad, kb, cout)
                    if pick is None:
                        continue
                    bn, S, kb_per_cta = pick
                    seen += 1
                    assert bn in (64, 128, 192, 256) and npad % bn == 0 and 2 <= S <= 8
                    assert bn % S == 0 and (bn // S) % 16 == 0 and cout % 8 == 0
                    kps = -(-kb // S)
                    assert (S - 1) * kps < kb and kps >= 3            # no empty split, a pipeline worth filling
                    assert m_tiles * (npad // bn) <= P.cluster_capacity(bn, S)
                    assert kb_per_cta == kps
    assert seen > 50
    assert P.pick_cluster_split(2, 1024, 144, 1023) is None  # Cout % 8 != 0: the vector epilogue cannot store it


def test_groupnorm_from_conv_epilogue_statistics():
    """opt-in path (CGD_GN_EPI_STATS / plan.gn_epi_stats): the conv reduces its fp16 output to per-(128-pixel tile, octet) sums
    (CONV flags 2) and GN_APPLY_EPI normalises in one trip; forward and the backward that consumes its (mean, rstd)."""
    import torch.nn.functional as F
    from clip_guided_diffusion_b200 import plan as P
    from tests.plan_interp import Interp
    th.manual_seed(0)
    N, H, W, Cin, C = 2, 32, 32, 64, 256
    w = th.randn(C, Cin, 3, 3) * (9 * Cin) ** -0.5
    b = th.randn(C) * 0.1
    gamma_t, beta_t, emb_t = 1 + 0.1 * th.randn(C), 0.1 * th.randn(C), 0.2 * th.randn(N * 2 * C)
    outs = {}
    for epi in (False, True):
        plan = P.Plan()
        plan.gn_epi_stats, plan.fused_gn, plan.grid_gn = epi, False, True
        cw = P.pack_conv(plan, w, b, need_bwd=True, name="w")
        x = plan.act(N, H, W, Cin, "x")
        res = plan.act(N, H, W, C, "res")
        h = plan.conv(x, cw, res=res, name="c")
        gamma, beta, emb = plan.const(gamma_t, "f", "g"), plan.const(beta_t, "f", "b"), plan.const(emb_t, "f", "e")
        y = plan.group_norm(h, gamma, beta, emb=(emb, 0), silu=True, name="gn")
        dy = plan.act(N, H, W, C, "dy")
        plan._grads[y.key()] = dy
        plan.mark("bwd")
        plan.backward()
        plan.finalize("cpu")
        codes = [o.code for o in plan.ops]
        assert (P.OP["GN_APPLY_EPI"] in codes) == epi and (P.OP["GN_FWD_GRID"] in codes) == (not epi)
        conv_op = plan.ops[0]
        assert bool(conv_op.flags & 2) == epi
        g = th.Generator().manual_seed(1)
        plan.view(x.buf, (N, H, W, Cin)).copy_(th.randn(N, H, W, Cin, generator=g))
        plan.view(res.buf, (N, H, W, C)).copy_(th.randn(N, H, W, C, generator=g))
        plan.view(dy.buf, (N, H, W, C)).copy_(th.randn(N, H, W, C, generator=g))
        Interp(plan).run()
        outs[epi] = (plan.view(y.buf, (N, H, W, C)).float().clone(), plan.view(plan.grad_of(x).buf, (N, H, W, Cin)).float().clone(),
                     plan.view(h.buf, (N, H, W, C)).float().clone())
    y0, dx0, h0 = outs[False]
    y1, dx1, h1 = outs[True]
    assert th.equal(h0, h1)
    assert float((y1 - y0).abs().max()) < 4e-3 * float(y0.abs().max())  # same statistics up to summation order, fp16 outputs
    assert float((dx1 - dx0).norm() / dx0.norm()) < 2e-3
    # and against torch directly: GroupNorm of the stored fp16 conv output, scale-shift, SiLU
    e = emb_t.view(N, 2 * C)
    ref = F.group_norm(h1.permute(0, 3, 1, 2), 32, gamma_t, beta_t, eps=1e-5) * (1 + e[:, :C, None, None]) + e[:, C:, None, None]
    ref = F.silu(ref).permute(0, 2, 3, 1)
    assert float((y1 - ref).abs().max()) < 4e-3 * float(ref.abs().max())


def test_engine_model_load_state_dict_repacks_in_place():
    """cgd/script_util.py:317: `model.load_state_dict(checkpoint)` on the engine's UNet handle re-packs the checkpoint into the
    kernel layouts in place: the arena must equal, byte for byte, the arena of an engine CONSTRUCTED from that checkpoint."""
    import pytest
    from clip_guided_diffusion_b200 import weights as pw
    from tests.step_parity import build_tiny
    a = build_tiny("cpu", B=1, cutn=2, image=32)["eng"]
    b = build_tiny("cpu", B=1, cutn=2, image=32)["eng"]
    sd2 = pw.seeded_state_dict(pw.unet_param_shapes(a.unet.cfg), seed=4321)  # other weights, same architecture (upstream keys)
    before = a.plan.arena.clone()
    res = a.model.load_state_dict(sd2)
    assert not res.missing_keys and not res.unexpected_keys
    assert not th.equal(a.plan.arena, before)
    b.model.load_state_dict(sd2)
    assert th.equal(a.plan.arena, b.plan.arena)
    # and equal to construction from sd2: compare the forward through the interpreter against the oracle loaded with sd2
    from oracle.unet import UNetModel
    from tests.plan_interp import Interp
    from tests.step_parity import tiny_config
    ocfg = tiny_config(image_size=32, model_channels=64, channel_mult=(1, 2), num_res_blocks=1, attention_resolutions=(16,), class_cond=True,
                       use_new_attention_order=False)
    ounet = UNetModel(ocfg).eval()
    ounet.load_state_dict(sd2)
    th.manual_seed(0)
    x, t, y = th.randn(1, 3, 32, 32), th.tensor([500.0]), th.tensor([3])
    a.unet.set_inputs(x, t, y)
    it = Interp(a.plan)
    it.run_range("unet_emb", "unet_bwd")
    got = a.unet.out_view.float()
    ref = ounet(x, t, y).detach()
    assert float((got - ref).norm() / ref.norm()) < 2e-2
    with pytest.raises(RuntimeError, match="missing"):
        a.model.load_state_dict({k: v for k, v in sd2.items() if k != "out.2.weight"})
    with pytest.raises(RuntimeError, match="unexpected"):
        a.model.load_state_dict({**sd2, "bogus.weight": th.zeros(1)})
    assert a.model.load_state_dict({**sd2, "bogus.weight": th.zeros(1)}, strict=False).unexpected_keys == ["bogus.weight"]
