"""GPU: the CLIP ModifiedResNet tower (rn.py) on the device -- a shallow tower op by op, the published RN50 / RN101 towers as a
whole, and a guided step with an RN tower, each against the fp32 oracle (oracle/clip_rn.py)."""
import os

import pytest
import torch as th

pytestmark = pytest.mark.gpu


def test_rn_tower_matches_oracle_on_device():
    from clip_guided_diffusion_b200 import rn as prn
    from clip_guided_diffusion_b200 import weights as pw
    from oracle import clip_rn as orn
    from tests.plan_interp import Interp
    n = 4
    cfg = prn.RNConfig(layers=(1, 2, 1, 1), output_dim=128, input_resolution=224, width=64)
    sd = pw.seeded_rn_state_dict(cfg, seed=3)
    oracle = orn.ModifiedResNet(orn.RNConfig(layers=(1, 2, 1, 1), output_dim=128, input_resolution=224, width=64)).eval()
    oracle.load_state_dict({k[len("visual."):]: v for k, v in sd.items()}, strict=False)
    tower = prn.RNB200(cfg, sd, n_images=n, device="cuda")
    g = th.Generator().manual_seed(1)
    img = th.randn(n, 3, 224, 224, generator=g)
    got = tower.encode_patches(Interp._patchify(img, 2, cfg.kpad).cuda().half()).float().cpu()
    xi = img.clone().requires_grad_()
    ref = oracle(xi)
    assert float((got - ref.detach()).norm() / ref.detach().norm()) < 3e-2
    d_emb = th.randn(n, cfg.output_dim, generator=g)
    dp = tower.backward_patches(d_emb.cuda()).float().cpu()
    (g_ref,) = th.autograd.grad((ref * d_emb).sum(), xi)
    d_img = Interp._unpatchify(dp, 2, 224)
    cos = float(th.nn.functional.cosine_similarity(d_img.flatten(), g_ref.flatten(), dim=0))
    assert cos > 0.99, cos


@pytest.mark.parametrize("name", ["RN50", "RN101", "RN50x4", "RN50x16"])
def test_published_rn_towers_vs_oracle_on_device(name):
    """the towers the reference lists (cgd/clip_util.py:17) and its own test uses (RN50, test.py:139-143) at their published depth /
    width / embedding size: forward and input gradient of the whole tower vs the fp32 oracle (oracle/clip_rn.py)"""
    from clip_guided_diffusion_b200 import rn as prn
    from clip_guided_diffusion_b200 import weights as pw
    from oracle import clip_rn as orn
    from tests.plan_interp import Interp
    n = 2 if name in ("RN50", "RN101") else 1  # the wide towers (288 / 384 px, zero-padded 80 / 96-wide layers): one image bounds the CPU oracle
    cfg = prn.RN_CONFIGS[name]
    sd = pw.seeded_rn_state_dict(cfg, seed=3)
    oracle = orn.ModifiedResNet(orn.RNConfig(layers=tuple(cfg.layers), output_dim=cfg.output_dim, input_resolution=cfg.input_resolution,
                                             width=cfg.width)).eval()
    oracle.load_state_dict({k[len("visual."):]: v for k, v in sd.items()}, strict=False)
    tower = prn.RNB200(cfg, sd, n_images=n, device="cuda")
    g = th.Generator().manual_seed(1)
    img = th.randn(n, 3, cfg.input_resolution, cfg.input_resolution, generator=g)
    got = tower.encode_patches(Interp._patchify(img, 2, cfg.kpad).cuda().half()).float().cpu()
    xi = img.clone().requires_grad_()
    ref = oracle(xi)
    assert got.shape == ref.shape == (n, cfg.output_dim)
    assert float((got - ref.detach()).norm() / ref.detach().norm()) < 3e-2
    d_emb = th.randn(n, cfg.output_dim, generator=g)
    dp = tower.backward_patches(d_emb.cuda()).float().cpu()
    (g_ref,) = th.autograd.grad((ref * d_emb).sum(), xi)
    d_img = Interp._unpatchify(dp, 2, cfg.input_resolution)
    cos = float(th.nn.functional.cosine_similarity(d_img.flatten(), g_ref.flatten(), dim=0))
    assert cos > 0.99, cos


@pytest.mark.parametrize("rn_width", [64, 80])  # 80: RN50x4's width, zero-padded to the 64-channel K slice layer by layer
def test_step_with_rn_tower_vs_oracle_and_ops(rn_width):
    from tests.gpu_harness import compare_ops
    from tests.step_parity import build_tiny, compare, engine_step, make_inputs, oracle_step
    ctx = build_tiny("cuda", image=64, use_graph=True, B=2, cutn=3, tower="rn", rn_width=rn_width)
    x, y, noise, nseed, coords = make_inputs(ctx)
    o = oracle_step(ctx, "ddim", x, 14, y, nseed, coords, fac_index=14)
    e = engine_step(ctx, "ddim", x, 14, y, noise, coords, fac_index=14, fused=True)
    res = compare(o, e)
    assert res["cos_g"] > 0.995 and res["rel_x0"] < 2e-2 and res["rel_sample"] < 2e-2, res
    n, failures = compare_ops(ctx["eng"].plan, [("cut_fwd", "sph"), ("vit_fwd", "vit_bwd"), ("vit_bwd", "vit_end")])
    assert not failures, failures[:10]
