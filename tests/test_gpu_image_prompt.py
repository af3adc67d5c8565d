"""GPU: image prompts on the device -- the RESIZE_AXIS kernel against the oracle resampler and the reference's own ResizeRight
(tests/golden/image_prompt_golden.npz), ``encode_image_prompt`` against the fp32 oracle towers on the same cutouts, and
``clip_guided_diffusion(image_prompts=...)`` end to end with the loop's first cutout windows replayed by the oracle."""
import os

import numpy as np
import pytest
import torch as th

from clip_guided_diffusion_b200 import cgd
from clip_guided_diffusion_b200 import guidance as pg
from clip_guided_diffusion_b200 import image_prompt as pip
from clip_guided_diffusion_b200 import resize_right as rr
from clip_guided_diffusion_b200 import rn as prn
from clip_guided_diffusion_b200 import unet as pu
from clip_guided_diffusion_b200 import vit as pv
from clip_guided_diffusion_b200 import weights as pw
from oracle import resize_right as orr
from oracle.guidance import MakeCutouts as OMakeCutouts
from tests import image_prompt_oracle as oip

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "image_prompt_golden.npz"))


def _close(got, ref, tol=1e-5):
    assert got.shape == ref.shape
    err, scale = float((got - ref).abs().max()), float(ref.abs().max())
    assert err <= tol * scale, (err, scale)


@pytest.mark.parametrize("name", ["landscape", "portrait", "heavy", "small"])
def test_resize_matches_the_reference_golden(name):
    H, W, image_size, *_ = (int(v) for v in GOLD[name + "_cfg"])
    x = th.from_numpy(GOLD[name + "_image"]).permute(2, 0, 1).unsqueeze(0).float().div(255)
    ref = th.from_numpy(GOLD[name + "_resized"])
    got = pip.resize_lanczos3(x.cuda(), pip.resized_shape(H, W, image_size)).cpu()
    _close(got, ref)
    _close(got, oip.resize(x, image_size))


@pytest.mark.parametrize("H,W,size", [(3000, 2000, 64), (2000, 3000, 64), (768, 1024, 256)])
def test_resize_large_downscales_match_the_oracle(H, W, size):
    """photos reduced to the diffusion size: 188 / 282 taps per output at 3000 x 2000 -> 96 x 64"""
    x = th.rand(1, 3, H, W, generator=th.Generator().manual_seed(H + W))
    out_hw = pip.resized_shape(H, W, size)
    got = pip.resize_lanczos3(x.cuda(), out_hw).cpu()
    _close(got, orr.resize_lanczos3(x, out_hw))


@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("S,O,other", [(4000, 64, 33), (40000, 300, 2), (64, 200, 70), (300, 299, 1)])
def test_resize_axis_op_matches_the_oracle(axis, S, O, other):
    """one RESIZE_AXIS launch per axis, any tap count (up to 800 here), down- and up-scaling; at 40000 -> 300 the input span of one
    block's outputs in the W pass covers several shared-memory tiles"""
    x = th.randn(2, 3, *((S, other) if axis == 0 else (other, S)), generator=th.Generator().manual_seed(S + O))
    left, wt, T = rr.tables(S, O, t_max=None)
    xd = x.cuda()
    out = th.empty(2, 3, *((O, other) if axis == 0 else (other, O)), device="cuda")
    pip._run_op("RESIZE_AXIS", [6, xd.shape[2], xd.shape[3], axis, O, T], p=[xd, out, left.cuda(), wt.cuda()])
    _close(out.cpu(), orr._resize_dim(x, 2 + axis, O))


def _vit_b32():
    from oracle.clip_vit import CLIPVisualOnly, ViTConfig as OViTConfig
    cfg = pv.VIT_CONFIGS["ViT-B/32"]
    sd = pw.seeded_state_dict(pw.vit_param_shapes(cfg), 1235)
    m = CLIPVisualOnly(OViTConfig(cfg.input_resolution, cfg.patch_size, cfg.width, cfg.layers, cfg.output_dim)).eval()
    m.load_state_dict(sd)
    return cfg, sd, m.encode_image


def _rn50():
    from oracle import clip_rn as orn
    cfg = prn.RN_CONFIGS["RN50"]
    sd = pw.seeded_rn_state_dict(cfg, seed=3)
    m = orn.ModifiedResNet(orn.RNConfig(layers=tuple(cfg.layers), output_dim=cfg.output_dim, input_resolution=cfg.input_resolution,
                                        width=cfg.width)).eval()
    m.load_state_dict({k[len("visual."):]: v for k, v in sd.items()}, strict=False)
    return cfg, sd, m


@pytest.mark.parametrize("tower", ["ViT-B/32", "RN50"])
def test_encode_image_prompt_matches_the_oracle_tower(tmp_path, tower):
    """same seed -> same windows; the device cutouts (resize, pool, CLIP_NORMALIZE, fp16 patches) and embeddings against the fp32
    oracle on the same cutouts, with the tower tests' tolerance"""
    cfg, sd, oracle = _vit_b32() if tower == "ViT-B/32" else _rn50()
    path = str(tmp_path / "p.png")
    oip.write_png(path, 300, 410, seed=5)
    th.manual_seed(7)
    emb, w = cgd.encode_image_prompt(path, 0.8, 256, 8, tower, clip_state_dict=sd)
    state = th.get_rng_state()
    th.manual_seed(7)
    ref, w_ref, ex = oip.encode_image_prompt(oip.load_image(path), 0.8, 256, 8, oracle, cfg.input_resolution)
    assert th.equal(th.get_rng_state(), state) and w == w_ref == [0.1] * 8
    assert emb.shape == ref.shape == (8, cfg.output_dim) and emb.is_cuda
    emb = emb.cpu()
    rel = float((emb - ref).norm() / ref.norm())
    assert rel < 3e-2, rel
    # the resized image and windows the encoder used
    enc = pip.ImagePromptEncoder(cfg, sd, 8)
    th.manual_seed(7)
    enc.encode(path, 0.8, 256)
    assert enc.last["coords"] == ex["coords"]
    _close(enc.last["image"].cpu(), ex["image"])


def test_clip_guided_diffusion_with_an_image_prompt(tmp_path, monkeypatch):
    """image prompt only (no text tower): frames are yielded, P = num_cutouts, and the loop's first cutout windows are the ones the
    oracle replays from the seed after the image prompt's own draws"""
    monkeypatch.chdir(tmp_path)
    ucfg, vcfg = pu.config_for(64, True), pv.VIT_CONFIGS["ViT-B/32"]
    usd, vsd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234), pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 1235)
    path = str(tmp_path / "prompt.png")
    oip.write_png(path, 120, 100, seed=11)
    windows, engines = [], []

    class Recording(pg.MakeCutouts):
        def coords_for(self, *a, **k):
            c = super().coords_for(*a, **k)
            windows.append(c)
            return c

    class Engine(pg.GuidedStepB200):
        def __init__(self, *a, **k):
            engines.append(k["max_prompts"])
            super().__init__(*a, **k)

    monkeypatch.setattr(cgd, "MakeCutouts", Recording)
    monkeypatch.setattr(cgd, "GuidedStepB200", Engine)
    monkeypatch.setattr(cgd, "_encode_text", lambda *a, **k: pytest.fail("an image-only run must not load the text tower"))
    got = list(cgd.clip_guided_diffusion(image_size=64, num_cutouts=4, prompts=[], image_prompts=[path + ":0.5"], batch_size=1,
                                         timestep_respacing="25", skip_timesteps=22, save_frequency=2, prefix_path=tmp_path / "out",
                                         progress=False, seed=5, unet_state_dict=usd, clip_state_dict=vsd))
    assert [b for b, _ in got] == [0, 0] and all(os.path.exists(p) for _, p in got)
    assert engines == [4] and len(windows) == 3
    th.manual_seed(5)
    x = oip.resize(oip.load_image(path), 64)
    OMakeCutouts(vcfg.input_resolution, 4)._generate_coords(x.shape[2], x.shape[3], 4)  # the image prompt's draws
    assert windows[0] == OMakeCutouts(vcfg.input_resolution, 4)._generate_coords(64, 64, 4)
