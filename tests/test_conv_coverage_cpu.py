"""Every CONV signature the shipped plans emit is a case of tests/test_gpu_conv_kernels.py.

Every engine the GPU suite runs at full size is built on the CPU with seeded weights: the cfg2, cfg3 (32 cutouts), cfg2 with progressive
cutout counts, cfg4, cfg5 (+ LPIPS),
default128, 64x64 and ViT-L/14@336 guided steps, the RN50 / RN50x4 / RN50x16 towers, the text towers and the image-prompt encoders.  The
signature of each CONV op (tests/test_gpu_conv_kernels.py `conv_signature`: shape, Npad, taps, BN, splits, cluster flag, flags, operand
presence, strides, in-place residual) is looked up in tests/conv_plan_table.py.  A plan change that introduces a launch no GPU test runs
fails here, on a machine without a GPU; `python scripts/conv_signatures.py` regenerates the table.  `plan.cluster_capacity` answers
with the H100's numbers when there is no device, so these builds choose what the card chooses (test_cfg2_signatures_on_the_device)."""
from __future__ import annotations

import functools

import pytest
import torch as th

from clip_guided_diffusion_b200 import guidance as pg
from clip_guided_diffusion_b200 import image_prompt as pip
from clip_guided_diffusion_b200 import rn as prn
from clip_guided_diffusion_b200 import text as ptx
from clip_guided_diffusion_b200 import unet as pu
from clip_guided_diffusion_b200 import vit as pv
from clip_guided_diffusion_b200 import weights as pw
from clip_guided_diffusion_b200._lib import OP
from tests import test_gpu_conv_kernels as K


def _step(size, clip, cutn, lpips=False, **kw):
    def build(device="cpu"):
        ucfg, vcfg = pu.config_for(size, class_cond=True), pv.VIT_CONFIGS[clip]
        extra = dict(lpips_sd=pw.seeded_lpips_state_dict(), init_scale=1000.0, **kw) if lpips else kw
        return pg.GuidedStepB200(ucfg, pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234), vcfg,
                                 pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 1235), device=device, batch=1, num_cutouts=cutn, **extra).plan
    return build


def _rn(name, n):
    return lambda: prn.RNB200(prn.RN_CONFIGS[name], pw.seeded_rn_state_dict(prn.RN_CONFIGS[name], seed=3), n_images=n, device="cpu").plan


def _text(width, n):
    cfg = ptx.TextConfig(width=width, layers=12, output_dim=width)
    return lambda: ptx.TextB200(cfg, pw.seeded_state_dict(pw.text_param_shapes(cfg), width), n, device="cpu").plan


def _image_prompt(name):
    if name.startswith("RN"):
        cfg = prn.RN_CONFIGS[name]
        return lambda: pip.ImagePromptEncoder(cfg, pw.seeded_rn_state_dict(cfg, seed=3), 8, device="cpu").tower.plan
    cfg = pv.VIT_CONFIGS[name]
    return lambda: pip.ImagePromptEncoder(cfg, pw.seeded_state_dict(pw.vit_param_shapes(cfg), 1235), 8, device="cpu").tower.plan


# name -> (plan builder, the kernel variants its plan must contain: the collector must not go blind to one)
ENGINES = {
    "cfg2": (_step(256, "ViT-B/32", 16), {"persistent", "ws", "cluster", "narrow"}),
    "cfg3": (_step(256, "ViT-B/32", 32), {"persistent", "ws", "cluster", "narrow"}),
    # progressive_cutout: the tower also runs at max(4, n // 4) and max(8, n // 2) cutouts (cgd/cgd.py:167-175)
    "cfg2_progressive": (_step(256, "ViT-B/32", 16, cutn_variants=pg.CondFnB200.progressive_counts(16)[:-1]), {"persistent", "ws", "cluster", "narrow"}),
    "cfg4": (_step(512, "ViT-B/16", 16), {"persistent", "ws", "cluster", "narrow"}),
    "cfg5": (_step(512, "ViT-L/14", 64, lpips=True), {"persistent", "ws", "cluster", "narrow"}),
    "default128": (_step(128, "ViT-B/32", 16), {"persistent", "ws", "cluster", "narrow"}),
    "64x64": (_step(64, "ViT-B/32", 16), {"persistent", "ws", "cluster"}),
    "vit_l14_336": (_step(256, "ViT-L/14@336px", 4), {"persistent", "ws", "cluster", "narrow"}),
    "rn50": (_rn("RN50", 2), {"persistent", "ws", "cluster"}),
    "rn50x4": (_rn("RN50x4", 1), {"persistent", "ws", "cluster"}),
    "rn50x16": (_rn("RN50x16", 1), {"persistent", "ws", "cluster"}),
    "text512x5": (_text(512, 5), {"persistent", "cluster"}),
    "text640x5": (_text(640, 5), {"persistent", "ws"}),
    "text768x5": (_text(768, 5), {"persistent", "cluster"}),
    "text512x1": (_text(512, 1), {"persistent", "cluster"}),
    "image_prompt_vit_b32": (_image_prompt("ViT-B/32"), {"persistent", "cluster"}),
    "image_prompt_rn50": (_image_prompt("RN50"), {"persistent", "ws", "cluster"}),
}


def plan_conv_signatures(plan) -> set:
    return {K.conv_signature(op) for op in plan.ops if op.code == OP["CONV"]}


@functools.lru_cache(maxsize=None)
def signatures(name) -> frozenset:
    th.manual_seed(0)
    return frozenset(plan_conv_signatures(ENGINES[name][0]()))


@pytest.mark.parametrize("name", list(ENGINES))
def test_plan_conv_signatures_are_tested(name):
    sigs = signatures(name)
    paths = {K.conv_path(s) for s in sigs}
    assert ENGINES[name][1] <= paths, f"{name}: no CONV on the {sorted(ENGINES[name][1] - paths)} path(s) found: the collector or the planner changed"
    covered = K.covered_signatures()
    missing = sorted((s for s in sigs if s not in covered), key=repr)
    assert not missing, f"{name}: {len(missing)} CONV signature(s) without a case in tests/conv_plan_table.py " \
        "(regenerate it with scripts/conv_signatures.py):\n" + "\n".join(f"{K.conv_id(s)}  {s!r}" for s in missing)


def test_table_has_nothing_but_plan_signatures():
    """the table is the union of the engines' signatures: a stale row would be a GPU case of a launch nothing makes (hand-written cases
    belong in CONV_EXTRA)"""
    union = set().union(*(signatures(n) for n in ENGINES))
    stale = sorted((s for s in K.CONV_PLAN if s not in union), key=repr)
    assert not stale and len(set(K.CONV_PLAN)) == len(K.CONV_PLAN), stale


@pytest.mark.gpu
def test_cfg2_signatures_on_the_device():
    """the plan built on the card (its SM count, its cluster capacity) makes the launches the CPU-built table describes"""
    th.manual_seed(0)
    assert plan_conv_signatures(ENGINES["cfg2"][0](device="cuda")) == set(signatures("cfg2"))
