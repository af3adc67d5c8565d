"""CPU: ResizeRight (lanczos3) cutouts on non-square images, with progressive cutout counts and after the use_augs pipeline -- the per-axis
host tables, whole guided steps through the plan interpreter against the oracle, the generators' consumption, the entry point with the
four options together, the new flags' argument checks, and the GPU owner of every new cutout launch at production sizes."""
import json
import os
import subprocess
import sys

import pytest
import torch as th

from clip_guided_diffusion_b200 import guidance as pg
from clip_guided_diffusion_b200 import resize_right as rr
from oracle import guidance as og
from oracle.resize_right import resize_lanczos3
from tests.rr_cutouts import AugResizeMakeCutouts, axis_matrix, interp_runner
from tests.step_parity import build_tiny, run_tiny_step_parity

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# (Sy, Sx, cs): rectangles, Sx = 1 (up-sampling a one-pixel column), an axis at S == cs (left untouched), and the largest down-scale the
# device tables hold (ceil(6 * 85 / 32) = 16 = T_MAX taps)
@pytest.mark.parametrize("sy,sx,cs", [(64, 40, 32), (17, 85, 32), (85, 1, 32), (32, 57, 32), (50, 32, 32), (224, 160, 224), (237, 100, 224),
                                      (1, 3, 16), (85, 85, 32)])
def test_per_axis_tables_match_the_oracle(sy, sx, cs):
    """each axis's tables (the y axis's from Sy, the x axis's from Sx) applied as A_y . crop . A_x^T equal ResizeRight on the rectangle"""
    g = th.Generator().manual_seed(sy * 1000 + sx)
    crop = th.randn(2, 3, sy, sx, generator=g)
    mats = []
    for S in (sy, sx):
        left, w, T = rr.tables(S, cs)
        assert T <= rr.T_MAX and bool((w[:, T:] == 0).all())
        mats.append(axis_matrix(left, w, T, S, cs, th.float64))
        if S == cs:
            assert T == 1 and th.equal(mats[-1], th.eye(cs, dtype=th.float64))
        inv = rr.inverse_ranges(left, T, S)  # the backward's gather ranges are exactly the outputs whose field of view holds r
        for r in range(S):
            touching = [o for o in range(cs) if int(left[o]) <= r < int(left[o]) + T]
            assert (int(inv[r, 0]), int(inv[r, 1])) == ((touching[0], touching[-1]) if touching else (int(inv[r, 0]), int(inv[r, 0]) - 1))
    got = mats[0] @ crop.double() @ mats[1].t()
    want = resize_lanczos3(crop, (cs, cs)).double()
    assert th.allclose(got, want, rtol=1e-5, atol=1e-5), float((got - want).abs().max())


CASES = [("ancestral", dict(B=1, cutn=4, image=64, hw=(64, 96))),
         ("ddim", dict(B=2, cutn=3, image=64, hw=(96, 64))),
         # progressive_cutout: an engine built for 8 cutouts with a 4-cutout variant runs either count from the same tables
         ("ancestral", dict(B=1, cutn=8, image=64, cutn_variants=(4,), run_cutn=4)),
         ("ddim", dict(B=1, cutn=8, image=64, cutn_variants=(4,), run_cutn=8)),
         ("ddim", dict(B=1, cutn=8, image=64, hw=(64, 96), cutn_variants=(4,), run_cutn=4)),
         ("ancestral", dict(B=2, cutn=3, image=64, use_augs=True)),
         ("ddim", dict(B=1, cutn=4, image=64, hw=(64, 96), use_augs=True)),
         ("ancestral", dict(B=1, cutn=4, image=64, hw=(96, 64), use_augs=True, cutn_variants=(2,), run_cutn=2))]


def _id(c):
    return c[0] + "-" + "-".join(f"{k}{v}" for k, v in c[1].items() if k != "image")


@pytest.mark.parametrize("mode,kw", CASES, ids=[_id(c) for c in CASES])
def test_step_plan_matches_oracle(mode, kw, monkeypatch):
    """teacher-forced step through the interpreter against the oracle's p_sample_with_grad / ddim_sample_with_grad (tests/test_step_cpu.py's
    tolerances); with use_augs the oracle augments each crop at its own resolution before resizing"""
    monkeypatch.setattr(og, "MakeCutouts", AugResizeMakeCutouts)
    res = run_tiny_step_parity(device="cpu", mode=mode, runner_factory=interp_runner, cutout_resize="lanczos3", **kw)
    assert res["cos_g"] > 0.999, res
    assert res["rel_g"] < 5e-2 and res["rel_x0"] < 2e-2 and res["rel_sample"] < 2e-2, res
    assert res["clip_loss_rel"] < 2e-2 and res["tv_loss_rel"] < 1e-3 and res["range_loss_rel"] < 1e-2, res


def test_progressive_counts_over_a_25_step_schedule(monkeypatch):
    """CondFnB200's progressive schedule over 25 steps (num_cutouts 8: 4, 8, 8 cutouts), each step's count teacher-forced against the oracle
    with that step's windows"""
    monkeypatch.setattr(og, "MakeCutouts", AugResizeMakeCutouts)
    ctx = build_tiny("cpu", B=1, cutn=8, image=64, hw=(64, 96), cutn_variants=(4,), cutout_resize="lanczos3")
    eng, pdiff = ctx["eng"], ctx["pdiff"]
    cf = pg.CondFnB200(eng, pdiff, pg.MakeCutouts(32, 8), progressive_cutout=True)
    from tests.step_parity import compare, engine_step, oracle_step
    seen, runner = [], interp_runner(eng)
    for step in range(25):
        c = cf.current_cutn()
        if step in (0, 8, 24):  # one step of each phase of the schedule
            g = th.Generator().manual_seed(step)
            x, y = th.randn(1, 3, 64, 96, generator=g), th.randint(0, 10, (1,), generator=g)
            th.manual_seed(step + 100)
            noise = th.randn_like(x)
            th.manual_seed(step + 200)
            coords = cf.next_coords(64, 96)
            t = 14  # the schedule decides the count; the step is teacher-forced at one mid-chain timestep
            o = oracle_step(dict(ctx, cutn=c), "ddim", x, t, y, step + 100, coords, fac_index=t)
            res = compare(o, engine_step(ctx, "ddim", x, t, y, noise, coords, fac_index=t, runner=runner))
            assert res["cos_g"] > 0.999 and res["rel_x0"] < 2e-2 and res["rel_sample"] < 2e-2, (step, c, res)
        seen.append(c)
        cf.step_done()
    assert sorted(set(seen)) == [4, 8] and seen[0] == 4 and seen[-1] == 8


def test_same_seed_draws_like_pool_mode():
    """for one seed, lanczos3 + use_augs stages the same aug parameters and noise fields as pool + use_augs and leaves the CPU generator
    where pool mode leaves it (the windows come from the same MakeCutouts draws in both modes)"""
    outs = []
    for resize in ("pool", "lanczos3"):
        ctx = build_tiny("cpu", B=2, cutn=4, image=64, hw=(64, 96), use_augs=True, cutout_resize=resize)
        eng = ctx["eng"]
        th.manual_seed(77)
        coords = pg.MakeCutouts(32, 4, use_augs=True).coords_for(64, 96)
        eng.stage_step(ctx["pdiff"].scalar_table(5, 5, 0.0), coords, ctx["pdiff"].model_timestep(5), th.zeros(2, dtype=th.long))
        outs.append((coords, eng.v(eng.aug_prm).clone(), eng.v(eng.aug_noise).clone(), th.random.get_rng_state().clone(), th.rand(3)))
    (c0, p0, n0, s0, r0), (c1, p1, n1, s1, r1) = outs
    assert c0 == c1 and th.equal(p0, p1) and th.equal(n0, n1) and th.equal(s0, s1) and th.equal(r0, r1)
    assert float(p0.abs().sum()) > 0 and float(n0.abs().sum()) > 0


def test_entry_point_combines_the_four_options(tmp_path, monkeypatch):
    """clip_guided_diffusion(cutout_resize="lanczos3") with height_offset, progressive_cutout and use_augs together yields every frame at
    the requested size (the engine's kernels interpreted; width_offset is exercised by the same x-axis tables)"""
    import numpy as np
    from PIL import Image
    from tests import test_entry_cpu
    from tests.rr_cutouts import RRInterp
    from tests.test_entry_options_cpu import _call
    monkeypatch.setattr(test_entry_cpu, "Interp", RRInterp)
    got = _call(tmp_path, monkeypatch, dict(cutout_resize="lanczos3", height_offset=32, progressive_cutout=True, num_cutouts=8, use_augs=True))
    assert len(got) == 3 and all(os.path.exists(p) for _, p in got)
    im = Image.open(got[-1][1])
    assert im.size == (64, 96) and np.isfinite(np.asarray(im, dtype=np.float32)).all()


def test_entry_point_accepts_width_offset(tmp_path, monkeypatch):
    """a wide image: the same swapped-side windows as pool mode, so a window may start past the last column and the run raises like the
    reference's empty crop does; the engine itself is built with its x-axis tables"""
    from tests import test_entry_cpu
    from tests.rr_cutouts import RRInterp
    from tests.test_entry_options_cpu import _call
    monkeypatch.setattr(test_entry_cpu, "Interp", RRInterp)
    with pytest.raises(RuntimeError, match="outside"):
        _call(tmp_path, monkeypatch, dict(cutout_resize="lanczos3", width_offset=64, timestep_respacing="ddim25"))


def test_empty_crop_still_raises():
    ctx = build_tiny("cpu", B=1, cutn=2, image=64, hw=(96, 64), cutout_resize="lanczos3")
    eng = ctx["eng"]
    with pytest.raises(RuntimeError, match="outside"):
        eng.stage_step(ctx["pdiff"].scalar_table(5, 5, 0.0), [(64, 0, 32), (0, 0, 64)], ctx["pdiff"].model_timestep(5), None)


NEW_MODES = [dict(B=1, cutn=3, image=64, hw=(64, 96), cutout_resize="lanczos3"),
             dict(B=1, cutn=2, image=64, hw=(96, 64), cutout_resize="lanczos3", use_augs=True),
             dict(B=2, cutn=4, image=64, cutout_resize="lanczos3", use_augs=True, cutn_variants=(2,))]


@pytest.mark.skipif(th.cuda.is_available(), reason="needs a box WITHOUT a GPU: only the argument checks may run")
@pytest.mark.parametrize("cfg", NEW_MODES, ids=["rect", "augs-rect", "augs-progressive"])
def test_malformed_ops_return_error_codes(cfg):
    """tests/test_abi_fuzz_cpu.py's child on the new modes' plans (every field of every distinct (code, flags) mutated): never a crash, a
    hang or a 0 without a device"""
    from tests.test_abi_fuzz_cpu import CHILD
    try:
        r = subprocess.run([sys.executable, "-c", CHILD, ROOT, json.dumps(cfg)], capture_output=True, text=True, timeout=240)
    except subprocess.TimeoutExpired:
        pytest.fail("cgd_run_op hung")
    lines = r.stdout.splitlines()
    assert r.returncode == 0 and lines and lines[-1].startswith("DONE"), f"crashed (rc {r.returncode}): {r.stderr[-400:]}"
    assert json.loads(lines[-1].split(" ", 3)[3]) == []


FLAG_CHILD = r'''
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from clip_guided_diffusion_b200 import _lib
from tests.plan_interp import CODE
from tests.step_parity import build_tiny
lib = _lib.load()
plan = build_tiny("cpu", **json.loads(sys.argv[2]))["eng"].plan
arr = plan.lower(1 << 40)
out = []
for k, op in enumerate(plan.ops):
    name = CODE[op.code]
    if not name.startswith(("CUTOUTS_RR", "CUTOUTS_AUG")):
        continue
    base = arr[k]
    muts = [("flags", None, f) for f in (op.flags | 4, op.flags | 8, op.flags | 1 << 20)] + [("p", j, 0) for j in range(12) if base.p[j]]
    if name == "CUTOUTS_RR_BWD" or op.flags & (2 if name == "CUTOUTS_RR_FWD" else 1):  # the ops that read Smax
        muts += [("i", 7, v) for v in (0, -1, 1)]
    for w, j, v in muts:
        if name == "CUTOUTS_AUG_BWD" and w == "flags" and v == 4:
            continue  # flags 4 is the stand-alone MakeCutouts backward's fp32 d cutouts
        o = type(base)()
        ctypes.memmove(ctypes.byref(o), ctypes.byref(base), ctypes.sizeof(base))
        if w == "flags":
            o.flags = v
        elif w == "p":
            o.p[j] = 0
        else:
            o.i[j] = v
        if name == "CUTOUTS_AUG_FWD" and w == "p" and j == 4:
            continue  # the noise fields are optional
        out.append((name, op.flags, w, j, v, lib.cgd_run_op(ctypes.byref(o), None)))
print(json.dumps(out))
'''


@pytest.mark.skipif(th.cuda.is_available(), reason="needs a box WITHOUT a GPU: only the argument checks may run")
def test_new_flags_and_pointers_are_checked_on_the_host():
    """unknown flag bits, a NULL table / workspace pointer and a Smax below min(H, W) are rejected as invalid arguments (-1) before any
    launch, on the new modes' CUTOUTS_RR_* / CUTOUTS_AUG_* ops"""
    for cfg in NEW_MODES[:2]:
        r = subprocess.run([sys.executable, "-c", FLAG_CHILD, ROOT, json.dumps(cfg)], capture_output=True, text=True, timeout=240)
        assert r.returncode == 0, r.stderr[-400:]
        res = json.loads(r.stdout.splitlines()[-1])
        flags = {(n, f) for n, f, *_ in res}
        assert {n for n, _ in flags} == {"CUTOUTS_RR_FWD", "CUTOUTS_RR_BWD"} | ({"CUTOUTS_AUG_FWD", "CUTOUTS_AUG_BWD"} if cfg.get("use_augs") else set())
        assert all(f & 1 for n, f in flags if n.startswith("CUTOUTS_RR")), flags  # non-square: the x-axis tables
        bad = [m for m in res if m[-1] != -1]
        assert not bad, bad


# ------------------------------------------------------------------------------------------------ every new launch has a GPU owner
def _prod_engine(H, W, clip, cutn, **kw):
    """the production CLIP tower and cutout geometry around a small UNet: the cutout launches depend on (B, H, W, cutn, cs, patch,
    Kpad) only, not on the UNet's width"""
    from clip_guided_diffusion_b200 import vit as pv
    from clip_guided_diffusion_b200 import weights as pw
    from oracle.unet import tiny_config
    from tests.step_parity import prod_unet_cfg
    ucfg = prod_unet_cfg(tiny_config(image_size=64, model_channels=64, channel_mult=(1, 2), num_res_blocks=1, attention_resolutions=(),
                                     class_cond=True))
    vcfg = pv.VIT_CONFIGS[clip]
    vcfg_small = pv.ViTConfig(vcfg.input_resolution, vcfg.patch_size, 64, 1, 32)  # same cutout geometry, a one-layer 64-wide trunk
    return pg.GuidedStepB200(ucfg, pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234), vcfg_small,
                             pw.seeded_state_dict(pw.vit_param_shapes(vcfg_small), 1235), device="cpu", batch=1, height=H, width=W,
                             num_cutouts=cutn, cutout_resize="lanczos3", **kw).plan


PROD = {  # cfg2 256² with +-64 offsets, cfg4 512² with ViT-B/16, ViT-L/14 and ViT-L/14@336px cut sizes; each with use_augs and progressive counts
    "cfg2_256x320": (256, 320, "ViT-B/32", {}), "cfg2_320x256": (320, 256, "ViT-B/32", {}), "cfg2_192x256": (192, 256, "ViT-B/32", {}),
    "cfg2_augs_256": (256, 256, "ViT-B/32", dict(use_augs=True)), "cfg2_augs_256x320": (256, 320, "ViT-B/32", dict(use_augs=True)),
    "cfg2_augs_320x256": (320, 256, "ViT-B/32", dict(use_augs=True)),
    "cfg2_progressive": (256, 256, "ViT-B/32", dict(cutn_variants=(4, 8))),
    "cfg4_512": (512, 512, "ViT-B/16", dict(use_augs=True, cutn_variants=(4, 8))), "cfg4_512x576": (512, 576, "ViT-B/16", {}),
    "vitl14_256x320": (256, 320, "ViT-L/14", dict(use_augs=True)), "vitl14_336_512x448": (512, 448, "ViT-L/14@336px", dict(use_augs=True)),
}


def plan_rr_signatures(plan) -> set:
    """(code, flags, B, H, W, cutn, cs, patch, Kpad, Smax | 0) of the plan's ResizeRight and use_augs cutout launches"""
    from tests.plan_interp import CODE
    out = set()
    for op in plan.ops:
        name = CODE[op.code]
        if name.startswith(("CUTOUTS_RR", "CUTOUTS_AUG")):
            i = [int(v) for v in op.i[:8]] + [0] * (8 - len(op.i[:8]))
            out.add((name, op.flags, *i))
    return out


@pytest.mark.parametrize("name", list(PROD))
def test_every_new_cutout_launch_has_a_gpu_owner(name):
    """the cutout launches of the new modes at production sizes are the signatures tests/test_gpu_rr_cutouts.py runs against float64 (or,
    for the augmentation passes, against the fp32 torchvision pipeline)"""
    from tests.test_gpu_rr_cutouts import covered_signatures
    H, W, clip, kw = PROD[name]
    sigs = plan_rr_signatures(_prod_engine(H, W, clip, 16, **kw))
    assert sigs, name
    missing = sorted(sigs - covered_signatures(), key=repr)
    assert not missing, f"{name}: no GPU case runs {missing}"
