"""GPU: CLIP visual towers under torch.autograd (clip_model.py, load_clip).

- CLIP_PATCHIFY / CLIP_SEED / CLIP_UNPATCHIFY bit for bit against float64 references at every published tower's geometry, 1, 16 and 64
  images on a 64-image layout;
- encode_image of all eight published towers (seeded weights) against the fp32 oracle, the bars tests/test_gpu_rn.py holds the towers to;
- CLIP_SEED's purpose: an upstream gradient d * 2^k gives exactly 2^k times the input gradient;
- retain_graph repeats bitwise, padding stays within split-K reordering;
- one cfg2-size step (256^2, ViT-B/32, 16 cutouts) with the oracle's cond_fn on load_clip's model and engine.model against the oracle;
- every CONV / attention / glue launch of load_clip's plans that the shipped-plan tables do not list, through the bit-exact harnesses of
  tests/test_gpu_conv_kernels.py and tests/test_gpu_unet_kernels.py (tests/clip_autograd_plan_table.py)."""
from __future__ import annotations

import math

import pytest
import torch as th

from tests.clip_autograd_plan_table import CLIP_CONV_PLAN, CLIP_OTHER_PLAN

pytestmark = pytest.mark.gpu

# (name, R, P, kpad, D) of the published towers
GEOMS = [("ViT-B/32", 224, 32, 3072, 512), ("ViT-B/16", 224, 16, 768, 512), ("ViT-L/14", 224, 14, 640, 768), ("ViT-L/14@336px", 336, 14, 640, 768),
         ("RN50", 224, 2, 64, 1024), ("RN101", 224, 2, 64, 512), ("RN50x4", 288, 2, 64, 640), ("RN50x16", 384, 2, 64, 768)]
NB = 64


def covered_conv_signatures() -> set:
    return set(CLIP_CONV_PLAN)


def covered_other_signatures() -> set:
    return set(CLIP_OTHER_PLAN)


def _bits16(t):
    return t.contiguous().view(th.int16)


def _patchify(img, P, kpad):
    n, _, R, _ = img.shape
    g = R // P
    t = img.reshape(n, 3, g, P, g, P).permute(0, 2, 4, 1, 3, 5).reshape(n, g * g, 3 * P * P)
    return th.nn.functional.pad(t, (0, kpad - 3 * P * P))


def _unpatchify(t, P, R):
    n, g = t.shape[0], R // P
    return t[:, :, :3 * P * P].reshape(n, g, g, 3, P, P).permute(0, 3, 1, 4, 2, 5).reshape(n, 3, R, R)


# ---------------------------------------------------------------------- the three kernels, bit for bit
@pytest.mark.parametrize("n", [1, 16, 64])
@pytest.mark.parametrize("geom", GEOMS, ids=[g[0] for g in GEOMS])
def test_patchify_unpatchify_bitwise(geom, n):
    from clip_guided_diffusion_b200._lib import run_op
    _, R, P, kpad, _ = geom
    G2 = (R // P) ** 2
    g = th.Generator(device="cuda").manual_seed(n * 7 + P)
    # magnitudes from 2^-30 to 2^4: near-zero normalised pixels keep their low bits through the one fp16 rounding
    x = th.randn(n, 3, R, R, device="cuda", generator=g) * th.exp2(th.randint(-30, 5, (n, 3, R, R), device="cuda", generator=g).float())
    rows = th.full((NB, G2, kpad), float("nan"), device="cuda", dtype=th.float16)
    run_op("CLIP_PATCHIFY", i=[n, NB, R, P, kpad], p=[x, rows])
    want = th.zeros(NB, G2, kpad, device="cuda", dtype=th.float16)
    want[:n] = _patchify(x.half(), P, kpad)
    assert th.equal(_bits16(rows), _bits16(want))
    # the transpose: pad columns and rows n.. hold NaN and must not be read; the scales span 2^-60 .. 2^60
    dp = (th.randn(NB, G2, kpad, device="cuda", generator=g) * 64).half()
    dp[:, :, 3 * P * P:] = float("nan")
    dp[n:] = float("nan")
    scale = th.exp2(th.randint(-60, 61, (NB,), device="cuda", generator=g).float())
    dx = th.full((n, 3, R, R), float("nan"), device="cuda")
    run_op("CLIP_UNPATCHIFY", i=[n, NB, R, P, kpad], p=[dp, scale, dx])
    ref = _unpatchify(dp[:n].double(), P, R) / scale[:n].double().view(n, 1, 1, 1)
    assert th.equal(ref.float().double(), ref) and th.equal(dx, ref.float())


def _seed_rows(n, D, g):
    d = th.randn(NB, D, device="cuda", generator=g) * th.exp2(th.randint(-100, 100, (NB, 1), device="cuda", generator=g).float())
    specials = {0: ("zero",), 1: ("nan", 5), 2: ("inf", 9), 3: ("tiny",), 4: ("huge",)}
    for r, (kind, *col) in specials.items():
        if r >= n:
            break
        if kind == "zero":
            d[r] = 0
        elif kind == "nan":
            d[r, col[0]] = float("nan")
        elif kind == "inf":
            d[r, col[0]] = -float("inf")
        elif kind == "tiny":
            d[r] *= 1e-30 / d[r].abs().max()
        else:
            d[r] *= 1e30 / d[r].abs().max()
    return d


def _seed_ref(d, band):
    out = []
    for row in d.double().cpu().tolist():
        vals = [min(abs(v), 3.0e38) for v in row if not math.isnan(v)]
        m = max(vals, default=0.0)
        out.append(1.0 if m == 0 else 2.0 ** min(max(math.floor(math.log2(band / m)), -60), 60))
    return th.tensor(out, dtype=th.float64, device=d.device)


@pytest.mark.parametrize("n", [1, 16, 64])
@pytest.mark.parametrize("D", sorted({g[4] for g in GEOMS}))
def test_seed_bitwise(D, n):
    from clip_guided_diffusion_b200._lib import run_op
    from clip_guided_diffusion_b200.clip_model import CLIP_SEED_BAND
    g = th.Generator(device="cuda").manual_seed(D + n)
    d = _seed_rows(n, D, g)
    d_emb = th.full((NB, D), float("nan"), device="cuda")
    dyn = th.full((NB,), float("nan"), device="cuda")
    run_op("CLIP_SEED", i=[n, NB, D], f=[CLIP_SEED_BAND], p=[d, d_emb, dyn])
    s = _seed_ref(d[:n], CLIP_SEED_BAND)
    assert th.equal(dyn[:n].double(), s) and th.equal(dyn[n:], th.ones(NB - n, device="cuda"))
    want = (d[:n].double() * s[:, None]).float()
    th.testing.assert_close(d_emb[:n], want, rtol=0, atol=0, equal_nan=True)
    assert th.equal(d_emb[n:], th.zeros(NB - n, D, device="cuda"))
    # rows whose scale is not clamped at 2^+-60 and that hold no inf land in (BAND / 2, BAND]
    ok = (s > 2.0 ** -60) & (s < 2.0 ** 60) & ~th.isinf(d[:n]).any(1) & (d[:n].abs().nan_to_num(nan=0.0).amax(1) > 0)
    top = d_emb[:n].abs().nan_to_num(nan=0.0).amax(1)[ok]
    assert bool(((top <= CLIP_SEED_BAND) & (top > CLIP_SEED_BAND / 2)).all())


# ---------------------------------------------------------------------- the published towers against the fp32 oracle
def _published(name, max_images):
    from clip_guided_diffusion_b200 import clip_util
    from clip_guided_diffusion_b200 import rn as prn
    from clip_guided_diffusion_b200 import vit as pv
    from clip_guided_diffusion_b200 import weights as pw
    from oracle import clip_rn as orn
    from oracle.clip_vit import VIT_CONFIGS, CLIPVisualOnly
    if name in pv.VIT_CONFIGS:
        sd = pw.seeded_state_dict(pw.vit_param_shapes(pv.VIT_CONFIGS[name]), 1235)
        oracle = CLIPVisualOnly(VIT_CONFIGS[name]).eval()
        oracle.load_state_dict(sd)
    else:
        cfg = prn.RN_CONFIGS[name]
        sd = pw.seeded_rn_state_dict(cfg, seed=3)
        oracle = orn.CLIPVisualRN(orn.RNConfig(tuple(cfg.layers), cfg.output_dim, cfg.input_resolution, cfg.width)).eval()
        oracle.load_state_dict(sd, strict=False)
    for prm in oracle.parameters():
        prm.requires_grad_(False)
    model, size = clip_util.load_clip(name, "cuda", clip_state_dict=sd, max_images=max_images)
    return model, size, oracle.cuda(), sd


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def _cos(a, b):
    return float(th.nn.functional.cosine_similarity(a.flatten().double(), b.flatten().double(), dim=0))


@pytest.mark.parametrize("name", [g[0] for g in GEOMS])
def test_published_towers_vs_oracle(name):
    model, R, oracle, _ = _published(name, 16)
    assert model.visual.input_resolution == R
    g = th.Generator(device="cuda").manual_seed(1)
    x = th.randn(2, 3, R, R, device="cuda", generator=g)
    w = th.randn(2, model.cfg.output_dim, device="cuda", generator=g)
    xe = x.clone().requires_grad_()
    emb = model.encode_image(xe)
    (ge,) = th.autograd.grad((w * emb).sum(), xe)
    xo = x.clone().requires_grad_()
    ref = oracle.encode_image(xo).float()
    (go,) = th.autograd.grad((w * ref).sum(), xo)
    vals = (_rel(emb.detach(), ref.detach()), _cos(ge, go))
    print(f"\n{name}: rel(embeds) {vals[0]:.3e} cos(d clip_in) {vals[1]:.5f}")
    assert emb.dtype == th.float32 and vals[0] < 3e-2 and vals[1] > 0.99, vals


def test_scale_invariance_bitwise():
    """d * 2^k upstream gives exactly 2^k times the k = 0 input gradient: CLIP_SEED absorbs any power of two"""
    model, R, _, _ = _published("ViT-B/32", 16)
    g = th.Generator(device="cuda").manual_seed(2)
    x = th.randn(16, 3, R, R, device="cuda", generator=g).requires_grad_()
    d = th.randn(16, 512, device="cuda", generator=g)
    grads = {}
    for k in (-40, -20, 0, 20, 40):
        emb = model.encode_image(x)
        (grads[k],) = th.autograd.grad(emb, x, grad_outputs=d * 2.0 ** k)
    assert grads[0].abs().max() > 0
    for k in (-40, -20, 20, 40):
        assert th.equal(grads[k], grads[0] * 2.0 ** k), k


def test_repeat_and_padding():
    model, R, _, sd = _published("RN50", 16)
    from clip_guided_diffusion_b200 import clip_util
    exact, _ = clip_util.load_clip("RN50", "cuda", clip_state_dict=sd, max_images=5)
    g = th.Generator(device="cuda").manual_seed(3)
    x = th.randn(5, 3, R, R, device="cuda", generator=g)
    w = th.randn(5, 1024, device="cuda", generator=g)
    out = []
    for m in (model, exact):
        xe = x.clone().requires_grad_()
        e = m.encode_image(xe)
        (g1,) = th.autograd.grad((w * e).sum(), xe, retain_graph=True)
        (g2,) = th.autograd.grad((w * e).sum(), xe)
        assert th.equal(g1, g2)
        out.append((e.detach(), g1))
    # RN50's fp16 backward is ~7 % (rel) from the fp32 oracle's (cos 0.998, test_published_towers_vs_oracle); another split-K order
    # rounds differently along the same 50 layers: measured 2.3e-4 (embeds) and 3.0e-2 (input gradient) on an H100
    vals = (_rel(out[0][0], out[1][0]), _rel(out[0][1], out[1][1]), _cos(out[0][1], out[1][1]))
    assert vals[0] < 2e-3 and vals[1] < 6e-2 and vals[2] > 0.998, vals


def test_encode_text_matches_text_tower():
    from clip_guided_diffusion_b200 import clip_util
    from clip_guided_diffusion_b200 import vit as pv
    from clip_guided_diffusion_b200 import weights as pw
    from clip_guided_diffusion_b200.text import TextB200, TextConfig
    tcfg = TextConfig()
    sd = pw.seeded_state_dict({**pw.vit_param_shapes(pv.VIT_CONFIGS["ViT-B/32"]), **pw.text_param_shapes(tcfg)}, 7)
    model, _ = clip_util.load_clip("ViT-B/32", "cuda", clip_state_dict=sd, max_images=1)
    ids = th.zeros(3, 77, dtype=th.int32)
    for r, length in enumerate((5, 12, 77)):
        ids[r, :length] = th.randint(1, 49000, (length,), generator=th.Generator().manual_seed(r))
        ids[r, length - 1] = 49407
    got = model.encode_text(ids)
    want = TextB200(tcfg, sd, 3, "cuda").encode(ids)
    assert got.dtype == th.float32 and got.shape == (3, 512) and th.equal(got, want)


# ---------------------------------------------------------------------- one cfg2-size step
@pytest.mark.parametrize("mode", ["ancestral", "ddim"])
def test_cfg2_step_with_load_clip_model(mode):
    from clip_guided_diffusion_b200 import clip_util
    from clip_guided_diffusion_b200 import guidance as pg
    from clip_guided_diffusion_b200 import unet as pu
    from clip_guided_diffusion_b200 import vit as pv
    from clip_guided_diffusion_b200 import weights as pw
    from oracle import diffusion as od
    from oracle import guidance as og
    from oracle.clip_vit import VIT_CONFIGS, CLIPVisualOnly
    from oracle.unet import UNetModel, config_for
    ucfg, vcfg = pu.config_for(256, True), pv.VIT_CONFIGS["ViT-B/32"]
    usd, vsd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234), pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 1235)
    eng = pg.GuidedStepB200(ucfg, usd, batch=1, device="cuda", input_grad=True)
    clip_model, clip_size = clip_util.load_clip("ViT-B/32", "cuda", clip_state_dict=vsd)
    clip_model = clip_model.eval().requires_grad_(False).to("cuda")
    ounet = UNetModel(config_for(256, True)).eval()
    ounet.load_state_dict(usd)
    oclip = CLIPVisualOnly(VIT_CONFIGS["ViT-B/32"]).eval()
    oclip.load_state_dict(vsd)
    ounet, oclip = ounet.cuda(), oclip.cuda()
    for prm in list(ounet.parameters()) + list(oclip.parameters()):
        prm.requires_grad_(False)
    odiff = od.create_gaussian_diffusion(1000, "linear", "ddim25" if mode == "ddim" else "25")
    th.manual_seed(0)
    tgt = th.randn(1, 512, device="cuda")
    coords = og.MakeCutouts(224, 16)._generate_coords(256, 256, 16)
    g = th.Generator().manual_seed(3)
    x, y = th.randn(1, 3, 256, 256, generator=g).cuda(), th.randint(0, 1000, (1,), generator=g).cuda()
    res = []
    for model, cm in ((eng.model, clip_model), (ounet, oclip)):
        cf = og.OracleCondFn(odiff, cm, tgt, th.ones(1, device="cuda"), cut_size=clip_size, num_cutouts=16)
        cf.current_timestep = 14
        seen = {}

        def cond_fn(xx, tt, out, y=None, cf=cf, seen=seen):
            seen["g"] = cf(xx, tt, out, y=y, coords=coords)
            return seen["g"]
        th.manual_seed(21)
        fn = odiff.p_sample_with_grad if mode == "ancestral" else odiff.ddim_sample_with_grad
        o = fn(model, x, th.full((1,), 14, dtype=th.long, device="cuda"), clip_denoised=False, cond_fn=cond_fn, model_kwargs={"y": y})
        res.append(dict(o, g=seen["g"].detach()))
    e, o = res
    vals = (_cos(e["g"], o["g"]), _rel(e["pred_xstart"], o["pred_xstart"]), _rel(e["sample"], o["sample"]))
    print(f"\ncfg2-size {mode} step, engine.model + load_clip vs oracle: cos(g) {vals[0]:.5f} rel(pred_xstart) {vals[1]:.3e} "
          f"rel(sample) {vals[2]:.3e}")
    assert clip_model.forward_generation == 1
    assert vals[0] > 0.995 and vals[1] < 2e-2 and vals[2] < 2e-2, vals


# ---------------------------------------------------------------------- launches of load_clip's plans outside the shipped-plan tables
def _conv_ids():
    from tests.test_gpu_conv_kernels import conv_id
    return [conv_id(s) for s in CLIP_CONV_PLAN]


@pytest.mark.parametrize("case", CLIP_CONV_PLAN, ids=_conv_ids())
def test_tower_conv_launches(case):
    from tests import test_gpu_conv_kernels as KC
    KC.test_conv_exact("cuda", case)
    KC.test_conv_randn("cuda", case)


# attention shapes at which the harness's fixed data seed (T * 7 + d + B) draws a "peaked" query row whose peak is less than 20 above
# another logit, so that its own data precondition fails before any kernel runs: RN50x16's attention pool (16 images x 48 heads x 145
# tokens, 22k peaked rows) on an H100.  These run on the next seed; the kernel, shape and checks are the same.
ATTN_SEED_SHIFT = {(16, 48, 145, 64): 1}


@pytest.mark.parametrize("sig", CLIP_OTHER_PLAN, ids=[repr(s) for s in CLIP_OTHER_PLAN])
def test_tower_other_launches(sig, monkeypatch):
    from tests import test_gpu_unet_kernels as KU
    kind, rest = sig[0], tuple(sig[1:])
    if kind in ("ATTN_FWD", "ATTN_BWD"):
        shift = ATTN_SEED_SHIFT.get(rest[:4], 0)
        if shift:
            inputs = KU.attn_inputs
            monkeypatch.setattr(KU, "attn_inputs", lambda device, B, heads, T, d, seed: inputs(device, B, heads, T, d, seed + shift))
        KU.test_attention("cuda", rest)
    elif kind in ("POOL2", "UP2"):
        KU.test_pool2_up2("cuda", (kind, rest))
    elif kind in ("ADD", "COPY"):
        KU.test_add_copy("cuda", (kind, rest))
    else:
        pytest.fail(f"no GPU harness for {kind}")
