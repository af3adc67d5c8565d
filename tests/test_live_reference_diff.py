"""CPU: differential tests against the reference on many random inputs -- its modules (`cgd.modules`, `cgd.losses`), the function
bodies of `cgd/script_util.py` and the `cond_fn` closure of `cgd/cgd.py`.  The inputs are generated here from fixed seeds;
`tests/golden/live_reference_golden.json.gz` / `.npz` hold what the reference returned for them (tests/golden/make_golden_live_reference.py
runs it).  Tensor outputs are stored as a fixed, seeded sample of their elements (plus the absolute maximum), to keep the files small."""
import gzip
import hashlib
import json
import os
import random

import numpy as np
import pytest
import torch as th

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
N_SAMPLE = 256


def _golden():
    with gzip.open(os.path.join(GOLDEN, "live_reference_golden.json.gz"), "rt", encoding="utf-8") as f:
        js = json.load(f)
    return js, dict(np.load(os.path.join(GOLDEN, "live_reference_golden.npz")))


def sample_index(numel: int, key: str) -> th.Tensor:
    """fixed element sample of a tensor output: all of it when small, else N_SAMPLE indices drawn from a generator seeded by `key`"""
    if numel <= N_SAMPLE:
        return th.arange(numel)
    seed = int(hashlib.sha256(key.encode()).hexdigest()[:8], 16)
    return th.randperm(numel, generator=th.Generator().manual_seed(seed))[:N_SAMPLE].sort().values


def summarize(t: th.Tensor, key: str) -> np.ndarray:
    """[absmax, sampled elements...] of a tensor output, float64"""
    flat = t.detach().double().flatten()
    return np.concatenate([[float(flat.abs().max()) if flat.numel() else 0.0], flat[sample_index(flat.numel(), key)].numpy()])


def rng_digest() -> str:
    return hashlib.sha256(th.get_rng_state().numpy().tobytes()).hexdigest()


def _close(got: th.Tensor, want: np.ndarray, key: str, rel: float):
    g = summarize(got, key)
    assert g.shape == want.shape, key
    assert abs(g[0] - want[0]) <= rel * want[0] + 1e-12, (key, g[0], want[0])
    assert np.abs(g[1:] - want[1:]).max(initial=0.0) <= rel * want[0] + 1e-12, key


# ---------------------------------------------------------------- inputs (shared with the golden script)
ALPHABET = "abc XYZ019_-.,:;!?/\\'\"()[]{}<>@#$%^&*+=~`|\t\néü中\U0001f600"
N_PROMPTS = 600


def prompt_cases():
    """(texts, b) for the filter / combine helpers, then prompts for parse_prompt"""
    rng = random.Random(7)
    combine = []
    for _ in range(N_PROMPTS):
        texts = ["".join(rng.choice(ALPHABET) for _ in range(rng.randint(0, n))) for n in (40, 300)]
        combine.append((texts, rng.randint(0, 99)))
    prompts = []
    for _ in range(2000):
        body = "".join(rng.choice("ab :/.-") for _ in range(rng.randint(0, 12)))
        prompts.append(rng.choice(["", "http://", "https://"]) + body + rng.choice(["", ":1", ":-0.5", ":2e-1", ":3", ":", ":x"]))
    return combine, prompts


def cutout_cases():
    rng = random.Random(11)
    out = []
    for trial in range(300):
        cs = rng.choice([32, 224, 288, 336, 384])
        side_x, side_y = rng.choice([64, 128, 256, 320, 512]), rng.choice([64, 128, 256, 320, 512])
        cutn, power = rng.randint(1, 40), rng.choice([1.0, 0.5, 2.0, 0.25])
        out.append((trial, cs, side_x, side_y, cutn, power))
    return out


def loss_cases():
    """per trial: (B, H, W, x, seed, e, t, cutout weight or None) -- drawn in the order the comparisons consume them"""
    g = th.Generator().manual_seed(5)
    out = []
    for trial in range(12):
        B, H, W = [1, 2, 3][trial % 3], [48, 64, 40][trial % 3], [48, 40, 64][(trial // 3) % 3]
        x = th.randn(B, 3, H, W, generator=g) * 1.5
        seed = th.randn(B, generator=g)
        e, t = th.randn(1, 5, B, 16, generator=g), th.randn(1, 1, 16, generator=g)
        w = th.randn(B * 4, 3, 32, 32, generator=g) if H >= W else None  # wide images: empty crops in the reference (no comparison)
        out.append((trial, B, H, W, x, seed, e, t, w))
    return out


def cond_cases():
    from oracle import diffusion as od
    rng = random.Random(3)
    out = []
    for trial in range(40):
        B = rng.choice([1, 1, 2, 3])
        P = 1 if B > 1 else rng.choice([1, 2, 4])  # quirk B1: the broadcast is only defined for B == 1 or P == 1
        H = rng.choice([32, 40, 48, 64])
        W = rng.choice([w for w in (32, 40, 48, 64) if w <= H])
        cutn, power, T = rng.randint(1, 7), rng.choice([1.0, 0.5, 2.0]), rng.choice([25, 50, 100])
        t, sat, mag = rng.randrange(T), rng.choice([0.0, 0.0, 12.5]), rng.random() < 0.5
        scales = dict(clip_guidance_scale=rng.choice([1000, 250.0]), tv_scale=rng.choice([150, 0.0, 20.0]), range_scale=rng.choice([50, 5.0]))
        g = th.Generator().manual_seed(1000 + trial)
        x = th.randn(B, 3, H, W, generator=g) * rng.choice([0.5, 1.0, 1.6])
        target = th.randn(P, 16, generator=g)
        w = th.randn(P, generator=g).abs() + 0.1
        w = w / w.sum().abs()
        diff = od.create_gaussian_diffusion(1000, "linear", str(T))
        out.append(dict(trial=trial, B=B, P=P, H=H, W=W, cutn=cutn, power=power, T=T, t=t, sat=sat, mag=mag, scales=scales, x=x, target=target,
                        w=w, diff=diff))
    return out


# ---------------------------------------------------------------- tests
def test_prompt_helpers_on_random_strings():
    from clip_guided_diffusion_b200 import cgd
    js, _ = _golden()
    combine, prompts = prompt_cases()
    want = js["prompts"]
    for (texts, b), (filt, comb) in zip(combine, want["combine"], strict=True):
        assert cgd.alphanumeric_filter(texts[0]) == filt
        assert cgd.clean_and_combine_prompts("base", texts, b) == comb
    for prompt, ref in zip(prompts, want["parse"], strict=True):
        if ref is None:  # "text:" / "text:x": float('') raises in the reference, so it must here
            with pytest.raises(ValueError):
                cgd.parse_prompt(prompt)
            continue
        assert list(cgd.parse_prompt(prompt)) == ref, prompt


def test_cutout_windows_follow_the_reference_generator_for_random_geometries():
    """same CPU-generator consumption and the same windows as cgd/modules.py:26-48 for random image sizes, cut sizes, counts, powers --
    fresh draws, cached draws and the `num_cutouts_override` prefix rule; product class and oracle class"""
    from clip_guided_diffusion_b200 import guidance as pg
    from oracle import guidance as og
    js, _ = _golden()
    for (trial, cs, side_x, side_y, cutn, power), ref in zip(cutout_cases(), js["cutouts"], strict=True):
        want = [tuple(c) for c in ref["coords"]]
        cached = [tuple(c) for c in ref["cached"]]
        for mk in (pg.MakeCutouts(cs, cutn, cutout_size_power=power), og.MakeCutouts(cs, cutn, power)):
            th.manual_seed(trial)
            assert [tuple(c) for c in mk._generate_coords(side_x, side_y, cutn)] == want
            assert rng_digest() == ref["rng"], "different consumption of the default generator"
            th.manual_seed(trial + 1)
            mk.cache_coordinates(side_x, side_y)
            assert [tuple(c) for c in mk.cached_coords] == cached
    # the product's coords_for() mirrors forward()'s choice between the cache and fresh draws (cgd/modules.py:50-58)
    mk = pg.MakeCutouts(224, 16)
    th.manual_seed(3)
    mk.cache_coordinates(256, 256)
    assert [tuple(c) for c in mk.coords_for(256, 256, use_cache=True, num_cutouts_override=4)] == [tuple(c) for c in js["coords_for"]["cached"][:4]]
    th.manual_seed(4)
    assert [tuple(c) for c in mk.coords_for(256, 256, use_cache=False, num_cutouts_override=8)] == [tuple(c) for c in js["coords_for"]["fresh"]]


def test_oracle_cutouts_and_losses_equal_the_reference_modules_on_random_inputs():
    from oracle import guidance as og
    _, gold = _golden()
    for trial, B, H, W, x, seed, e, t, w in loss_cases():
        x = x.clone().requires_grad_()
        for name, fn in (("range", og.range_loss), ("tv", og.tv_loss)):
            a = fn(x)
            ga = th.autograd.grad((a * seed).sum(), x)[0]
            _close(a, gold[f"loss{trial}_{name}"], f"loss{trial}_{name}", 1e-6)
            _close(ga, gold[f"loss{trial}_{name}_grad"], f"loss{trial}_{name}_grad", 1e-6)
        e = e.clone().requires_grad_()
        a = og.spherical_dist_loss(e, t)
        _close(a, gold[f"loss{trial}_sph"], f"loss{trial}_sph", 1e-6)
        _close(th.autograd.grad(a.sum(), e)[0], gold[f"loss{trial}_sph_grad"], f"loss{trial}_sph_grad", 1e-6)
        if w is not None:
            th.manual_seed(trial)
            got = og.MakeCutouts(32, 4)(x)
            _close(got, gold[f"loss{trial}_cut"], f"loss{trial}_cut", 1e-6)
            _close(th.autograd.grad((got * w).sum(), x)[0], gold[f"loss{trial}_cut_grad"], f"loss{trial}_cut_grad", 1e-6)


def test_oracle_cond_fn_equals_the_live_reference_closure_on_random_configurations():
    """the committed cond_fn goldens widened: 40 random (batch, prompts, image size, cutouts, power, chain length, timestep, scales,
    saturation, magnitude) configurations, reference closure (cgd/cgd.py:151-239, compiled from its source) vs `OracleCondFn`"""
    from oracle import guidance as og
    from tests.test_cond_fn_reference import StubClip, stub_pred_xstart
    _, gold = _golden()
    for c in cond_cases():
        trial, B, t = c["trial"], c["B"], c["t"]
        cond = og.OracleCondFn(c["diff"], StubClip(32, 16), c["target"], c["w"], cut_size=32, num_cutouts=c["cutn"], cutout_power=c["power"],
                               sat_scale=c["sat"], use_magnitude=c["mag"], **c["scales"])
        cond.current_timestep = t
        th.manual_seed(trial)
        xr = c["x"].clone().requires_grad_()
        got = cond(xr, th.full((B,), t), {"pred_xstart": stub_pred_xstart(xr)})
        _close(got, gold[f"cond{trial}"], f"cond{trial}", 1e-5)
