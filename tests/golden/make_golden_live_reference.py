"""Writes tests/golden/live_reference_golden.{json.gz,npz}: what the reference returns for the random inputs of
tests/test_live_reference_diff.py -- its prompt helpers (function bodies of cgd/script_util.py cut out with `ast`; the module itself
does not import), `cgd.modules.MakeCutouts`, `cgd.losses` and the `cond_fn` closure of cgd/cgd.py.

    python tests/golden/make_golden_live_reference.py <path of a checkout of the reference>
"""
import ast
import gzip
import json
import os
import re
import sys

import numpy as np
import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main(ref_root):
    sys.path.insert(0, ROOT)
    from tests import test_live_reference_diff as T
    from tests.test_cond_fn_reference import StubClip, stub_pred_xstart
    sys.path.insert(0, ref_root)
    from cgd import losses, modules

    # prompt helpers
    ns = {"os": os, "re": re}
    src = open(os.path.join(ref_root, "cgd", "script_util.py")).read()
    for node in ast.parse(src).body:
        if isinstance(node, ast.FunctionDef) and node.name in ("parse_prompt", "alphanumeric_filter", "clean_and_combine_prompts"):
            exec(compile(ast.Module([node], []), "cgd/script_util.py", "exec"), ns)
    combine, prompts = T.prompt_cases()
    parse = []
    for p in prompts:
        try:
            parse.append(list(ns["parse_prompt"](p)))
        except ValueError:
            parse.append(None)
    js = {"prompts": {"combine": [[ns["alphanumeric_filter"](texts[0]), ns["clean_and_combine_prompts"]("base", texts, b)] for texts, b in combine],
                      "parse": parse}}

    # cutout windows and generator consumption
    ints = lambda cs: [[int(v) for v in c] for c in cs]
    cut = []
    for trial, cs, side_x, side_y, cutn, power in T.cutout_cases():
        ref = modules.MakeCutouts(cs, cutn, cutout_size_power=power)
        th.manual_seed(trial)
        coords = ints(ref._generate_coords(side_x, side_y, cutn))
        digest = T.rng_digest()
        th.manual_seed(trial + 1)
        ref.cache_coordinates(side_x, side_y)
        cut.append({"coords": coords, "rng": digest, "cached": ints(ref.cached_coords)})
    js["cutouts"] = cut
    ref = modules.MakeCutouts(224, 16)
    th.manual_seed(3)
    ref.cache_coordinates(256, 256)
    cached = ints(ref.cached_coords)
    th.manual_seed(4)
    js["coords_for"] = {"cached": cached, "fresh": ints(ref._generate_coords(256, 256, 8))}

    # losses and cutouts
    gold = {}
    for trial, B, H, W, x, seed, e, t, w in T.loss_cases():
        x = x.clone().requires_grad_()
        for name, fn in (("range", losses.range_loss), ("tv", losses.tv_loss)):
            a = fn(x)
            gold[f"loss{trial}_{name}"] = T.summarize(a, f"loss{trial}_{name}")
            gold[f"loss{trial}_{name}_grad"] = T.summarize(th.autograd.grad((a * seed).sum(), x)[0], f"loss{trial}_{name}_grad")
        e = e.clone().requires_grad_()
        a = losses.spherical_dist_loss(e, t)
        gold[f"loss{trial}_sph"] = T.summarize(a, f"loss{trial}_sph")
        gold[f"loss{trial}_sph_grad"] = T.summarize(th.autograd.grad(a.sum(), e)[0], f"loss{trial}_sph_grad")
        if w is not None:
            th.manual_seed(trial)
            want = modules.MakeCutouts(32, 4)(x)
            assert want.shape == w.shape, (want.shape, w.shape)
            gold[f"loss{trial}_cut"] = T.summarize(want, f"loss{trial}_cut")
            gold[f"loss{trial}_cut_grad"] = T.summarize(th.autograd.grad((want * w).sum(), x)[0], f"loss{trial}_cut_grad")

    # cond_fn closure: the nested function of clip_guided_diffusion() compiled from the reference's source, its free variables supplied
    import types
    import torchvision.transforms as tvt
    tree = ast.parse(open(os.path.join(ref_root, "cgd", "cgd.py")).read())
    outer = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "clip_guided_diffusion")
    code = compile(ast.Module([next(n for n in ast.walk(outer) if isinstance(n, ast.FunctionDef) and n.name == "cond_fn")], []), "cgd/cgd.py", "exec")
    tree = ast.parse(open(os.path.join(ref_root, "cgd", "clip_util.py")).read())
    node = next(n for n in tree.body if isinstance(n, ast.Assign) and getattr(n.targets[0], "id", "") == "CLIP_NORMALIZE")
    clip_normalize = eval(compile(ast.Expression(node.value), "cgd/clip_util.py", "eval"), {"tvt": tvt})

    def make_closure(**free):
        ns = dict(th=th, losses=losses, tqdm=types.SimpleNamespace(write=lambda *a, **k: None), wandb_project=None, progress=False,
                  clip_util=types.SimpleNamespace(CLIP_NORMALIZE=clip_normalize), lpips_vgg=None, init_tensor=None, init_scale=0,
                  reduce_clip=False, progressive_cutout=False, cached_cutouts=False, timestep_respacing="25")
        ns.update(free)
        exec(code, ns)
        return ns

    for c in T.cond_cases():
        trial, B, t, T_ = c["trial"], c["B"], c["t"], c["T"]
        nsc = make_closure(diffusion=types.SimpleNamespace(num_timesteps=T_, sqrt_one_minus_alphas_cumprod=c["diff"].sqrt_one_minus_alphas_cumprod),
                              current_timestep=t, num_cutouts=c["cutn"], make_cutouts=modules.MakeCutouts(32, c["cutn"], cutout_size_power=c["power"]),
                              clip_model=StubClip(32, 16), target_embeds=c["target"], weights=c["w"], sat_scale=c["sat"], use_saturation=c["sat"] != 0,
                              use_magnitude=c["mag"], **c["scales"])
        th.manual_seed(trial)
        xr = c["x"].clone().requires_grad_()
        want = nsc["cond_fn"](xr, th.full((B,), t), {"pred_xstart": stub_pred_xstart(xr)}).detach()
        gold[f"cond{trial}"] = T.summarize(want, f"cond{trial}")

    with gzip.open(os.path.join(ROOT, "tests", "golden", "live_reference_golden.json.gz"), "wt", encoding="utf-8") as f:
        json.dump(js, f, ensure_ascii=False, separators=(",", ":"))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "live_reference_golden.npz"), **gold)


if __name__ == "__main__":
    main(sys.argv[1])
