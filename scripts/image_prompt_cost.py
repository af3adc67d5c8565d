"""What image prompts cost on the device, printed as one JSON line beside the card's name and power limit:

1. ``encode_image_prompt`` for a 1024 x 768 PNG at 256^2 with ViT-B/32 and 16 cutouts (seeded weights): the whole call (the
   forward-only tower is built inside it) and the encode alone on an already built ``ImagePromptEncoder``;
2. the SPHERICAL op (spherical distance loss and its gradient over P target embeddings) at P = 1, 17 (text + one image prompt at
   16 cutouts) and 65 (text + one image prompt at 64 cutouts, ViT-L/14's D = 768), CUDA events over many launches;
3. the cfg2 guided step (256^2, ddim250, ViT-B/32, 16 cutouts) with one text prompt (P = 1) against one text and one image prompt
   (P = 17), CUDA events around replays of the step's graph.

    python scripts/image_prompt_cost.py [--out DIR]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (v.strip() for v in q.split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001 -- the numbers stay valid, only their label is missing
        return {"gpu": th.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def time_encode(tmp):
    from PIL import Image
    from clip_guided_diffusion_b200 import cgd, image_prompt as pip, vit as pv, weights as pw
    cfg = pv.VIT_CONFIGS["ViT-B/32"]
    sd = pw.seeded_state_dict(pw.vit_param_shapes(cfg), 1235)
    path = os.path.join(tmp, "prompt.png")
    g = th.Generator().manual_seed(0)
    Image.fromarray(th.randint(0, 256, (768, 1024, 3), generator=g, dtype=th.uint8).numpy()).save(path)
    cgd.encode_image_prompt(path, 1.0, 256, 16, clip_state_dict=sd)  # warm-up: module load, kernel attributes
    th.cuda.synchronize()
    calls = []
    for _ in range(3):
        t0 = time.perf_counter()
        cgd.encode_image_prompt(path, 1.0, 256, 16, clip_state_dict=sd)
        th.cuda.synchronize()
        calls.append(time.perf_counter() - t0)
    enc = pip.ImagePromptEncoder(cfg, sd, 16)
    enc.encode(path, 1.0, 256)
    th.cuda.synchronize()
    alone = []
    for _ in range(10):
        t0 = time.perf_counter()
        enc.encode(path, 1.0, 256)
        th.cuda.synchronize()
        alone.append(time.perf_counter() - t0)
    return {"encode_image_prompt_call_ms": round(1e3 * min(calls), 2), "encode_with_built_tower_ms": round(1e3 * min(alone), 3)}


def time_spherical():
    from clip_guided_diffusion_b200 import _lib
    lib = _lib.load()
    out = {}
    for P, cutn, D in ((1, 16, 512), (17, 16, 512), (65, 64, 768)):
        g = th.Generator(device="cuda").manual_seed(P)
        emb, tgt = th.randn(cutn, D, device="cuda", generator=g), th.randn(P, D, device="cuda", generator=g)
        w, d_emb, loss = th.full((P,), 1.0 / P, device="cuda"), th.empty(cutn, D, device="cuda"), th.zeros(1, device="cuda")
        op = _lib.CgdOp()
        op.code = _lib.OP["SPHERICAL"]
        for j, v in enumerate([cutn, 1, P, D]):
            op.i[j] = v
        op.f[0], op.f[1] = 1000.0, 1.0
        for j, t in enumerate([emb, tgt, w, d_emb, loss]):
            op.p[j] = t.data_ptr()
        st = ctypes.c_void_p(th.cuda.current_stream().cuda_stream)

        def run(n):
            for _ in range(n):
                _lib.check(lib.cgd_run_op(ctypes.byref(op), st), "spherical")
        run(50)
        a, b = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
        best = None
        for _ in range(5):
            a.record()
            run(500)
            b.record()
            b.synchronize()
            us = 1e3 * a.elapsed_time(b) / 500
            best = us if best is None else min(best, us)
        out[f"spherical_us_P{P}_cutn{cutn}_D{D}"] = round(best, 2)
    return out


def time_step(P, steps=30, warmup=5):
    import bench
    eng, diff, cond = bench.build_engine(th.device("cuda", 0), 0, 1)
    if P > 1:  # one text prompt and one image prompt's 16 cutout embeddings (weights as the entry normalises them)
        D = eng.towers[0].cfg.output_dim
        del eng, cond  # rebuilt with room for P targets
        th.cuda.empty_cache()
        from clip_guided_diffusion_b200 import guidance as pg
        from clip_guided_diffusion_b200 import unet as pu
        from clip_guided_diffusion_b200 import vit as pv
        from clip_guided_diffusion_b200 import weights as pw
        ucfg, vcfg = pu.config_for(256, class_cond=True), pv.VIT_CONFIGS["ViT-B/32"]
        eng = pg.GuidedStepB200(ucfg, pw.seeded_state_dict(pw.unet_param_shapes(ucfg), seed=1234), vcfg,
                                pw.seeded_state_dict(pw.vit_param_shapes(vcfg), seed=1235), batch=1, num_cutouts=16, max_prompts=P,
                                device="cuda")
        th.manual_seed(0)
        w = th.tensor([1.0] + [0.5 / (P - 1)] * (P - 1))
        eng.set_targets(th.nn.functional.normalize(th.randn(P, D), dim=-1), w / w.sum())
        cond = pg.CondFnB200(eng, diff, pg.MakeCutouts(vcfg.input_resolution, 16))
    th.manual_seed(0)
    img = eng.draw_initial_noise()
    i = diff.num_timesteps - 1
    for k in range(warmup + steps):
        if k == warmup:
            th.cuda.synchronize()
            a, b = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
            a.record()
        img = eng.fused_step(diff, "ddim", i, img, eng.draw_classes(), cond, 0.0)["sample"]
        cond.step_done()
        i -= 1
    b.record()
    b.synchronize()
    ms = a.elapsed_time(b) / steps
    del eng, cond
    th.cuda.empty_cache()
    return round(ms, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/image_prompt_cost.json")
    args = ap.parse_args()
    if not th.cuda.is_available():
        sys.exit("image_prompt_cost.py measures on the GPU; there is no CPU measurement")
    res = card()
    with tempfile.TemporaryDirectory() as tmp:
        res.update(time_encode(tmp))
    res.update(time_spherical())
    res["cfg2_step_ms_text_only_P1"] = time_step(1)
    res["cfg2_step_ms_text_and_image_P17"] = time_step(17)
    res["cfg2_step_ms_text_only_P1_again"] = time_step(1)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "image_prompt_cost.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
