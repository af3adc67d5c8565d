"""What encoding text prompts on the device costs, printed as one JSON line beside the card's name and power limit:

1. building the forward-only text tower (``TextB200``: weight packing, upload, plan creation) and one encode, for 1, 8 and 32
   prompts, at the B/32 text tower's size (width 512) and L/14's (width 768), 12 layers, 77 tokens, seeded weights;
2. ATTN_FWD at T = 77 (8 heads of 64, 32 sequences: the B/32 tower at 32 prompts) causal against non-causal, CUDA events over
   many launches.

    python scripts/text_encode_cost.py [--out DIR]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
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


def _ids(cfg, n, seed=0):
    g = th.Generator().manual_seed(seed)
    ids = th.zeros(n, cfg.context_length, dtype=th.int32)
    for i in range(n):
        L = int(th.randint(3, cfg.context_length + 1, (1,), generator=g))
        ids[i, 0], ids[i, L - 1] = cfg.vocab_size - 2, cfg.vocab_size - 1
        ids[i, 1:L - 1] = th.randint(1, cfg.vocab_size - 2, (L - 2,), generator=g)
    return ids


def time_towers():
    from clip_guided_diffusion_b200 import text as ptx, weights as pw
    res = {}
    for width in (512, 768):
        cfg = ptx.TextConfig(width=width, layers=12, output_dim=width)
        sd = pw.seeded_state_dict(pw.text_param_shapes(cfg), width)
        ptx.TextB200(cfg, sd, 1).encode(_ids(cfg, 1))  # warm-up: module load, kernel attributes
        th.cuda.synchronize()
        for n in (1, 8, 32):
            ids = _ids(cfg, n, seed=n)
            builds, first, again = [], [], []
            for _ in range(3):
                t0 = time.perf_counter()
                tower = ptx.TextB200(cfg, sd, n)
                th.cuda.synchronize()
                t1 = time.perf_counter()
                tower.encode(ids)
                th.cuda.synchronize()
                t2 = time.perf_counter()
                builds.append(t1 - t0)
                first.append(t2 - t1)
                for _ in range(5):
                    t3 = time.perf_counter()
                    tower.encode(ids)
                    th.cuda.synchronize()
                    again.append(time.perf_counter() - t3)
                del tower
            res[f"w{width}_n{n}"] = {"build_ms": round(1e3 * sorted(builds)[1], 2), "first_encode_ms": round(1e3 * sorted(first)[1], 3),
                                     "encode_ms": round(1e3 * sorted(again)[len(again) // 2], 3)}
    return res


def time_attention(iters=2000):
    from clip_guided_diffusion_b200 import _lib
    B, heads, T, d = 32, 8, 77, 64
    C = heads * d
    qkv = th.randn(B, T, 3 * C, device="cuda").half()
    out = th.empty(B, T, C, device="cuda", dtype=th.float16)
    lse = th.empty(B, heads, T, device="cuda")
    lib = _lib.load()
    st = ctypes.c_void_p(th.cuda.current_stream().cuda_stream)
    ops = {}
    for name, flags in (("non_causal", 0), ("causal", 1)):
        op = _lib.CgdOp()
        op.code, op.flags = _lib.OP["ATTN_FWD"], flags
        for j, v in enumerate([B, heads, T, d, T * 3 * C, 3 * C, d, T * C, C, d]):
            op.i[j] = v
        op.f[0] = d ** -0.5
        for j, t in enumerate([qkv, qkv[..., C:], qkv[..., 2 * C:], out, lse]):
            op.p[j] = t.data_ptr()
        ops[name] = op
    times = {k: [] for k in ops}
    for rnd in range(7):
        for name, op in (ops.items() if rnd % 2 == 0 else reversed(list(ops.items()))):
            for _ in range(50):
                _lib.check(lib.cgd_run_op(ctypes.byref(op), st))
            a, b = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                lib.cgd_run_op(ctypes.byref(op), st)
            b.record()
            b.synchronize()
            times[name].append(1e3 * a.elapsed_time(b) / iters)
    return {f"attn_fwd_T77_B32_h8_{k}_us": round(sorted(v)[len(v) // 2], 3) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/text_encode_cost.json")
    args = ap.parse_args()
    if not th.cuda.is_available():
        raise SystemExit("text_encode_cost.py measures the device: no CUDA device found")
    res = {**card(), "towers": time_towers(), **time_attention()}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "text_encode_cost.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
