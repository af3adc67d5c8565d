"""Fixed cost per output tile of the one-CTA conv path (csrc/conv_tc.cu), separated from the cost per K-block.

Times 256 x 256 3x3 convs with Cout = 256 at Cin = 64, 128, 256, 512 (9, 18, 36, 72 K-blocks of 64 channels).  The plan picks
BN = 256 for all four: 512 tiles of 128 pixels x 256 channels, so ceil(512 / SMs) rounds of one tile per SM.  A least-squares line
through (K-blocks, time / rounds) gives `a`, the cost of a tile that is not the K loop (launch, pipeline fill, epilogue, stores,
drain), and `b`, the cost of one K-block (four wgmma.m64n256k16 per consumer warpgroup).  Times: CUDA events over rotating buffers
larger than the L2.

    python scripts/conv_tile_overhead.py
"""
import os, subprocess, sys
import numpy as np
import torch as th
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from clip_guided_diffusion_b200 import plan as P

CINS = (64, 128, 256, 512)


def time_conv(cin, cout=256, hw=256, reps=48):
    th.manual_seed(0)
    plan = P.Plan()
    cw = P.pack_conv(plan, th.randn(cout, cin, 3, 3) * (9 * cin) ** -0.5, th.zeros(cout), need_bwd=False, name="w")
    nbuf = max(2, min(16, int(300e6 // (hw * hw * (cin + cout) * 2)) + 1))
    for _ in range(nbuf):
        plan.conv(plan.act(1, hw, hw, cin, "x"), cw, name="c")
    plan.finalize("cuda")
    bn = plan.ops[-1].i[16]
    for b in plan.bufs:
        if b.name == "x":
            plan.view(b).normal_()
    for _ in range(2):
        plan.run()
    th.cuda.synchronize()
    e0, e1 = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
    rounds = max(1, reps // nbuf)
    ts = []
    for _ in range(5):
        e0.record()
        for _ in range(rounds):
            plan.run()
        e1.record()
        th.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e-3 / (rounds * nbuf))
    return sorted(ts)[2], bn


def main():
    assert th.cuda.is_available(), "conv_tile_overhead.py times kernels: it needs a CUDA device"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    print(f"GPU: {th.cuda.get_device_name(0)} | nvidia-smi name, power limit, max SM clock: {smi}", flush=True)
    sms = th.cuda.get_device_properties(0).multi_processor_count
    sampler = bench.ClockSampler(0)
    sampler.start()
    xs, ys = [], []
    print(f"{'Cin':>4s} {'kblocks':>7s} {'BN':>3s} {'tiles':>5s} {'rounds':>6s} | {'us':>7s} {'us/round':>8s} {'TF/s':>6s}")
    for cin in CINS:
        t, bn = time_conv(cin)
        kb = 9 * cin // 64
        tiles = P.conv_tile_count(1, 256, 256) * (256 // bn)
        rounds = -(-tiles // sms)
        fl = 2.0 * 256 * 256 * 256 * 9 * cin
        xs.append(kb)
        ys.append(t / rounds)
        print(f"{cin:4d} {kb:7d} {bn:3d} {tiles:5d} {rounds:6d} | {t * 1e6:7.1f} {t / rounds * 1e6:8.2f} {fl / t / 1e12:6.1f}", flush=True)
    b, a = np.polyfit(np.array(xs, float), np.array(ys, float), 1)
    print(f"fit t/round = a + b * kblocks: a = {a * 1e6:.2f} us per tile, b = {b * 1e6:.3f} us per K-block")
    print(f"SM clock during the timings: {sampler.stop()}")


if __name__ == "__main__":
    main()
