"""L2 -> SM operand traffic of the wide conv launches of the cfg2 step (one 128-pixel x BN tile per CTA, no split-K), next to their
measured time: does a layer run near a bandwidth limit of the L2, or does the same kernel move more bytes per second on another shape?
Bytes are the operand tiles the TMA copies from L2 into shared memory: per tile and K-block, 128 x 64 activations plus the BN x 64
weight slice (epilogue reads and writes are not counted).  The "half B" column is what the launch would move if pairs of CTAs shared
each weight slice (TMA multicast in a 2-CTA cluster).  Times: CUDA events over rotating buffers larger than the L2.

    python scripts/conv_l2_traffic.py
"""
import collections, os, subprocess, sys
import torch as th
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from clip_guided_diffusion_b200 import guidance as pg
from clip_guided_diffusion_b200 import plan as P
from clip_guided_diffusion_b200 import weights as pw
from clip_guided_diffusion_b200._lib import OP


def step_shapes():
    """{(NB, H, W, Cin, Cout, taps, res): [BN, launches per step]} over the CONV ops of one cfg2 step that run without split-K or a
    cluster split, BN >= 64, fp16 output.  The plan is built on the CPU with shapes only; the patched methods are restored afterwards."""
    saved = (P.Plan.const, P.Plan.finalize, pw.seeded_state_dict, pg.GuidedStepB200.set_targets)
    P.Plan.const = lambda self, t, dt, name="": self.new(t.numel(), dt, name)
    P.Plan.finalize = lambda self, device: self
    pw.seeded_state_dict = lambda shapes, seed=0: {k: th.empty(v) for k, v in shapes.items()}
    pg.GuidedStepB200.set_targets = lambda *a, **k: None
    try:
        eng, _, _ = bench.build_engine(th.device("cpu"), 0, 1)
    finally:
        P.Plan.const, P.Plan.finalize, pw.seeded_state_dict, pg.GuidedStepB200.set_targets = saved
    plan, m = eng.plan, eng.plan.marks
    segs = [("unet_emb", "unet_bwd"), ("vit_fwd", "vit_bwd"), ("vit_bwd", "vit_end"), ("unet_bwd", "unet_end")]
    out = collections.OrderedDict()
    for a, b in segs:
        for op in plan.ops[m[a]:m[b]]:
            i = op.i
            if op.code != OP["CONV"] or i[17] != 1 or i[23] or i[16] < 64 or op.flags & 1:
                continue
            key = (i[0], i[1], i[2], i[3], i[4], i[6], op.p[3] is not None)
            out.setdefault(key, [i[16], 0])[1] += 1
    return out


def time_launch(shape):
    NB, H, W, Cin, Cout, taps, res = shape
    th.manual_seed(0)
    plan = P.Plan()
    k = 3 if taps == 9 else 1
    cw = P.pack_conv(plan, th.randn(Cout, Cin, k, k) * (taps * Cin) ** -0.5, th.zeros(Cout), need_bwd=False, name="w")
    act_bytes = NB * H * W * (Cin + Cout * (2 if res else 1)) * 2
    nbuf = max(2, min(16, int(300e6 // act_bytes) + 1))
    for _ in range(nbuf):
        x = plan.act(NB, H, W, Cin, "x")
        r = plan.act(NB, H, W, Cout, "r") if res else None
        plan.conv(x, cw, res=r, name="c")
    plan.finalize("cuda")
    for b in plan.bufs:
        if b.name in ("x", "r"):
            plan.view(b).normal_()
    for _ in range(2):
        plan.run()
    th.cuda.synchronize()
    e0, e1 = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
    rounds = max(1, 48 // nbuf)
    ts = []
    for _ in range(3):
        e0.record()
        for _ in range(rounds):
            plan.run()
        e1.record()
        th.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e-3 / (rounds * nbuf))
    return sorted(ts)[1]


def l2_bytes(shape, bn, half_b=False):
    NB, H, W, Cin, Cout, taps, _ = shape
    npad = -(-Cout // bn) * bn
    tiles = P.conv_tile_count(NB, H, W) * (npad // bn)
    return tiles * (taps * Cin // 64) * (128 * 64 * 2 + (bn // 2 if half_b else bn) * 64 * 2)


def main():
    assert th.cuda.is_available(), "conv_l2_traffic.py times kernels: it needs a CUDA device"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    print(f"GPU: {th.cuda.get_device_name(0)} | nvidia-smi name, power limit, max SM clock: {smi}", flush=True)
    shapes = step_shapes()
    sampler = bench.ClockSampler(0)
    sampler.start()
    print(f"{'shape':34s} {'BN':>3s} {'n/step':>6s} | {'us':>7s} {'TF/s':>6s} | {'L2->SM MB':>9s} {'TB/s':>5s} | {'half B MB':>9s}")
    for shape, (bn, n) in shapes.items():
        NB, H, W, Cin, Cout, taps, res = shape
        t = time_launch(shape)
        fl = 2.0 * NB * H * W * Cout * taps * Cin
        b = l2_bytes(shape, bn)
        name = f"{NB}x{H}x{W} {Cin}->{Cout} {'3x3' if taps == 9 else '1x1'}{' res' if res else ''}"
        print(f"{name:34s} {bn:3d} {n:6d} | {t * 1e6:7.1f} {fl / t / 1e12:6.1f} | {b / 1e6:9.0f} {b / t / 1e12:5.2f} | {l2_bytes(shape, bn, True) / 1e6:9.0f}",
              flush=True)
    print(f"SM clock during the timings: {sampler.stop()}")


if __name__ == "__main__":
    main()
