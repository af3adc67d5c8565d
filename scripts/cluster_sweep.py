"""In-cluster split-K (csrc/conv_tc.cu, CONV i23) against the workspace split-K + reduce launch, per latency-bound layer shape: cluster
capacities of the device, then every (BN, S) timed inside a CUDA graph over rotating buffers.  python scripts/cluster_sweep.py"""
import os, sys
import torch as th
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from clip_guided_diffusion_b200 import plan as P
from clip_guided_diffusion_b200 import _lib

lib = _lib.load()
print("cluster capacity (clusters co-resident) by (BN, S):",
      {(bn, S): lib.cgd_conv_cluster_capacity(bn, S) for bn in (64, 128, 192, 256) for S in (1, 2, 4, 8)}, flush=True)
SHAPES = [(1, 8, 8, 1024, 1024, 9), (1, 16, 16, 1024, 1024, 9), (1, 32, 32, 512, 512, 9), (1, 1, 800, 3072, 768, 1), (1, 1, 800, 2304, 768, 1),
          (1, 16, 16, 3072, 1024, 1), (1, 64, 64, 256, 256, 9)]
dev = th.device("cuda", 0)
ORIG_PICK = P.pick_cluster_split


def time_plan(NB, H, W, Cin, Cout, taps):
    th.manual_seed(0)
    plan = P.Plan()
    k = 3 if taps == 9 else 1
    cw = P.pack_conv(plan, th.randn(Cout, Cin, k, k) * (taps * Cin) ** -0.5, th.zeros(Cout), need_bwd=False, name="w")
    nbuf = 8
    for _ in range(nbuf):
        plan.conv(plan.act(NB, H, W, Cin, "x"), cw, name="c")
    plan.finalize(dev)
    for b in plan.bufs:
        if b.name == "x":
            plan.view(b).normal_()
    plan.run(); plan.run()
    th.cuda.synchronize()
    g = th.cuda.CUDAGraph()
    with th.cuda.graph(g):
        for _ in range(4):
            plan.run()
    g.replay(); th.cuda.synchronize()
    e0, e1 = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        g.replay()
    e1.record(); th.cuda.synchronize()
    op = [o for o in plan.ops if o.code == 1][0]
    return e0.elapsed_time(e1) * 1e-3 / (5 * 4 * nbuf) * 1e6, op


for shp in SHAPES:
    NB, H, W, Cin, Cout, taps = shp
    kb = taps * Cin // 64
    mt = P.conv_tile_count(NB, H, W)
    P.pick_cluster_split = lambda *a: None
    t, op = time_plan(*shp)
    print(f"{NB}x{H}x{W} {Cin}->{Cout} t{taps}: workspace split BN{op.i[16]} sp{op.i[17]}: {t:6.1f} us", flush=True)
    P.pick_cluster_split = ORIG_PICK
    t, op = time_plan(*shp)
    print(f"    plan's pick: BN{op.i[16]} {'cl' if op.i[23] else 'sp'}{op.i[17]}: {t:6.1f} us", flush=True)
    for bn in (64, 128, 192, 256):
        if P._npad(Cout) % bn:
            continue
        for S in (2, 4, 8):
            kps = -(-kb // S)
            if bn % S or (bn // S) % 16 or kps < 2 or (S - 1) * kps >= kb:
                continue
            P.pick_cluster_split = lambda m, n, k, c, bn=bn, S=S: (bn, S, 0.0)
            t, op = time_plan(*shp)
            tiles = mt * (P._npad(Cout) // bn)
            print(f"    BN{bn:3d} cl{S}: {tiles:3d} clusters x {S:2d} CTAs, {kps:3d} K-blocks/CTA: {t:6.1f} us", flush=True)
    P.pick_cluster_split = ORIG_PICK
