"""Times single conv layers alone (rotating buffers > L2, CUDA events) for a list of shapes.  Usage: python scripts/conv_microbench.py [bn]"""
import os, sys
import torch as th
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from clip_guided_diffusion_b200 import plan as P

SHAPES = [  # NB, H, W, Cin, Cout, taps, res
    (1, 256, 256, 256, 256, 9, False),
    (1, 256, 256, 256, 256, 9, True),
    (1, 128, 128, 256, 256, 9, False),
    (1, 128, 128, 512, 512, 9, False),
    (1, 64, 64, 512, 512, 9, False),
    (1, 32, 32, 512, 512, 9, False),
    (1, 16, 16, 1024, 1024, 9, False),
    (1, 8, 8, 1024, 1024, 9, False),
    (1, 256, 256, 256, 512, 1, False),
    (1, 256, 256, 512, 256, 1, False),
    (1, 1, 800, 768, 3072, 1, False),
    (1, 1, 800, 3072, 768, 1, False),
    (1, 1, 800, 768, 768, 1, False),
]
force_bn = int(sys.argv[1]) if len(sys.argv) > 1 else 0
if force_bn:
    P.pick_bn = lambda npad, m_tiles, kblocks=0: force_bn
dev = th.device("cuda", 0)
for (NB, H, W, Cin, Cout, taps, res) in SHAPES:
    th.manual_seed(0)
    plan = P.Plan()
    k = 3 if taps == 9 else 1
    w = th.randn(Cout, Cin, k, k) * (taps * Cin) ** -0.5
    cw = P.pack_conv(plan, w, th.zeros(Cout), need_bwd=False, name="w")
    act_bytes = NB * H * W * (Cin + Cout * (2 if res else 1)) * 2
    nbuf = max(2, min(16, int(300e6 // act_bytes) + 1))
    for _ in range(nbuf):
        x = plan.act(NB, H, W, Cin, "x")
        r = plan.act(NB, H, W, Cout, "r") if res else None
        plan.conv(x, cw, res=r, name="c")
    plan.finalize(dev)
    for b in plan.bufs:
        if b.name in ("x", "r"):
            plan.view(b).normal_()
    for _ in range(2):
        plan.run()
    th.cuda.synchronize()
    e0, e1 = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
    rounds = max(1, 48 // nbuf)
    e0.record()
    for _ in range(rounds):
        plan.run()
    e1.record()
    th.cuda.synchronize()
    t = e0.elapsed_time(e1) * 1e-3 / (rounds * nbuf)
    op = [o for o in plan.ops if o.code == 1][0]
    fl = 2.0 * NB * H * W * Cout * taps * Cin
    print(f"{NB}x{H}x{W} {Cin}->{Cout} t{taps} res{int(res)} BN{op.i[16]} sp{op.i[17]}: {t * 1e6:8.1f} us {fl / t / 1e12:8.1f} TF/s", flush=True)
    del plan
