"""Where the time of a tile goes in the persistent conv kernel (csrc/conv_tc.cu `conv_tc_persistent_kernel`).

Builds a copy of the library with -DCGD_CONV_PHASES in a temporary directory: the kernel then records %globaltimer stamps per CTA
and tile (see `CGD_PHASE` in conv_tc.cu).  Runs the four 256 x 256 3x3 convs of scripts/conv_tile_overhead.py (Cout 256, Cin 64 …
512, BN 256) and the Cin 256 layer with a residual, each once after warm-up, and prints per-tile means over all CTAs:
    wait   consumer thread 0 enters the tile's K loop -> its first full-barrier pass (operands not yet in the ring)
    K loop first full-barrier pass -> the end of the K loop (wgmma wait_group 0)
    epi    end of the K loop -> end of the epilogue as seen by consumer thread 0
    blocked the producer's time blocked on empty barriers while loading the tile
The first tile of each CTA (launch and pipeline fill) and the later ones are shown apart.

    python scripts/conv_tile_phases.py
"""
import ctypes, os, shutil, subprocess, sys, tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CTAS, SLOTS, FIELDS = 256, 32, 5  # kPhaseCtas, kPhaseTiles, kPhaseFields of conv_tc.cu
SHAPES = [(64, False), (128, False), (256, False), (512, False), (256, True)]


def build_variant(tmp):
    pkg = os.path.join(ROOT, "clip_guided_diffusion_b200")
    shutil.copytree(pkg, os.path.join(tmp, "clip_guided_diffusion_b200"),
                    ignore=shutil.ignore_patterns("__pycache__", "*.so", "conv_tc.o"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, "include"))
    env = dict(os.environ, CGD_NVCC_EXTRA=(os.environ.get("CGD_NVCC_EXTRA", "") + " -DCGD_CONV_PHASES").strip())
    subprocess.run([sys.executable, "-c", "from clip_guided_diffusion_b200 import build; build.build()"], cwd=tmp, env=env, check=True)


def stamps_of_one_launch(cin, res, read):
    import torch as th
    from clip_guided_diffusion_b200 import plan as P
    th.manual_seed(0)
    plan = P.Plan()
    cw = P.pack_conv(plan, th.randn(256, cin, 3, 3) * (9 * cin) ** -0.5, th.zeros(256), need_bwd=False, name="w")
    x = plan.act(1, 256, 256, cin, "x")
    r = plan.act(1, 256, 256, 256, "r") if res else None
    plan.conv(x, cw, res=r, name="c")
    plan.finalize("cuda")
    for b in plan.bufs:
        if b.name in ("x", "r"):
            plan.view(b).normal_()
    for _ in range(3):
        plan.run()
    read()
    plan.run()
    return read(), plan.ops[-1].i[16], -(-P.conv_tile_count(1, 256, 256) * 256 // plan.ops[-1].i[16])


def main():
    import numpy as np
    with tempfile.TemporaryDirectory() as tmp:
        build_variant(tmp)
        sys.path.insert(0, tmp)
        import torch as th
        from clip_guided_diffusion_b200 import _lib  # the instrumented copy: imported before bench puts ROOT first on sys.path
        assert _lib.LIB_PATH.startswith(tmp), _lib.LIB_PATH
        sys.path.insert(1, ROOT)
        import bench
        assert th.cuda.is_available(), "conv_tile_phases.py times kernels: it needs a CUDA device"
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True).stdout.strip()
        print(f"GPU: {th.cuda.get_device_name(0)} | nvidia-smi name, power limit, max SM clock: {smi}", flush=True)
        lib = _lib.load()
        fn = lib.cgd_conv_phases
        fn.argtypes = [ctypes.c_void_p, ctypes.c_int]
        buf = np.zeros(CTAS * SLOTS * FIELDS, np.uint64)

        def read():
            assert fn(buf.ctypes.data, buf.size) == 0, "cgd_conv_phases failed"
            return buf.reshape(CTAS, SLOTS, FIELDS).astype(np.int64).copy()

        sampler = bench.ClockSampler(0)
        sampler.start()
        print(f"{'layer':24s} {'BN':>3s} {'tiles':>5s} | {'tile':5s} {'n':>4s} {'wait':>6s} {'K loop':>7s} {'us/kb':>6s} {'epi':>6s} {'blocked':>7s}  (us)")
        for cin, res in SHAPES:
            s, bn, tiles = stamps_of_one_launch(cin, res, read)
            kb = 9 * cin // 64
            name = f"256x256 {cin}->256 3x3{' res' if res else ''}"
            done = s[:, :, 3] > 0
            for label, sel in (("first", np.arange(SLOTS) == 0), ("later", np.arange(SLOTS) > 0)):
                m = done & sel[None, :]
                if not m.any():
                    continue
                ph = s[m]
                wait, kl, epi = (ph[:, 1] - ph[:, 0]) / 1e3, (ph[:, 2] - ph[:, 1]) / 1e3, (ph[:, 3] - ph[:, 2]) / 1e3
                print(f"{name:24s} {bn:3d} {tiles:5d} | {label:5s} {int(m.sum()):4d} {wait.mean():6.2f} {kl.mean():7.2f} {kl.mean() / kb:6.3f} "
                      f"{epi.mean():6.2f} {ph[:, 4].mean() / 1e3:7.2f}", flush=True)
        print(f"SM clock during the runs: {sampler.stop()}")


if __name__ == "__main__":
    main()
