"""One launch of every kernel family of the cfg2 guided step inside a cudaProfilerStart/Stop range, for
    ncu --set full --clock-control none --import-source on --profile-from-start off -o profiles/families python scripts/profile_families.py
The engine runs two eager steps first (every buffer holds real data), then the chosen ops are launched one by one: for each op code
the instance(s) with the most work, for CONV one per kernel variant / regime (wgmma tile kernel 3x3 dominant, with residual, 1x1, in-cluster
split-K, workspace split-K + reduce, fp32 NCHW head / stem dgrad, ViT GEMMs)."""
import os
import sys

import torch as th

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from tests.plan_interp import CODE  # noqa: E402  (op code -> name only)

th.cuda.set_device(0)
eng, diff, cond = bench.build_engine(th.device("cuda", 0), 0, 1)
eng.use_graph = False
th.manual_seed(0)
img = eng.draw_initial_noise()
i = diff.num_timesteps - 1
for _ in range(2):
    img = eng.fused_step(diff, "ddim", i, img, eng.draw_classes(), cond, 0.0)["sample"]
    cond.step_done()
    i -= 1
th.cuda.synchronize()
plan = eng.plan
m = plan.marks
step_ops = [k for a, b in (("unet_emb", "unet_bwd"), ("pmv", "cond"), ("cut_fwd", "sph"), ("vit_fwd", "vit_bwd"), ("sph", "cut_bwd"), ("vit_bwd", "vit_end"),
                           ("cut_bwd", "cut_end"), ("guide", "final"), ("unet_bwd", "unet_end"), ("final", "upd_anc_g"), ("upd_ddim_g", "upd_ddim"))
            for k in range(m[a], m[b])]


def work(op):
    name = CODE[op.code]
    if name == "CONV":
        return 2.0 * op.i[0] * op.i[1] * op.i[2] * op.i[3] * op.i[4] * op.i[6]
    if name.startswith("ATTN"):
        return float(op.i[0] * op.i[1] * op.i[2] * op.i[2])
    if name.startswith("GN_") or name.startswith("LN_"):
        return float(op.i[0] * op.i[1] * op.i[2])
    return float(max(1, op.i[0]) * max(1, op.i[1] if len(op.i) > 1 else 1))


chosen, seen = [], set()
for k in sorted(step_ops, key=lambda k: -work(plan.ops[k])):
    op = plan.ops[k]
    name = CODE[op.code]
    if name == "CONV":
        NB, H, W, Cin, Cout, npad, taps = op.i[:7]
        bn, splits, cluster, f32 = op.i[16], op.i[17], op.i[23], op.flags & 1
        key = ("CONV", taps, "hw%d" % (H * W if H * W in (65536, 16384, 4096, 1024, 256, 64) else 0), bn, min(splits, 2), cluster, f32, bool(op.p[3]))
    elif name.startswith("ATTN"):
        key = (name, op.i[2])
    elif name.startswith("GN_"):
        key = (name, op.i[1] >= 16384)
    else:
        key = (name,)
    if key in seen:
        continue
    seen.add(key)
    chosen.append(k)
only = [v for v in os.environ.get("PF_ONLY", "").split(",") if v]
if only:  # e.g. PF_ONLY=GN_APPLY_EPI,CONV_STATS with CGD_GN_EPI_STATS=1
    def label(op):
        return "CONV_STATS" if CODE[op.code] == "CONV" and (op.flags & 2) else CODE[op.code]
    chosen = [k for k in chosen if label(plan.ops[k]) in only]
    for want in only:  # make sure the biggest instance of each requested kind is there even if its key collided
        cands = [k for k in step_ops if label(plan.ops[k]) == want]
        if cands and not any(label(plan.ops[k]) == want for k in chosen):
            chosen.append(max(cands, key=lambda k: work(plan.ops[k])))
chosen.sort()
print("profiling", len(chosen), "launch groups:")
for k in chosen:
    op = plan.ops[k]
    print(f"  op {k:4d} {CODE[op.code]:18s} {op.tag[:40]:40s} i={list(op.i)[:8]} f={op.flags}")
th.cuda.synchronize()
th.cuda.profiler.start()
for k in chosen:
    plan.run(k, 1)
th.cuda.synchronize()
th.cuda.profiler.stop()
print("done")
