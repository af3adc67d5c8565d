"""Pair every op of the cfg2 step plan (or of the bench workload named by CGD_PROFILE_WORKLOAD; rebuilt on the CPU, shapes only) with its
launch(es) in an ncu gpu__time_duration launch list of scripts/profile_step.py eager, and print time by op kind and shape.

    python scripts/op_report.py profiles/launches_cfg2_step.csv [kind-filter]
"""
import collections, csv, os, re, sys
import torch as th
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from clip_guided_diffusion_b200 import plan as P

P.Plan.const = lambda self, t, dt, name="": self.new(t.numel(), dt, name)
P.Plan.finalize = lambda self, device: self
import bench
from clip_guided_diffusion_b200 import weights as pw
from clip_guided_diffusion_b200 import guidance as pg
pw.seeded_state_dict = lambda shapes, seed=0: {k: th.empty(v) for k, v in shapes.items()}
pg.GuidedStepB200.set_targets = lambda *a, **k: None


def load_launches(path):
    rows = list(csv.reader(open(path)))
    for i, r in enumerate(rows):
        if 'Kernel Name' in r:
            hdr, start = r, i + 1
            break
    ki, mi, ui = hdr.index('Kernel Name'), hdr.index('Metric Value'), hdr.index('Metric Unit')
    out = []
    for r in rows[start:]:
        if len(r) <= mi:
            continue
        v = float(r[mi].replace(',', ''))
        v = v / 1e3 if r[ui] == 'ns' else (v * 1e3 if r[ui] == 'ms' else v)
        name = re.sub(r'\(.*', '', r[ki])
        if name.startswith('void at::'):
            continue
        out.append((name, v))
    return out


def shape_of(kind, op):
    i = op.i
    if kind == "CONV":
        return f"{i[0]}x{i[1]}x{i[2]} {i[3]}->{i[4]} t{i[6]} BN{i[16]} {'cl' if len(i) > 23 and i[23] else 'sp'}{i[17]}" + (" res" if op.p[3] is not None else "") + (" f32" if op.flags & 1 else "")
    if kind.startswith("GN_"):
        return f"N{i[0]} HW{i[1]} C{i[2]} fl{op.flags}" + (f" CS{i[5] if kind == 'GN_FWD_FUSED' else i[6]}" if "FUSED" in kind else "")
    return " ".join(str(v) for v in i[:6])


def main():
    launches = load_launches(sys.argv[1])
    filt = sys.argv[2] if len(sys.argv) > 2 else None
    if os.environ.get("CGD_PROFILE_WORKLOAD"):
        bench.CFG = bench.WORKLOADS[os.environ["CGD_PROFILE_WORKLOAD"]]
    ddim = bench.CFG["respacing"].startswith("ddim")
    eng, diff, cond = bench.build_engine(th.device("cpu"), 0, 1)
    plan, m = eng.plan, eng.plan.marks
    segs = [("unet_emb", "unet_bwd"), ("pmv", "cond"), ("cut_fwd", "sph"), ("vit_fwd", "vit_bwd"), ("sph", "cut_bwd"), ("vit_bwd", "vit_end"),
            ("cut_bwd", "guide"), ("guide", "final"), ("unet_bwd", "unet_end"), ("final", "upd_anc_g"), ("upd_ddim_g", "upd_ddim") if ddim else ("upd_anc_g", "upd_anc")]
    ops = []
    for a, b in segs:
        ops += plan.ops[m[a]:m[b]]
    inv = {v: k for k, v in P.OP.items()}
    li = 0
    kinds = collections.defaultdict(lambda: [0, 0.0])
    shapes = collections.defaultdict(lambda: [0, 0.0])
    for op in ops:
        kind = inv[op.code]
        n = 1
        if kind == "CONV" and op.i[17] > 1 and not (len(op.i) > 23 and op.i[23]):
            n = 2
        elif kind == "ATTN_BWD":
            n = 1 if op.i[2] <= 64 and op.i[3] == 64 else 2
        elif kind == "FINAL_GRAD" and op.flags & 1:
            n = 2
        t = sum(v for _, v in launches[li:li + n])
        li += n
        kinds[kind][0] += 1; kinds[kind][1] += t
        s = shapes[(kind, shape_of(kind, op))]; s[0] += 1; s[1] += t
    assert li == len(launches), (li, len(launches))
    tot = sum(v[1] for v in kinds.values())
    print(f"total {tot:.1f} us over {li} launches")
    for k, (n, t) in sorted(kinds.items(), key=lambda kv: -kv[1][1]):
        print(f"{k:16s} n={n:4d} {t:9.1f} us {100 * t / tot:5.1f}%")
    print("--- by shape")
    for (k, s), (n, t) in sorted(shapes.items(), key=lambda kv: -kv[1][1]):
        if filt and filt not in k:
            continue
        print(f"{k:14s} {s:48s} n={n:3d} {t:9.1f} us ({t / n:7.1f} each) {100 * t / tot:5.1f}%")


main()
