"""GPU test helpers: run a plan natively (libcgd_b200) and with the PyTorch interpreter on identical inputs, op by op."""
import copy

import torch as th

from clip_guided_diffusion_b200._lib import OP
from clip_guided_diffusion_b200.plan import _DT
from tests.plan_interp import CODE, Interp

# output pointer slots per op code (whole owning buffers are compared)
OUT_PTRS = {"CONV": [4], "GN_STATS": [2], "GN_APPLY": [5], "GN_BWD_STATS": [7], "GN_BWD_APPLY": [7], "POOL2": [1], "UP2": [1], "ADD": [2],
            "COPY": [1], "ATTN_FWD": [3, 4], "ATTN_BWD": [6], "LINEAR_SMALL": [3], "TIMESTEP_EMB": [1], "LABEL_ADD": [0], "NCHW_TO_PM": [1],
            "PM_TO_NCHW": [1], "LN_FWD": [3, 4], "LN_BWD": [4], "QGELU_FWD": [1], "QGELU_BWD": [2], "VIT_EMBED": [0], "CUTOUTS_FWD": [2],
            "CUTOUTS_BWD": [2], "SPHERICAL": [3, 4], "PMV_BLEND": [3, 4, 5, 6, 7], "GUIDE_GRAD": [4, 5, 6, 7, 8], "FINAL_GRAD": [2, 4], "SEED_QUANT": [1, 2], "MAG_CLAMP": [0], "ATTNPOOL_EMBED_FWD": [2], "ATTNPOOL_EMBED_BWD": [1],
            "SAMPLE_ANCESTRAL": [6], "SAMPLE_DDIM": [5],
            "GN_FWD_FUSED": [4, 5], "GN_BWD_FUSED": [6], "GN_FWD_GRID": [4, 5], "GN_BWD_GRID": [6],
            "CUTOUTS_AUG_FWD": [2], "CUTOUTS_AUG_BWD": [2], "RELU_FWD": [1], "RELU_BWD": [2], "MAXPOOL2_FWD": [1], "MAXPOOL2_BWD": [2], "LPIPS_TAP": [3, 4], "FILL": [0], "CUTOUTS_RR_FWD": [2], "CUTOUTS_RR_BWD": [2]}


def cpu_twin(plan):
    twin = copy.copy(plan)
    twin.handle = None
    twin.arena = plan.arena.cpu()
    return twin


def buf_view(arena, buf):
    return arena[buf.off:buf.off + buf.nbytes].view(_DT[buf.dt][1])


def compare_ops(plan, ranges, tol_h=4e-3, tol_f=2e-4, verbose=False):
    """Execute `ranges` (list of (mark_a, mark_b)) op by op.  Before each op the CPU twin arena is refreshed from the GPU
    arena, so every kernel is checked on identical inputs.  Returns (n_ops, failures)."""
    twin = cpu_twin(plan)
    it = Interp(twin)
    failures, n = [], 0
    for a, b in ranges:
        for k in range(plan.marks[a], plan.marks[b]):
            op = plan.ops[k]
            name = CODE[op.code]
            twin.arena.copy_(plan.arena)
            it.run(k, 1)
            plan.run(k, 1)
            th.cuda.synchronize()
            gpu = plan.arena.cpu()
            n += 1
            for slot in OUT_PTRS[name]:
                if slot >= len(op.p) or op.p[slot] is None:
                    continue
                buf = op.p[slot][0]
                ref = buf_view(twin.arena, buf).float()
                got = buf_view(gpu, buf).float()
                scale = float(ref.abs().max()) + 1e-12
                err = float((ref - got).abs().max()) / scale
                bad = not th.isfinite(got).all()
                tol = tol_h if buf.dt == "h" else tol_f
                if name.startswith("CUTOUTS_AUG"):
                    # nearest-neighbour sampling: a source coordinate within float round-off of .5 may pick the other pixel than
                    # torchvision's grid does (a handful of pixels per cutout) -- judged by the L2 error, not the worst element
                    err, tol = float((ref - got).norm() / (ref.norm() + 1e-20)), 1e-2
                if name in ("ATTN_FWD", "ATTN_BWD", "SPHERICAL", "GN_BWD_APPLY", "GN_BWD_STATS", "GN_BWD_FUSED", "GN_BWD_GRID", "LN_BWD", "CUTOUTS_BWD", "CUTOUTS_RR_BWD"):
                    tol = max(tol, 4e-3)
                if verbose or bad or err > tol:
                    rec = dict(op=k, code=name, tag=op.tag, slot=slot, buf=buf.name, err=err, ref_max=scale, got_max=float(got.abs().max()),
                               nonfinite=bad, i=list(op.i))
                    if bad or err > tol:
                        failures.append(rec)
                    if verbose:
                        print(rec)
    return n, failures
