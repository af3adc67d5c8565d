"""CPU: every op a plan emits passes the C side's ARGUMENT validation (the launch_* / conv_tc_prepare checks of csrc/) -- without a GPU.
Each op is lowered to the C struct with fake, aligned, non-null pointers and handed to `cgd_run_op`: with no device the call must fail
with a CUDA error (rc > 0: the launch itself), never with rc = -1 (an argument rejected).  Convs stop at the tensor-map encoder
("cuTensorMapEncodeTiled unavailable") after their dimension / alignment / stride checks.  This is how op layouts that have not run on
a device yet (ModifiedResNet tower) are checked against the kernels' contracts."""
import ctypes

import pytest
import torch as th

from clip_guided_diffusion_b200 import _lib
from clip_guided_diffusion_b200 import plan as P
from tests.plan_interp import CODE

pytestmark = pytest.mark.skipif(th.cuda.is_available(), reason="needs a box WITHOUT a GPU: launches must fail, only the checks run")


def _check_plan(plan, what):
    lib = _lib.load()
    base = 1 << 40  # fake device address, 256-byte aligned; nothing is dereferenced: no kernel can launch here
    arr = plan.lower(base)
    bad = []
    for k, op in enumerate(plan.ops):
        rc = lib.cgd_run_op(ctypes.byref(arr[k]), None)
        msg = lib.cgd_last_error().decode("utf-8", "replace")
        if rc > 0 or (rc == -1 and CODE[op.code] == "CONV" and "cuTensorMapEncodeTiled unavailable" in msg):
            continue
        bad.append((k, CODE[op.code], op.tag, rc, msg))
    assert not bad, f"{what}: {len(bad)} op(s) rejected by the C-side argument checks, first: {bad[:3]}"
    return len(plan.ops)


def test_guided_step_ops_pass_c_side_checks():
    from tests.step_parity import build_tiny
    for kw in (dict(B=2, cutn=3, image=32), dict(B=1, cutn=4, image=32, use_magnitude=True, sat_scale=30.0, cutn_variants=(2, 4)),
               dict(B=2, cutn=2, image=32, init_scale=1000.0), dict(B=1, cutn=3, image=64, cutout_resize="lanczos3"),
               dict(B=2, cutn=3, image=32, tower="rn"), dict(B=1, cutn=2, image=32, hw=(32, 64))):
        ctx = build_tiny("cpu", **kw)
        assert _check_plan(ctx["eng"].plan, str(kw)) > 100


def test_resnet_tower_ops_pass_c_side_checks():
    from clip_guided_diffusion_b200 import rn as prn
    from clip_guided_diffusion_b200 import weights as pw
    cfg = prn.RNConfig(layers=(1, 2, 1, 1), output_dim=128, input_resolution=224, width=64)  # real spatial sizes: 112 .. 7, 50 tokens
    sd = {k: th.zeros(v) for k, v in pw.rn_param_shapes(cfg).items()}
    for k in sd:
        if k.endswith("running_var"):
            sd[k] += 1
    tower = prn.RNB200(cfg, sd, n_images=4, device="cpu")
    assert _check_plan(tower.plan, "RN tower") > 60


FULL_SIZE = {  # every configuration that runs on the device at full size (tests/test_gpu_baseline_configs.py, test_gpu_fullsize.py, test_gpu_rn.py)
    "cfg1": dict(size=64, cutn=4, clip="ViT-B/32", mag=True),
    "cfg2": dict(size=256, cutn=16, clip="ViT-B/32"),
    "cfg3": dict(size=256, cutn=32, clip="ViT-B/32"),
    "cfg4": dict(size=512, cutn=16, clip="ViT-B/16"),
    "cfg5": dict(size=512, cutn=64, clip="ViT-L/14", lpips=True),
    "default128": dict(size=128, cutn=16, clip="ViT-B/32"),
    "vit_l14_336": dict(size=256, cutn=4, clip="ViT-L/14@336px"),
    "rn50x16": dict(size=256, cutn=4, clip="RN50x16"),
    "rn101": dict(size=256, cutn=8, clip="RN101"),
}


@pytest.mark.parametrize("name", list(FULL_SIZE))
def test_full_size_step_plans_pass_c_side_checks(name, monkeypatch):
    """the op lists of the published architectures, built shapes-only (no weight data is packed: `Plan.const` only reserves the bytes),
    against the library's argument checks -- a check tightened in csrc/ must not reject a layer of a real checkpoint"""
    from clip_guided_diffusion_b200 import guidance as pg
    from clip_guided_diffusion_b200 import rn as prn
    from clip_guided_diffusion_b200 import unet as pu
    from clip_guided_diffusion_b200 import vit as pv
    from clip_guided_diffusion_b200 import weights as pw
    monkeypatch.setattr(P.Plan, "const", lambda self, t, dt, name="": self.new(t.numel(), dt, name))
    monkeypatch.setattr(P.Plan, "finalize", lambda self, device: self)
    c = FULL_SIZE[name]
    empty = lambda shapes: {k: th.empty(v) for k, v in shapes.items()}  # noqa: E731
    ucfg = pu.config_for(c["size"], True)
    if c["clip"].startswith("RN"):
        vcfg = prn.RN_CONFIGS[c["clip"]]
        vsd = {k: (th.ones(v) if k.endswith("running_var") else th.zeros(v)) for k, v in pw.rn_param_shapes(vcfg).items()}  # BatchNorm is folded on the host
    else:
        vcfg = pv.VIT_CONFIGS[c["clip"]]
        vsd = empty(pw.vit_param_shapes(vcfg))
    extra = dict(lpips_sd=empty(pw.lpips_param_shapes()), init_scale=1000.0) if c.get("lpips") else {}
    eng = pg.GuidedStepB200(ucfg, empty(pw.unet_param_shapes(ucfg)), vcfg, vsd, batch=1, num_cutouts=c["cutn"], device="cpu",
                            use_magnitude=c.get("mag", False), **extra)
    assert _check_plan(eng.plan, name) > 600
