"""ctypes binding of libcgd_b200.so (include/cgd_b200.h).  There is no fallback: if the library is missing or
fails to load, every product entry point raises."""
from __future__ import annotations

import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libcgd_b200.so")

CGD_OP_NI, CGD_OP_NF, CGD_OP_NP = 24, 8, 12


class CgdOp(ctypes.Structure):
    _fields_ = [("code", ctypes.c_int32), ("flags", ctypes.c_int32), ("i", ctypes.c_int64 * CGD_OP_NI),
                ("f", ctypes.c_float * CGD_OP_NF), ("p", ctypes.c_void_p * CGD_OP_NP)]


# op codes / scalar slots -- keep in sync with include/cgd_b200.h (checked by tests/test_abi.py)
OP = dict(CONV=1, GN_STATS=2, GN_APPLY=3, GN_BWD_STATS=4, GN_BWD_APPLY=5, POOL2=6, UP2=7, ADD=8, ATTN_FWD=9, ATTN_BWD=10,
          LINEAR_SMALL=11, TIMESTEP_EMB=12, LABEL_ADD=13, NCHW_TO_PM=14, PM_TO_NCHW=15, LN_FWD=16, LN_BWD=17, QGELU_FWD=18,
          QGELU_BWD=19, VIT_EMBED=20, CUTOUTS_FWD=21, CUTOUTS_BWD=22, SPHERICAL=23, PMV_BLEND=24, GUIDE_GRAD=25,
          FINAL_GRAD=26, SAMPLE_ANCESTRAL=27, SAMPLE_DDIM=28, COPY=29, TRANSPOSE=30, SOFTMAX_FWD=31, SOFTMAX_BWD=32,
          GN_FWD_FUSED=33, GN_BWD_FUSED=34, GN_FWD_GRID=35, GN_BWD_GRID=36,
          RELU_FWD=37, RELU_BWD=38, MAXPOOL2_FWD=39, MAXPOOL2_BWD=40, LPIPS_TAP=41, FILL=42, CUTOUTS_RR_FWD=43, CUTOUTS_RR_BWD=44, SEED_QUANT=45, MAG_CLAMP=46, ATTNPOOL_EMBED_FWD=47, ATTNPOOL_EMBED_BWD=48, GN_APPLY_EPI=49, CUTOUTS_AUG_FWD=50, CUTOUTS_AUG_BWD=51)
SC = dict(SQRT_RECIP_AC=0, SQRT_RECIPM1_AC=1, POST_COEF1=2, POST_COEF2=3, MIN_LOG=4, MAX_LOG=5, FAC=6, NONZERO=7,
          SQRT_1M_AC=8, AC_PREV=9, AC=10, ETA=11, ONE_MINUS_FAC=12, COUNT=16)

EXPORTS = ["cgd_abi_version", "cgd_last_error", "cgd_conv_cluster_capacity", "cgd_plan_create", "cgd_plan_run", "cgd_plan_num_launches",
           "cgd_plan_destroy", "cgd_run_op", "cgd_unet_create", "cgd_unet_fwd", "cgd_unet_bwd_input", "cgd_unet_destroy",
           "cgd_vit_create", "cgd_vit_fwd", "cgd_vit_bwd_input", "cgd_vit_destroy", "cgd_step_create", "cgd_step",
           "cgd_step_destroy", "cgd_cutouts_fwd", "cgd_cutouts_bwd", "cgd_spherical_fwd_bwd",
           "cgd_guidance_losses_fwd_bwd", "cgd_sample_update_ancestral", "cgd_sample_update_ddim"]

_lib = None


class CgdError(RuntimeError):
    pass


def load():
    """Load (once) and return the ctypes handle.  Raises if the CUDA library has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise CgdError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(nvcc, sm_90a).  There is no CPU / PyTorch fallback for the sampling step.")
    lib = ctypes.CDLL(LIB_PATH)
    lib.cgd_last_error.restype = ctypes.c_char_p
    lib.cgd_abi_version.restype = ctypes.c_int
    lib.cgd_conv_cluster_capacity.argtypes = [ctypes.c_int32, ctypes.c_int32]
    vp, i32 = ctypes.c_void_p, ctypes.c_int32
    lib.cgd_plan_create.argtypes = [ctypes.POINTER(CgdOp), i32, ctypes.POINTER(vp)]
    lib.cgd_plan_run.argtypes = [vp, i32, i32, vp]
    lib.cgd_plan_num_launches.argtypes = [vp, i32, i32]
    lib.cgd_plan_destroy.argtypes = [vp]
    lib.cgd_run_op.argtypes = [ctypes.POINTER(CgdOp), vp]
    for name in ("cgd_unet_create", "cgd_vit_create"):
        getattr(lib, name).argtypes = [ctypes.POINTER(CgdOp), i32, i32, ctypes.POINTER(vp)]
    lib.cgd_step_create.argtypes = [ctypes.POINTER(CgdOp), i32, ctypes.POINTER(vp)]
    for name in ("cgd_unet_fwd", "cgd_unet_bwd_input", "cgd_vit_fwd", "cgd_vit_bwd_input", "cgd_step"):
        getattr(lib, name).argtypes = [vp, vp]
    for name in ("cgd_unet_destroy", "cgd_vit_destroy", "cgd_step_destroy"):
        getattr(lib, name).argtypes = [vp]
    if lib.cgd_abi_version() != 2:
        raise CgdError("libcgd_b200.so ABI version mismatch")
    _lib = lib
    return lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().cgd_last_error().decode("utf-8", "replace")
        raise CgdError(f"{what + ': ' if what else ''}libcgd_b200 error {rc}: {msg}")
