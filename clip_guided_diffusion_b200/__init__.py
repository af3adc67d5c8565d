"""clip_guided_diffusion_b200 -- H100 (sm_90a) implementation of the CLIP-guided diffusion sampling step.

Host side is Python (PyTorch tensors for device memory, streams and torch.distributed); every per-timestep kernel
lives in libcgd_b200.so (include/cgd_b200.h) and is loaded with ctypes.  No CPU / PyTorch fallback exists for the
step: without the built library the product raises.
"""
from ._lib import CgdError, LIB_PATH, load  # noqa: F401

__all__ = ["CgdError", "LIB_PATH", "load"]
