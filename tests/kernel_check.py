"""Shared harness of the one-kernel-at-a-time tests (tests/test_gpu_kernels_fullshape.py, tests/test_gpu_unet_kernels.py): run a
stand-alone plan on the native kernels or through the test interpreter, and compare with a float64 reference element by element."""
import pytest
import torch as th

from tests.ensemble_oracle import EnsembleInterp  # the plan interpreter, with CUTOUTS_BWD flags 2 (accumulate)

U = 2.0 ** -24  # fp32 unit round-off
D64 = th.float64


def run(plan, device, inputs):
    """Finalize `plan` on `device`, write `inputs` ([(Buf, tensor)]) into its arena, execute every op -- the CUDA kernels on "cuda",
    the test interpreter on "cpu" -- and return a reader Buf -> CPU tensor."""
    plan.finalize(device)
    for b, t in inputs:
        v = plan.view(b)
        v.copy_(t.reshape(-1).to(v.dtype))
    if device == "cuda":
        plan.run()
        th.cuda.synchronize()
    else:
        EnsembleInterp(plan).run()
    return lambda b, shape=None: plan.view(b, shape).cpu().clone()


def cases(gpu, cpu):
    """pytest params: the production-size cases on the GPU, the reduced ones through the interpreter"""
    return ([pytest.param("cuda", c, marks=pytest.mark.gpu, id="gpu-" + k) for k, c in gpu.items()]
            + [pytest.param("cpu", c, id="cpu-" + k) for k, c in cpu.items()])


def ulp16(ref):
    """spacing of fp16 numbers at |ref| (2^-24 in the subnormal range)"""
    return th.exp2(th.floor(th.log2(ref.abs().clamp(min=2.0 ** -14))) - 10)


def check(what, got, ref, tol):
    got, ref = got.to(D64), ref.to(D64)
    if th.is_tensor(tol):
        tol = tol.to(got.device)
    ref = ref.to(got.device)
    err = (got - ref).abs()
    bad = ~(err <= tol)  # NaN fails too
    if bool(bad.any()):
        j = int(th.nonzero(bad.flatten())[0])
        tol_j = float(tol.flatten()[j]) if th.is_tensor(tol) and tol.numel() > 1 else float(tol)
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside tolerance; first at flat index {j}: "
                             f"got {float(got.flatten()[j])!r}, float64 {float(ref.flatten()[j])!r}, tol {tol_j!r}")


def check16(what, got, ref, floor):
    """fp16 output: one fp16 ulp of the float64 value plus `floor`"""
    check(what, got, ref, ulp16(ref) + floor)
