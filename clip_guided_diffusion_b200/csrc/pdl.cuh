// pdl.cuh -- programmatic dependent launch (griddepcontrol) helpers.
//
// A guided step is ~900 back-to-back kernels on one stream; most of them are short, so the drain -> launch ->
// prologue bubble between two kernels is a first-order cost.  Kernels that use these helpers are launched with
// cudaLaunchAttributeProgrammaticStreamSerialization: the next kernel's CTAs become resident as soon as every CTA of the
// current one has executed `pdl_launch_dependents()` (or exited), run their prologue (barrier init, descriptor
// prefetch, loads of step-invariant parameters) and block in `pdl_wait()` until the previous grid has completed and its
// writes are visible.  Rules followed by every kernel in this library:
//   * nothing that another kernel of the step writes is read, and no global memory is written, before pdl_wait();
//   * pdl_wait() is executed by every thread that touches global memory afterwards (it is a no-op when the kernel was
//     launched without the attribute);
//   * launches carry the attribute only for kernels that contain pdl_wait().
#pragma once
#include <cuda_runtime.h>

namespace cgd {

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

bool pdl_enabled();  // api.cu: CGD_PDL environment switch (default on)

// <<<grid, block, smem, stream>>> with the programmatic-serialization attribute (when enabled)
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace cgd
