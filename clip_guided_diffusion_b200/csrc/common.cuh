// common.cuh -- shared device helpers for libcgd_b200 (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/cgd_b200.h"

#ifndef __CUDA_ARCH_FEAT_SM90_ALL
#if defined(__CUDA_ARCH__)
#error "libcgd_b200 must be compiled for sm_90a (-gencode arch=compute_90a,code=sm_90a)"
#endif
#endif

namespace cgd {

typedef __half act_t;  // activation / weight storage type of the networks (wgmma fp16 operands, fp32 accumulate)

// ---------------------------------------------------------------- error plumbing (host)
void set_error(const char* fmt, ...);
#define CGD_CHECK_ARG(cond, ...)        \
  do {                                  \
    if (!(cond)) {                      \
      cgd::set_error(__VA_ARGS__);      \
      return -1;                        \
    }                                   \
  } while (0)
#define CGD_CUDA(expr)                                                                   \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      cgd::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return (int)_e;                                                                    \
    }                                                                                    \
  } while (0)
#define CGD_LAUNCH_CHECK()                                                               \
  do {                                                                                   \
    cudaError_t _e = cudaGetLastError();                                                 \
    if (_e != cudaSuccess) {                                                             \
      cgd::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
      return (int)_e;                                                                    \
    }                                                                                    \
  } while (0)

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// "done once per device": function attributes (opt-in dynamic shared memory), occupancy checks and the SM count belong to the
// CURRENT device, and one process may drive several GPUs (one engine per device).  Not a lock: a race sets an attribute twice.
struct DeviceOnce {
  bool done[64] = {};
  int value[64] = {};
  static int cur() {
    int d = 0;
    return (cudaGetDevice(&d) == cudaSuccess && d >= 0 && d < 64) ? d : 0;
  }
  bool needed() const { return !done[cur()]; }
  void mark(int v = 0) {
    const int d = cur();
    value[d] = v;
    done[d] = true;
  }
  int get() const { return value[cur()]; }
};
// SM count of the current device (132 on an H100 SXM; grids of the persistent kernels are sized from it, not from the constant)
static inline int device_sm_count() {
  static DeviceOnce once;
  if (once.needed()) {
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
    once.mark(sms);
  }
  return once.get();
}

// ---------------------------------------------------------------- small device helpers
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// block-wide sum, result broadcast to all threads; `red` = >= 32 floats of shared memory
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  float r = (threadIdx.x < nw) ? red[threadIdx.x] : 0.f;
  if (wid == 0) {
    r = warp_sum(r);
    if (lane == 0) red[0] = r;
  }
  __syncthreads();
  return red[0];
}

// sigmoid on the SFU: ex2.approx.ftz + rcp.approx.ftz (2 MUFU + 2 FP32 ops, ~2 ulp).  These run per element in the
// HBM-bound normalisation kernels: the libdevice forms (__expf, __fdividef) carry denormal-range guards (FSETP + 2 FMUL per
// call in SASS) that made GroupNorm-apply issue-bound; with flush-to-zero the limits are exact: v -> -inf gives
// ex2 = +inf, rcp = 0; v -> +inf gives ex2 = 0, rcp(1) = 1.
__device__ __forceinline__ float ex2_ftz(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_ftz(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// sigmoid(v) = 1/2 + 1/2 tanh(v / 2): ONE MUFU op (tanh.approx.f32, relative error 2^-11) instead of two (ex2 + rcp).  Why it matters:
// the SFU issues 16 lanes / clk / SM, so two MUFU ops per element can put a floor under a streaming GroupNorm-apply kernel that is
// higher than its memory traffic; every SiLU / SiLU' in the GroupNorm kernels has the same per-element cost.  Accuracy: |sigmoid error| <= 2.5e-4 absolute, i.e. |silu error| <= 2.5e-4 |v| -- the
// size of the fp16 rounding of the output itself; the full-size parity tests (tests/test_gpu_baseline_configs.py) bound the effect.
// -DCGD_SIGMOID_EX2RCP restores the two-MUFU form (A/B builds).
__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
#ifdef CGD_SIGMOID_EX2RCP
__device__ __forceinline__ float sigmoid_fast(float v) { return rcp_ftz(1.f + ex2_ftz(-1.4426950408889634f * v)); }
#else
__device__ __forceinline__ float sigmoid_fast(float v) { return fmaf(0.5f, tanh_approx(0.5f * v), 0.5f); }
#endif
__device__ __forceinline__ float silu_f(float v) { return v * sigmoid_fast(v); }
// d silu(v)/dv
__device__ __forceinline__ float silu_grad_f(float v) {
  const float s = sigmoid_fast(v);
  return s * (1.f + v * (1.f - s));
}

// fp32 pairs, one rounding per lane
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
#ifdef CGD_SIGMOID_EX2RCP
// d silu / dt on a pair: s * (1 + t * (1 - s))
__device__ __forceinline__ float2 silu_grad2(float2 t) {
  const float2 u = mul2(t, make_float2(-1.4426950408889634f, -1.4426950408889634f));
  const float2 d = add2(make_float2(ex2_ftz(u.x), ex2_ftz(u.y)), make_float2(1.f, 1.f));
  const float2 s = make_float2(rcp_ftz(d.x), rcp_ftz(d.y));
  const float2 one = make_float2(1.f, 1.f);
  const float2 w = fma2(t, fma2(s, make_float2(-1.f, -1.f), one), one);  // 1 + t * (1 - s)
  return mul2(s, w);
}
#else
// d silu / dt on a pair: s * (1 + t * (1 - s)), s = 1/2 + 1/2 tanh(t / 2)
__device__ __forceinline__ float2 silu_grad2(float2 t) {
  const float2 half2v = make_float2(0.5f, 0.5f), one = make_float2(1.f, 1.f);
  const float2 h = mul2(t, half2v);
  const float2 s = fma2(make_float2(tanh_approx(h.x), tanh_approx(h.y)), half2v, half2v);
  const float2 w = fma2(t, fma2(s, make_float2(-1.f, -1.f), one), one);  // 1 + t * (1 - s)
  return mul2(s, w);
}
#endif

// ---------------------------------------------------------------- global-memory barrier among co-resident CTAs
// bar[0] = arrival count (returns to 0), bar[1] = generation (only ever incremented): reusable across launches / graph replays
// without a reset.  Called by ONE thread per CTA after a block-level barrier; acquire / release atomics instead of
// __threadfence(): each MEMBAR.SC.GPU of a fence-based version invalidates the L1, which makes a barrier over every SM of the
// device cost several microseconds.
__device__ __forceinline__ void global_barrier_arrive_wait(unsigned int* bar, unsigned int n) {
  unsigned int gen, old, cur;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(gen) : "l"(bar + 1) : "memory");  // before arriving: cannot advance yet
  asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], 1;" : "=r"(old) : "l"(bar) : "memory");
  if (old == n - 1u) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(bar), "r"(0u) : "memory");
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar + 1) : "memory");
  } else {
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(cur) : "l"(bar + 1) : "memory");
    } while (cur == gen);
  }
}

struct __align__(16) half8 {
  __half2 a, b, c, d;
};
__device__ __forceinline__ void unpack8(const half8& h, float* f) {
  float2 t;
  t = __half22float2(h.a); f[0] = t.x; f[1] = t.y;
  t = __half22float2(h.b); f[2] = t.x; f[3] = t.y;
  t = __half22float2(h.c); f[4] = t.x; f[5] = t.y;
  t = __half22float2(h.d); f[6] = t.x; f[7] = t.y;
}
__device__ __forceinline__ half8 pack8(const float* f) {
  half8 h;
  h.a = __floats2half2_rn(f[0], f[1]);
  h.b = __floats2half2_rn(f[2], f[3]);
  h.c = __floats2half2_rn(f[4], f[5]);
  h.d = __floats2half2_rn(f[6], f[7]);
  return h;
}
// 128-bit accesses go through the built-in uint4: a struct of four __half2 is scalarised by nvcc into four 32-bit LDG / STG
// (seen in SASS: not one 128-bit access in norm.cu / elementwise.cu), which quarters the bytes per memory instruction
union Half8Bits {
  uint4 u;
  half8 h;
  __device__ Half8Bits() {}
};
__device__ __forceinline__ half8 ld8(const __half* p) {
  Half8Bits b;
  b.u = *reinterpret_cast<const uint4*>(p);
  return b.h;
}
__device__ __forceinline__ void st8(__half* p, const half8& v) {
  Half8Bits b;
  b.h = v;
  *reinterpret_cast<uint4*>(p) = b.u;
}

}  // namespace cgd
