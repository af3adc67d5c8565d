// autograd.cu -- the UNet under torch.autograd: a PyTorch cond_fn's d loss / d model_out becomes the fp16 seed of the UNet input-gradient
// plan, and the plan's input gradient becomes d loss / d x (include/cgd_b200.h, CGD_OP_GRAD_SEED / GRAD_UNSCALE / PMV_BWD).
//
// The seed is scaled per image by the power of two of SEED_QUANT (guidance.cu): the largest |element| lands in (2048, 4096], so an
// arbitrary upstream gradient -- a user's loss may be 1e-6 or 1e6 -- neither underflows nor overflows the fp16 backward.
#include <stdint.h>

#include <algorithm>

#include "common.cuh"
#include "ops.cuh"
#include "pdl.cuh"

namespace cgd {

static inline bool aligned4(const void* p) { return ((uintptr_t)p & 3) == 0; }

// grid-stride elementwise kernels: at most 8 CTAs of 256 threads per SM
static inline int elem_blocks(int64_t items) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(items, 256), 132 * 8)); }

// the grid of the per-image kernels: (chunks, B), about 592 CTAs in all (4.5 waves of 132 SMs at 256 threads)
static inline int per_image_chunks(int64_t items, int64_t B) {
  return (int)std::min<int64_t>(ceil_div(items, 256 * 4), std::max<int64_t>(1, 592 / B));
}

// pass 1: dyn[b] = max |d_out[b]| as ordered int bits (non-negative floats order like ints).  fmaxf drops a NaN, an inf saturates to
// 3e38, an all-zero image leaves 0 (scale 1).  dyn[0..B) must be 0 on entry: GRAD_UNSCALE re-arms it.
__global__ void grad_seed_max_kernel(const float* __restrict__ d_out, float* __restrict__ dyn, int64_t HW) {
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.y;
  const int64_t per = 6 * HW;
  const float* src = d_out + (int64_t)b * per;
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < per; i += (int64_t)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(src[i]));
  m = fminf(warp_max(m), 3.0e38f);
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(reinterpret_cast<int*>(dyn) + b, __float_as_int(m));
}

// pass 2: seed[b, p, c] = fp16(clamp(d_out[b, c, p] * scale_b, +-60000)) for c < 6, dyn[B + b] = scale_b (SEED_QUANT's rule)
__global__ void grad_seed_quant_kernel(const float* __restrict__ d_out, float* __restrict__ dyn, __half* __restrict__ seed, int B, int64_t HW,
                                       int64_t ld) {
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.y;
  const float m = dyn[b];
  float scale = 1.f;
  if (m > 0.f) scale = exp2f(fminf(fmaxf(floorf(log2f(4096.f / m)), -60.f), 60.f));
  if (blockIdx.x == 0 && threadIdx.x == 0) dyn[B + b] = scale;
  const float* src = d_out + (int64_t)b * 6 * HW;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (int64_t)gridDim.x * blockDim.x) {
    float v[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) v[c] = fminf(fmaxf(src[c * HW + p] * scale, -60000.f), 60000.f);
    __half2* dst = reinterpret_cast<__half2*>(seed + ((int64_t)b * HW + p) * ld);
#pragma unroll
    for (int c = 0; c < 3; ++c) dst[c] = __halves2half2(__float2half_rn(v[2 * c]), __float2half_rn(v[2 * c + 1]));
  }
}

int launch_grad_seed(const CgdOp& op, cudaStream_t st) {
  const int64_t B = op.i[0], HW = op.i[1], ld = op.i[2];
  CGD_CHECK_ARG(B > 0 && B <= 65535 && HW > 0 && HW <= (int64_t(1) << 30), "grad_seed: B %lld / HW %lld out of range", (long long)B, (long long)HW);
  CGD_CHECK_ARG(ld >= 6 && ld <= 4096 && ld % 2 == 0, "grad_seed: seed row stride %lld must be even and in [6, 4096]", (long long)ld);
  CGD_CHECK_ARG(op.p[0] && op.p[1] && op.p[2] && aligned4(op.p[0]) && aligned4(op.p[1]) && aligned4(op.p[2]), "grad_seed: null or misaligned pointer");
  CGD_CUDA(launch_pdl(grad_seed_max_kernel, dim3(per_image_chunks(6 * HW, B), (unsigned)B), dim3(256), 0, st, (const float*)op.p[0], (float*)op.p[1], HW));
  CGD_LAUNCH_CHECK();
  CGD_CUDA(launch_pdl(grad_seed_quant_kernel, dim3(per_image_chunks(HW, B), (unsigned)B), dim3(256), 0, st, (const float*)op.p[0], (float*)op.p[1],
                      (__half*)op.p[2], (int)B, HW, ld));
  CGD_LAUNCH_CHECK();
  return 0;
}

// dx = dx_unet * (1 / scale_b) (+ dx_direct): the scale is a power of two, the reciprocal and the product are exact.  Then re-arms the
// maxima and zeroes seed channels 0..5: the fused step's GUIDE_GRAD / SEED_QUANT write channels 0..2 only and rely on 3..5 being zero.
__global__ void grad_unscale_kernel(const float* __restrict__ dxu, const float* __restrict__ dxd, float* __restrict__ dyn, __half* __restrict__ seed,
                                    float* __restrict__ dx, int B, int64_t HW, int64_t ld) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t n = (int64_t)B * 3 * HW, npix = (int64_t)B * HW, stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (int64_t i = t0; i < n; i += stride) {
    float v = dxu[i] * (1.f / dyn[B + i / (3 * HW)]);
    if (dxd) v += dxd[i];
    dx[i] = v;
  }
  const __half2 z = __floats2half2_rn(0.f, 0.f);
  for (int64_t p = t0; p < npix; p += stride) {
    __half2* s = reinterpret_cast<__half2*>(seed + p * ld);
    s[0] = z;
    s[1] = z;
    s[2] = z;
  }
  if (blockIdx.x == 0)
    for (int b = threadIdx.x; b < B; b += blockDim.x) dyn[b] = 0.f;
}

int launch_grad_unscale(const CgdOp& op, cudaStream_t st) {
  const int64_t B = op.i[0], HW = op.i[1], ld = op.i[2];
  CGD_CHECK_ARG(B > 0 && B <= 65535 && HW > 0 && HW <= (int64_t(1) << 30), "grad_unscale: B %lld / HW %lld out of range", (long long)B, (long long)HW);
  CGD_CHECK_ARG(ld >= 6 && ld <= 4096 && ld % 2 == 0, "grad_unscale: seed row stride %lld must be even and in [6, 4096]", (long long)ld);
  CGD_CHECK_ARG(op.p[0] && op.p[2] && op.p[3] && op.p[4], "grad_unscale: null pointer (only p1 dx_direct may be null)");
  CGD_CHECK_ARG(aligned4(op.p[0]) && aligned4(op.p[1]) && aligned4(op.p[2]) && aligned4(op.p[3]) && aligned4(op.p[4]), "grad_unscale: misaligned pointer");
  CGD_CUDA(launch_pdl(grad_unscale_kernel, dim3(elem_blocks(B * 3 * HW)), dim3(256), 0, st, (const float*)op.p[0], (const float*)op.p[1], (float*)op.p[2],
                      (__half*)op.p[3], (float*)op.p[4], (int)B, HW, ld));
  CGD_LAUNCH_CHECK();
  return 0;
}

// transpose of pmv_blend_kernel (guidance.cu).  Forward: x0 = a x - bb eps, mean = c1 x0 + c2 x, lv = (v + 1) / 2 * maxl + (1 - (v + 1) / 2) * minl,
// var = exp(lv).  Backward, G = g_x0 + c1 g_mean: d eps = -bb G, d v = (maxl - minl) / 2 * (g_lv + var g_var), direct dx = a G + c2 g_mean.
__global__ void pmv_bwd_kernel(const float* __restrict__ sc, const float* __restrict__ var, const float* __restrict__ gx0, const float* __restrict__ gmean,
                               const float* __restrict__ gvar, const float* __restrict__ glv, float* __restrict__ d_out, float* __restrict__ dxd, int B,
                               int64_t HW) {
  pdl_wait();
  pdl_launch_dependents();
  const float a = sc[CGD_SC_SQRT_RECIP_AC], bb = sc[CGD_SC_SQRT_RECIPM1_AC], c1 = sc[CGD_SC_POST_COEF1], c2 = sc[CGD_SC_POST_COEF2];
  const float hr = (sc[CGD_SC_MAX_LOG] - sc[CGD_SC_MIN_LOG]) * 0.5f;
  const int64_t total = (int64_t)B * 3 * HW;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = idx % HW, bc = idx / HW;
    const int64_t b = bc / 3, c = bc % 3;
    const float gm = gmean ? gmean[idx] : 0.f;
    const float G = (gx0 ? gx0[idx] : 0.f) + c1 * gm;
    float gl = glv ? glv[idx] : 0.f;
    if (gvar) gl += var[idx] * gvar[idx];
    d_out[(b * 6 + c) * HW + p] = -bb * G;
    d_out[(b * 6 + 3 + c) * HW + p] = hr * gl;
    dxd[idx] = a * G + c2 * gm;
  }
}

int launch_pmv_bwd(const CgdOp& op, cudaStream_t st) {
  const int64_t B = op.i[0], HW = op.i[1];
  CGD_CHECK_ARG(B > 0 && B <= 65535 && HW > 0 && HW <= (int64_t(1) << 30), "pmv_bwd: B %lld / HW %lld out of range", (long long)B, (long long)HW);
  CGD_CHECK_ARG(op.p[0] && op.p[6] && op.p[7] && (!op.p[4] || op.p[1]), "pmv_bwd: null pointer (p1 variance is needed with p4 g_variance)");
  for (int k = 0; k < 8; ++k) CGD_CHECK_ARG(aligned4(op.p[k]), "pmv_bwd: misaligned pointer p%d", k);
  CGD_CUDA(launch_pdl(pmv_bwd_kernel, dim3(elem_blocks(B * 3 * HW)), dim3(256), 0, st, (const float*)op.p[0], (const float*)op.p[1], (const float*)op.p[2],
                      (const float*)op.p[3], (const float*)op.p[4], (const float*)op.p[5], (float*)op.p[6], (float*)op.p[7], (int)B, HW));
  CGD_LAUNCH_CHECK();
  return 0;
}

}  // namespace cgd
