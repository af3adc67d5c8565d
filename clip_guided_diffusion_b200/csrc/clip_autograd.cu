// clip_autograd.cu -- a CLIP visual tower under torch.autograd: a user's NCHW image batch becomes the tower's fp16 patch rows, a user's
// d loss / d embeds becomes the scaled seed of the tower backward, and the tower's d_patches become d loss / d image
// (include/cgd_b200.h, CGD_OP_CLIP_PATCHIFY / CLIP_SEED / CLIP_UNPATCHIFY).
//
// The seed is scaled per image by a power of two that puts its largest |element| near BAND (op f0): a user's loss may put 1e-8 or 1e8
// into d_embeds, and the tower's first fp16 store (LINEAR_SMALL flags 8 -> d_cls / d_query_row) would flush or overflow either.
#include <stdint.h>

#include <algorithm>

#include "common.cuh"
#include "ops.cuh"
#include "pdl.cuh"

namespace cgd {

static inline bool aligned(const void* p, uintptr_t a) { return ((uintptr_t)p & (a - 1)) == 0; }

// grid-stride elementwise kernels: at most 8 CTAs of 256 threads per SM
static inline int elem_blocks(int64_t items) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(items, 256), 132 * 8)); }

// the patch geometry shared by both directions: 0, or -1 with the error set when a dimension is out of range
static int check_patch_dims(const CgdOp& op, const char* what) {
  const int64_t n = op.i[0], nb = op.i[1], R = op.i[2], P = op.i[3], kpad = op.i[4];
  CGD_CHECK_ARG(op.flags == 0, "%s: flags must be 0", what);
  CGD_CHECK_ARG(n > 0 && nb >= n && nb <= 65535, "%s: n %lld / n_built %lld out of range", what, (long long)n, (long long)nb);
  CGD_CHECK_ARG(P >= 1 && P <= 64 && R >= P && R <= 4096 && R % P == 0, "%s: image side %lld / patch %lld invalid", what, (long long)R,
                (long long)P);
  CGD_CHECK_ARG(kpad >= 3 * P * P && kpad <= 16384 && kpad % 8 == 0, "%s: kpad %lld must be a multiple of 8 and >= 3 * P * P", what,
                (long long)kpad);
  return 0;
}

// one thread = 8 consecutive columns of one patch row (one 128-bit store)
__global__ void clip_patchify_kernel(const float* __restrict__ x, __half* __restrict__ patches, int n, int64_t rows, int R, int P, int kpad) {
  pdl_wait();
  pdl_launch_dependents();
  const int G = R / P, PP = P * P, chunks = kpad / 8;
  const int64_t G2 = (int64_t)G * G, items = rows * chunks;
  for (int64_t it = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; it < items; it += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = it / chunks;
    const int k0 = (int)(it % chunks) * 8;
    const int64_t b = r / G2;
    const int g = (int)(r % G2), gy = g / G, gx = g % G;
    __align__(16) __half h[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = k0 + j;
      float v = 0.f;
      if (b < n && k < 3 * PP) {
        const int c = k / PP, rem = k % PP;
        v = x[((b * 3 + c) * R + gy * P + rem / P) * (int64_t)R + gx * P + rem % P];
      }
      h[j] = __float2half_rn(v);
    }
    reinterpret_cast<uint4*>(patches)[it] = *reinterpret_cast<const uint4*>(h);
  }
}

int launch_clip_patchify(const CgdOp& op, cudaStream_t st) {
  if (check_patch_dims(op, "clip_patchify")) return -1;
  CGD_CHECK_ARG(op.p[0] && op.p[1] && aligned(op.p[0], 4) && aligned(op.p[1], 16), "clip_patchify: null or misaligned pointer");
  const int64_t nb = op.i[1], R = op.i[2], P = op.i[3], kpad = op.i[4];
  const int64_t rows = nb * (R / P) * (R / P);
  CGD_CUDA(launch_pdl(clip_patchify_kernel, dim3(elem_blocks(rows * (kpad / 8))), dim3(256), 0, st, (const float*)op.p[0], (__half*)op.p[1],
                      (int)op.i[0], rows, (int)R, (int)P, (int)kpad));
  CGD_LAUNCH_CHECK();
  return 0;
}

// one CTA of 256 threads per image row: D <= 1024 floats, four per thread kept in registers between the maximum and the store
__global__ void __launch_bounds__(256) clip_seed_kernel(const float* __restrict__ d, float* __restrict__ d_emb, float* __restrict__ dyn, int n,
                                                        int D, float band) {
  __shared__ float red[32];
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.x;
  const float* src = d + (int64_t)b * D;
  float v[4], m = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int k = threadIdx.x + j * 256;
    v[j] = (b < n && k < D) ? src[k] : 0.f;
    m = fmaxf(m, fabsf(v[j]));  // fmaxf drops a NaN
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = warp_max(threadIdx.x < 8 ? red[threadIdx.x] : 0.f);
    if (threadIdx.x == 0) red[0] = fminf(m, 3.0e38f);
  }
  __syncthreads();
  m = red[0];
  const float scale = m > 0.f ? exp2f(fminf(fmaxf(floorf(log2f(band / m)), -60.f), 60.f)) : 1.f;
  if (threadIdx.x == 0) dyn[b] = scale;
  float* dst = d_emb + (int64_t)b * D;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int k = threadIdx.x + j * 256;
    if (k < D) dst[k] = v[j] * scale;
  }
}

int launch_clip_seed(const CgdOp& op, cudaStream_t st) {
  const int64_t n = op.i[0], nb = op.i[1], D = op.i[2];
  const float band = op.f[0];
  CGD_CHECK_ARG(op.flags == 0, "clip_seed: flags must be 0");
  CGD_CHECK_ARG(n > 0 && nb >= n && nb <= 65535 && D > 0 && D <= 1024, "clip_seed: n %lld / n_built %lld / D %lld out of range", (long long)n,
                (long long)nb, (long long)D);
  int e = 0;
  CGD_CHECK_ARG(band >= 1.f && band <= 32768.f && frexpf(band, &e) == 0.5f, "clip_seed: BAND %g must be a power of two in [1, 2^15]", band);
  CGD_CHECK_ARG(op.p[0] && op.p[1] && op.p[2] && aligned(op.p[0], 4) && aligned(op.p[1], 4) && aligned(op.p[2], 4),
                "clip_seed: null or misaligned pointer");
  CGD_CUDA(launch_pdl(clip_seed_kernel, dim3((unsigned)nb), dim3(256), 0, st, (const float*)op.p[0], (float*)op.p[1], (float*)op.p[2], (int)n,
                      (int)D, band));
  CGD_LAUNCH_CHECK();
  return 0;
}

// one thread = one output pixel of the NCHW gradient (coalesced stores; the reads walk kx within a patch row)
__global__ void clip_unpatchify_kernel(const __half* __restrict__ dp, const float* __restrict__ dyn, float* __restrict__ dx, int64_t total, int R,
                                       int P, int kpad) {
  pdl_wait();
  pdl_launch_dependents();
  const int G = R / P, PP = P * P;
  const int64_t plane = (int64_t)R * R, G2 = (int64_t)G * G;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t bc = idx / plane;
    const int64_t b = bc / 3;
    const int c = (int)(bc % 3), yx = (int)(idx % plane), y = yx / R, xx = yx % R;
    const int64_t row = b * G2 + (int64_t)(y / P) * G + xx / P;
    const int k = c * PP + (y % P) * P + xx % P;
    dx[idx] = __half2float(dp[row * kpad + k]) * (1.f / dyn[b]);
  }
}

int launch_clip_unpatchify(const CgdOp& op, cudaStream_t st) {
  if (check_patch_dims(op, "clip_unpatchify")) return -1;
  CGD_CHECK_ARG(op.p[0] && op.p[1] && op.p[2] && aligned(op.p[0], 2) && aligned(op.p[1], 4) && aligned(op.p[2], 4),
                "clip_unpatchify: null or misaligned pointer");
  const int64_t total = op.i[0] * 3 * op.i[2] * op.i[2];
  CGD_CUDA(launch_pdl(clip_unpatchify_kernel, dim3(elem_blocks(total)), dim3(256), 0, st, (const __half*)op.p[0], (const float*)op.p[1],
                      (float*)op.p[2], total, (int)op.i[2], (int)op.i[3], (int)op.i[4]));
  CGD_LAUNCH_CHECK();
  return 0;
}

}  // namespace cgd
