// lpips.cu -- the non-conv pieces of the LPIPS-VGG16 perceptual loss and its input gradient ([3P] lpips.LPIPS(net='vgg'), used by
// the reference when an init image is given: cgd/cgd.py:147-148, 220-224; SURVEY.md A.4, K21).  The 13 conv3x3 layers run on the
// wgmma conv kernel (conv_tc.cu); here: ReLU, 2x2 max-pool, and the per-tap "unit-normalise over channels, squared difference
// to the (precomputed, normalised) init-image features, 1x1 lin, spatial mean" with its analytic gradient.  All HBM-bound
// elementwise / per-pixel kernels on pixel-major fp16 activations, 128-bit accesses.
#include "common.cuh"
#include "ops.cuh"
#include "pdl.cuh"

namespace cgd {

static inline int lp_blocks(int64_t n, int per_block = 256) {
  int64_t b = (n + per_block - 1) / per_block;
  if (b > 132 * 8) b = 132 * 8;
  return (int)(b < 1 ? 1 : b);
}

// y = max(x, 0) over n8 vectors of 8 halfs (in place allowed)
__global__ void relu_fwd_kernel(const __half* __restrict__ x, __half* __restrict__ y, int64_t n8) {
  pdl_wait();
  pdl_launch_dependents();
  const __half2 z = __floats2half2_rn(0.f, 0.f);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
    half8 v = ld8(x + i * 8);
    v.a = __hmax2(v.a, z); v.b = __hmax2(v.b, z); v.c = __hmax2(v.c, z); v.d = __hmax2(v.d, z);
    st8(y + i * 8, v);
  }
}
// dx (=|+=) dy where y > 0 (y = the ReLU output)
__global__ void relu_bwd_kernel(const __half* __restrict__ dy, const __half* __restrict__ y, __half* __restrict__ dx, int64_t n8, int accumulate) {
  pdl_wait();
  pdl_launch_dependents();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
    float g[8], o[8], a[8];
    unpack8(ld8(dy + i * 8), g);
    unpack8(ld8(y + i * 8), o);
    if (accumulate) unpack8(ld8(dx + i * 8), a);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float r = o[j] > 0.f ? g[j] : 0.f;
      a[j] = accumulate ? a[j] + r : r;
    }
    st8(dx + i * 8, pack8(a));
  }
}

// 2x2 / stride 2 max pool on [N, H, W, C] (H, W even)
__global__ void maxpool2_fwd_kernel(const __half* __restrict__ x, __half* __restrict__ y, int N, int H, int W, int C) {
  pdl_wait();
  pdl_launch_dependents();
  const int V = C / 8, Ho = H / 2, Wo = W / 2;
  const int64_t total = (int64_t)N * Ho * Wo * V;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % V);
    int64_t r = i / V;
    const int xo = (int)(r % Wo);
    r /= Wo;
    const int yo = (int)(r % Ho), n = (int)(r / Ho);
    const __half* p = x + (((int64_t)n * H + 2 * yo) * W + 2 * xo) * C + v * 8;
    half8 a = ld8(p), b = ld8(p + C), c = ld8(p + (int64_t)W * C), d = ld8(p + (int64_t)W * C + C);
    a.a = __hmax2(__hmax2(a.a, b.a), __hmax2(c.a, d.a));
    a.b = __hmax2(__hmax2(a.b, b.b), __hmax2(c.b, d.b));
    a.c = __hmax2(__hmax2(a.c, b.c), __hmax2(c.c, d.c));
    a.d = __hmax2(__hmax2(a.d, b.d), __hmax2(c.d, d.d));
    st8(y + i * 8, a);
  }
}
// dx[window] = dy at the FIRST position (row-major order of the window, like ATen) that holds the window maximum, 0 elsewhere
__global__ void maxpool2_bwd_kernel(const __half* __restrict__ dy, const __half* __restrict__ x, __half* __restrict__ dx, int N, int H, int W,
                                    int C) {
  pdl_wait();
  pdl_launch_dependents();
  const int V = C / 8, Ho = H / 2, Wo = W / 2;
  const int64_t total = (int64_t)N * Ho * Wo * V;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % V);
    int64_t r = i / V;
    const int xo = (int)(r % Wo);
    r /= Wo;
    const int yo = (int)(r % Ho), n = (int)(r / Ho);
    const int64_t base = (((int64_t)n * H + 2 * yo) * W + 2 * xo) * C + v * 8;
    const int64_t off[4] = {0, C, (int64_t)W * C, (int64_t)W * C + C};
    float w[4][8], g[8], o[4][8];
#pragma unroll
    for (int k = 0; k < 4; ++k) unpack8(ld8(x + base + off[k]), w[k]);
    unpack8(ld8(dy + i * 8), g);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int best = 0;
#pragma unroll
      for (int k = 1; k < 4; ++k)
        if (w[k][j] > w[best][j]) best = k;
#pragma unroll
      for (int k = 0; k < 4; ++k) o[k][j] = k == best ? g[j] : 0.f;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) st8(dx + base + off[k], pack8(o[k]));
  }
}

// One warp per pixel of one LPIPS tap.  f = features [B, HW, C] (post-ReLU), tn = normalised init-image features [Bt, HW, C]
// (Bt = 1 broadcasts), w = lin weights [C].  xh = f / (||f|| + 1e-10); loss_b += (1 / HW) sum_p sum_c w_c (xh_c - tn_c)^2;
// df = gscale / HW * d loss / d f saturated at +-60000, with d xh_c / d f_k = delta_ck / n - f_c f_k / (n^2 r), n = r + 1e-10, r = ||f||.
__global__ void lpips_tap_kernel(const __half* __restrict__ f, const __half* __restrict__ tn, const float* __restrict__ w, __half* __restrict__ df,
                                 float* __restrict__ loss_part, int B, int64_t HW, int C, int Bt, float gscale) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int64_t total = (int64_t)B * HW;
  const int nv = C / 8;  // 8 .. 64 vectors per pixel, lanes take v = lane, lane + 32
  float lsum = 0.f;
  int bcur = -1;
  for (int64_t pix = (int64_t)blockIdx.x * nw + wid; pix < total; pix += (int64_t)gridDim.x * nw) {
    const int b = (int)(pix / HW);
    const int64_t p = pix % HW;
    if (b != bcur) {  // a warp's pixel sequence crosses an image boundary at most a few times: flush the running loss
      if (bcur >= 0) {
        const float t = warp_sum(lsum);
        if (lane == 0) atomicAdd(loss_part + bcur, t / (float)HW);  // logged value only; the gradient path has no atomics
      }
      lsum = 0.f;
      bcur = b;
    }
    const __half* fp = f + pix * C;
    const __half* tp = tn + ((int64_t)(Bt == 1 ? 0 : b) * HW + p) * C;
    float x[2][8], t[2][8], ww[2][8];
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int v = lane + k * 32;
      if (v < nv) {
        unpack8(ld8(fp + v * 8), x[k]);
        unpack8(ld8(tp + v * 8), t[k]);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          ww[k][j] = w[v * 8 + j];
          ss = fmaf(x[k][j], x[k][j], ss);
        }
      }
    }
    ss = warp_sum(ss);
    const float r = sqrtf(ss), n = r + 1e-10f, inv_n = 1.f / n;
    float gx = 0.f, l = 0.f;  // sum_c g_c f_c, sum_c w_c (xh_c - t_c)^2
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int v = lane + k * 32;
      if (v < nv) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = x[k][j] * inv_n - t[k][j];
          const float g = 2.f * ww[k][j] * d;
          l = fmaf(ww[k][j] * d, d, l);
          gx = fmaf(g, x[k][j], gx);
          t[k][j] = g;  // keep g
        }
      }
    }
    gx = warp_sum(gx);
    lsum += l;
    const float c2 = r > 0.f ? gx / (n * n * r) : 0.f;
    const float sc = gscale / (float)HW;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int v = lane + k * 32;
      if (v < nv) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          // saturate like LPIPS_PAIR_BWD: at a pixel whose channels are all zero n = 1e-10 and the finite value is ~1e10 times
          // the usual size, which fp16 would store as inf; inf and NaN pass through
          const float u = (t[k][j] * inv_n - x[k][j] * c2) * sc;
          o[j] = isfinite(u) ? fminf(fmaxf(u, -60000.f), 60000.f) : u;
        }
        st8(df + pix * C + v * 8, pack8(o));
      }
    }
  }
  if (bcur >= 0) {
    const float t = warp_sum(lsum);
    if (lane == 0) atomicAdd(loss_part + bcur, t / (float)HW);
  }
}

__global__ void fill_f32_kernel(float* __restrict__ dst, int64_t n, float v) {
  pdl_wait();
  pdl_launch_dependents();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) dst[i] = v;
}
int launch_fill(const CgdOp& op, cudaStream_t st) {
  CGD_CHECK_ARG(op.i[0] > 0 && op.p[0], "fill: bad args");
  CGD_CUDA(launch_pdl(fill_f32_kernel, dim3(lp_blocks(op.i[0])), dim3(256), 0, st, (float*)op.p[0], op.i[0], op.f[0]));
  return 0;
}

int launch_relu_fwd(const CgdOp& op, cudaStream_t st) {
  const int64_t n = op.i[0];
  CGD_CHECK_ARG(n > 0 && n % 8 == 0 && op.p[0] && op.p[1], "relu_fwd: bad args");
  CGD_CUDA(launch_pdl(relu_fwd_kernel, dim3(lp_blocks(n / 8)), dim3(256), 0, st, (const __half*)op.p[0], (__half*)op.p[1], n / 8));
  return 0;
}
int launch_relu_bwd(const CgdOp& op, cudaStream_t st) {
  const int64_t n = op.i[0];
  CGD_CHECK_ARG(n > 0 && n % 8 == 0 && op.p[0] && op.p[1] && op.p[2], "relu_bwd: bad args");
  CGD_CUDA(launch_pdl(relu_bwd_kernel, dim3(lp_blocks(n / 8)), dim3(256), 0, st, (const __half*)op.p[0], (const __half*)op.p[1], (__half*)op.p[2], n / 8,
                      (int)((op.flags & 2) ? 1 : 0)));
  return 0;
}
int launch_maxpool2_fwd(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], H = op.i[1], W = op.i[2], C = op.i[3];
  CGD_CHECK_ARG(N > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && C % 8 == 0 && op.p[0] && op.p[1], "maxpool2: bad args");
  CGD_CUDA(launch_pdl(maxpool2_fwd_kernel, dim3(lp_blocks(N * (H / 2) * (W / 2) * (C / 8))), dim3(256), 0, st, (const __half*)op.p[0], (__half*)op.p[1],
                      (int)N, (int)H, (int)W, (int)C));
  return 0;
}
int launch_maxpool2_bwd(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], H = op.i[1], W = op.i[2], C = op.i[3];
  CGD_CHECK_ARG(N > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && C % 8 == 0 && op.p[0] && op.p[1] && op.p[2], "maxpool2_bwd: bad args");
  CGD_CUDA(launch_pdl(maxpool2_bwd_kernel, dim3(lp_blocks(N * (H / 2) * (W / 2) * (C / 8))), dim3(256), 0, st, (const __half*)op.p[0], (const __half*)op.p[1],
                      (__half*)op.p[2], (int)N, (int)H, (int)W, (int)C));
  return 0;
}
int launch_lpips_tap(const CgdOp& op, cudaStream_t st) {
  const int64_t B = op.i[0], HW = op.i[1], C = op.i[2], Bt = op.i[3];
  CGD_CHECK_ARG(B > 0 && HW > 0 && C % 8 == 0 && C >= 8 && C <= 512 && (Bt == 1 || Bt == B), "lpips_tap: bad dims (C <= 512)");
  CGD_CHECK_ARG(op.p[0] && op.p[1] && op.p[2] && op.p[3] && op.p[4], "lpips_tap: null pointer");
  CGD_CUDA(launch_pdl(lpips_tap_kernel, dim3(lp_blocks(B * HW, 8)), dim3(256), 0, st, (const __half*)op.p[0], (const __half*)op.p[1], (const float*)op.p[2],
                      (__half*)op.p[3], (float*)op.p[4], (int)B, HW, (int)C, (int)Bt, op.f[0]));
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// LPIPS(in0, in1) under torch.autograd (clip_guided_diffusion_b200/lpips.py, LPIPS): both sides are VGG trunks of the plan, so a tap
// holds the raw post-ReLU features of both, f0 [N0, HW, C] and f1 [N1, HW, C]; N0, N1 are B or 1 (broadcast: row 0 serves every image).
// Deterministic throughout: the value is reduced in a fixed order (LPIPS_PAIR_FWD partials, LPIPS_LOSS), the gradient has no sums across
// threads other than fixed warp butterflies and a fixed per-row loop over the images a broadcast row serves.

static inline bool lp_aligned(const void* p, uintptr_t a) { return ((uintptr_t)p & (a - 1)) == 0; }

// shared dims of the two per-tap ops: 0, or -1 with the error set
static int check_pair_dims(const CgdOp& op, const char* what) {
  const int64_t B = op.i[0], HW = op.i[1], C = op.i[2], N0 = op.i[3], N1 = op.i[4];
  CGD_CHECK_ARG(B > 0 && B <= 65535 && HW > 0 && HW <= (1LL << 26), "%s: B %lld / HW %lld out of range", what, (long long)B, (long long)HW);
  CGD_CHECK_ARG(C >= 8 && C <= 512 && C % 8 == 0, "%s: C %lld must be a multiple of 8 in [8, 512]", what, (long long)C);
  CGD_CHECK_ARG((N0 == B || N0 == 1) && (N1 == B || N1 == 1), "%s: N0 %lld / N1 %lld must be B (%lld) or 1", what, (long long)N0,
                (long long)N1, (long long)B);
  return 0;
}

// one warp per pixel: lanes hold channel vectors v = lane, lane + 32 (8 halfs each); returns ||f|| summed by the warp butterfly
__device__ __forceinline__ float lp_load_pixel(const __half* __restrict__ p, int nv, int lane, float (&x)[2][8]) {
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int v = lane + k * 32;
    if (v < nv) {
      unpack8(ld8(p + v * 8), x[k]);
#pragma unroll
      for (int j = 0; j < 8; ++j) ss = fmaf(x[k][j], x[k][j], ss);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) x[k][j] = 0.f;
    }
  }
  return __fsqrt_rn(warp_sum(ss));
}

// grid (nblk, B), 8 warps: warp w of block x takes pixels x * 8 + w + k * nblk * 8 of image blockIdx.y; each lane keeps its own running
// sum of w_c (xh0_c - xh1_c)^2; the warp and then the block (warps 0..7 in order) reduce it into partial[b * nblk + x]
__global__ void __launch_bounds__(256, 1) lpips_pair_fwd_kernel(const __half* __restrict__ f0, const __half* __restrict__ f1, const float* __restrict__ w,
                                                             float* __restrict__ partial, int64_t HW, int C, int N0, int N1, int nblk) {
  __shared__ float red[8];
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, b = blockIdx.y, nv = C / 8;
  const __half* a0 = f0 + (int64_t)(N0 == 1 ? 0 : b) * HW * C;
  const __half* a1 = f1 + (int64_t)(N1 == 1 ? 0 : b) * HW * C;
  float ww[2][8];
#pragma unroll
  for (int k = 0; k < 2; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) ww[k][j] = (lane + k * 32 < nv) ? w[(lane + k * 32) * 8 + j] : 0.f;
  float l = 0.f;
  for (int64_t p = (int64_t)blockIdx.x * 8 + wid; p < HW; p += (int64_t)nblk * 8) {
    float x[2][8], y[2][8];
    const float i0 = __frcp_rn(lp_load_pixel(a0 + p * C, nv, lane, x) + 1e-10f);
    const float i1 = __frcp_rn(lp_load_pixel(a1 + p * C, nv, lane, y) + 1e-10f);
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = x[k][j] * i0 - y[k][j] * i1;
        l = fmaf(ww[k][j] * d, d, l);
      }
  }
  l = warp_sum(l);
  if (lane == 0) red[wid] = l;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += red[k];
    partial[(int64_t)b * nblk + blockIdx.x] = s;
  }
}

int launch_lpips_pair_fwd(const CgdOp& op, cudaStream_t st) {
  CGD_CHECK_ARG(op.flags == 0, "lpips_pair_fwd: flags must be 0");
  if (check_pair_dims(op, "lpips_pair_fwd")) return -1;
  const int64_t nblk = op.i[5];
  CGD_CHECK_ARG(nblk >= 1 && nblk <= 4096, "lpips_pair_fwd: %lld blocks per image, want 1..4096", (long long)nblk);
  CGD_CHECK_ARG(op.p[0] && op.p[1] && op.p[2] && op.p[3] && lp_aligned(op.p[0], 16) && lp_aligned(op.p[1], 16) && lp_aligned(op.p[2], 4) &&
                    lp_aligned(op.p[3], 4),
                "lpips_pair_fwd: null or misaligned pointer");
  CGD_CUDA(launch_pdl(lpips_pair_fwd_kernel, dim3((unsigned)nblk, (unsigned)op.i[0]), dim3(256), 0, st, (const __half*)op.p[0], (const __half*)op.p[1],
                      (const float*)op.p[2], (float*)op.p[3], op.i[1], (int)op.i[2], (int)op.i[3], (int)op.i[4], (int)nblk));
  CGD_LAUNCH_CHECK();
  return 0;
}

// one CTA of 256 threads per image: tap k's nblk_k partials summed thread-strided then by block_sum's fixed tree, times 1 / HW_k, and
// the five taps added in order 0..4
struct LpipsLossArgs {
  const float* part[5];
  int nblk[5];
  float inv_hw[5];
};
__global__ void __launch_bounds__(256) lpips_loss_kernel(LpipsLossArgs a, float* __restrict__ loss) {
  __shared__ float red[32];
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.x;
  float total = 0.f;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    float s = 0.f;
    for (int j = threadIdx.x; j < a.nblk[k]; j += blockDim.x) s += a.part[k][(int64_t)b * a.nblk[k] + j];
    total += block_sum(s, red) * a.inv_hw[k];
  }
  if (threadIdx.x == 0) loss[b] = total;
}

int launch_lpips_loss(const CgdOp& op, cudaStream_t st) {
  CGD_CHECK_ARG(op.flags == 0, "lpips_loss: flags must be 0");
  const int64_t B = op.i[0];
  CGD_CHECK_ARG(B > 0 && B <= 65535, "lpips_loss: B %lld out of range", (long long)B);
  LpipsLossArgs a;
  for (int k = 0; k < 5; ++k) {
    CGD_CHECK_ARG(op.i[1 + k] >= 1 && op.i[1 + k] <= 4096, "lpips_loss: tap %d has %lld partials per image, want 1..4096", k, (long long)op.i[1 + k]);
    CGD_CHECK_ARG(op.f[k] > 0.f && op.f[k] <= 1.f, "lpips_loss: 1 / HW of tap %d must be in (0, 1]", k);
    CGD_CHECK_ARG(op.p[k] && lp_aligned(op.p[k], 4), "lpips_loss: null or misaligned partials of tap %d", k);
    a.part[k] = (const float*)op.p[k];
    a.nblk[k] = (int)op.i[1 + k];
    a.inv_hw[k] = op.f[k];
  }
  CGD_CHECK_ARG(op.p[5] && lp_aligned(op.p[5], 4), "lpips_loss: null or misaligned loss");
  CGD_CUDA(launch_pdl(lpips_loss_kernel, dim3((unsigned)B), dim3(256), 0, st, a, (float*)op.p[5]));
  CGD_LAUNCH_CHECK();
  return 0;
}

// one thread per trunk row j of [trunk 0 rows | trunk 1 rows]: m = |d[j]| for a row of its own image, the maximum over every image for a
// broadcast row (NaN dropped, inf counted as 3e38); s = 2^clamp(floor(log2(band / m)), -60, 60), 1 where m == 0
__global__ void lpips_seed_kernel(const float* __restrict__ d, float* __restrict__ dyn, int B, int N0, int N1, float band) {
  pdl_wait();
  pdl_launch_dependents();
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < N0 + N1; j += gridDim.x * blockDim.x) {
    const int side_n = j < N0 ? N0 : N1, r = j < N0 ? j : j - N0;
    float m = 0.f;
    if (side_n == B) {
      m = fmaxf(m, fabsf(d[r]));  // fmaxf drops a NaN
    } else {
      for (int b = 0; b < B; ++b) m = fmaxf(m, fabsf(d[b]));
    }
    m = fminf(m, 3.0e38f);
    dyn[j] = m > 0.f ? exp2f(fminf(fmaxf(floorf(log2f(band / m)), -60.f), 60.f)) : 1.f;
  }
}

int launch_lpips_seed(const CgdOp& op, cudaStream_t st) {
  const int64_t B = op.i[0], N0 = op.i[1], N1 = op.i[2];
  const float band = op.f[0];
  CGD_CHECK_ARG(op.flags == 0, "lpips_seed: flags must be 0");
  CGD_CHECK_ARG(B > 0 && B <= 65535 && (N0 == B || N0 == 1) && (N1 == B || N1 == 1), "lpips_seed: B %lld / N0 %lld / N1 %lld invalid",
                (long long)B, (long long)N0, (long long)N1);
  int e = 0;
  CGD_CHECK_ARG(band >= 1.f && band <= 1073741824.f && frexpf(band, &e) == 0.5f, "lpips_seed: BAND %g must be a power of two in [1, 2^30]", band);
  CGD_CHECK_ARG(op.p[0] && op.p[1] && lp_aligned(op.p[0], 4) && lp_aligned(op.p[1], 4), "lpips_seed: null or misaligned pointer");
  CGD_CUDA(launch_pdl(lpips_seed_kernel, dim3((unsigned)ceil_div(N0 + N1, 256)), dim3(256), 0, st, (const float*)op.p[0], (float*)op.p[1], (int)B,
                      (int)N0, (int)N1, band));
  CGD_LAUNCH_CHECK();
  return 0;
}

// one warp per (side, row, pixel).  The row's seed is sum over the images b it serves (b = row, or every image for a broadcast row, in
// order) of a_b * d LPIPS_b / d f, a_b = (d_loss[b] * s_row) / HW, with d / d f_k of sum_c w_c (xh_c - xo_c)^2 = g_k / n - f_k (g . f) / (n^2 r),
// g = 2 w (xh - xo), r = ||f||, n = r + 1e-10 (the other side's xo is a constant).  fp32 throughout, one fp16 rounding; finite values
// saturate at +-60000 (a pixel whose channels are all zero has n = 1e-10: its finite seed is ~1e10 times the usual size), inf and NaN pass.
__global__ void __launch_bounds__(256) lpips_pair_bwd_kernel(const __half* __restrict__ f0, const __half* __restrict__ f1, const float* __restrict__ w,
                                                             const float* __restrict__ d_loss, const float* __restrict__ dyn, __half* __restrict__ df0,
                                                             __half* __restrict__ df1, int B, int64_t HW, int C, int N0, int N1, float inv_hw) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31, nv = C / 8;
  const int64_t items0 = df0 ? (int64_t)N0 * HW : 0, total = items0 + (df1 ? (int64_t)N1 * HW : 0);
  const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  float ww[2][8];
#pragma unroll
  for (int k = 0; k < 2; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) ww[k][j] = (lane + k * 32 < nv) ? 2.f * w[(lane + k * 32) * 8 + j] : 0.f;
  for (int64_t it = gw; it < total; it += nw) {
    const bool side1 = it >= items0;
    const int64_t loc = side1 ? it - items0 : it;
    const int r = (int)(loc / HW);
    const int64_t p = loc % HW;
    const __half* fs = side1 ? f1 : f0;
    const __half* fo = side1 ? f0 : f1;
    const int ns = side1 ? N1 : N0, no = side1 ? N0 : N1;
    const float srow = dyn[(side1 ? N0 : 0) + r];
    float x[2][8], acc[2][8];
    const float rs = lp_load_pixel(fs + ((int64_t)r * HW + p) * C, nv, lane, x);
    const float n = rs + 1e-10f, inv_n = __frcp_rn(n);
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[k][j] = 0.f;
    const int b0 = ns == B ? r : 0, b1 = ns == B ? r + 1 : B;
    for (int b = b0; b < b1; ++b) {
      float y[2][8];
      const float io = __frcp_rn(lp_load_pixel(fo + ((int64_t)(no == 1 ? 0 : b) * HW + p) * C, nv, lane, y) + 1e-10f);
      const float a = (d_loss[b] * srow) * inv_hw;
      float gx = 0.f;
#pragma unroll
      for (int k = 0; k < 2; ++k)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          y[k][j] = ww[k][j] * (x[k][j] * inv_n - y[k][j] * io);  // g
          gx = fmaf(y[k][j], x[k][j], gx);
        }
      gx = warp_sum(gx);
      const float c2 = rs > 0.f ? gx / (n * n * rs) : 0.f;
#pragma unroll
      for (int k = 0; k < 2; ++k)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[k][j] = fmaf(a, y[k][j] * inv_n - x[k][j] * c2, acc[k][j]);
    }
    __half* dst = (side1 ? df1 : df0) + ((int64_t)r * HW + p) * C;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int v = lane + k * 32;
      if (v < nv) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = isfinite(acc[k][j]) ? fminf(fmaxf(acc[k][j], -60000.f), 60000.f) : acc[k][j];
        st8(dst + v * 8, pack8(o));
      }
    }
  }
}

int launch_lpips_pair_bwd(const CgdOp& op, cudaStream_t st) {
  CGD_CHECK_ARG(op.flags >= 1 && op.flags <= 3, "lpips_pair_bwd: flags must be 1 (d f0), 2 (d f1) or 3 (both)");
  if (check_pair_dims(op, "lpips_pair_bwd")) return -1;
  const bool s0 = op.flags & 1, s1 = op.flags & 2;
  CGD_CHECK_ARG(op.p[0] && op.p[1] && op.p[2] && op.p[3] && op.p[4] && lp_aligned(op.p[0], 16) && lp_aligned(op.p[1], 16) &&
                    lp_aligned(op.p[2], 4) && lp_aligned(op.p[3], 4) && lp_aligned(op.p[4], 4),
                "lpips_pair_bwd: null or misaligned pointer");
  CGD_CHECK_ARG((s0 ? op.p[5] != nullptr && lp_aligned(op.p[5], 16) : op.p[5] == nullptr) &&
                    (s1 ? op.p[6] != nullptr && lp_aligned(op.p[6], 16) : op.p[6] == nullptr),
                "lpips_pair_bwd: d f0 / d f1 pointers must be set (16-byte aligned) exactly for the sides the flags select");
  const int64_t rows = (s0 ? op.i[3] : 0) + (s1 ? op.i[4] : 0);
  CGD_CUDA(launch_pdl(lpips_pair_bwd_kernel, dim3(lp_blocks(rows * op.i[1], 8)), dim3(256), 0, st, (const __half*)op.p[0], (const __half*)op.p[1],
                      (const float*)op.p[2], (const float*)op.p[3], (const float*)op.p[4], (__half*)op.p[5], (__half*)op.p[6], (int)op.i[0], op.i[1],
                      (int)op.i[2], (int)op.i[3], (int)op.i[4], 1.f / (float)op.i[1]));
  CGD_LAUNCH_CHECK();
  return 0;
}

}  // namespace cgd
