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
// df = gscale / HW * d loss / d f, with d xh_c / d f_k = delta_ck / n - f_c f_k / (n^2 r), n = r + 1e-10, r = ||f||.
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
        for (int j = 0; j < 8; ++j) o[j] = (t[k][j] * inv_n - x[k][j] * c2) * sc;
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

}  // namespace cgd
