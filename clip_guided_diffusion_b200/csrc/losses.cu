// losses.cu -- the reference's loss functions (cgd/losses.py:5-22) as stand-alone differentiable ops, for a cond_fn written in
// PyTorch (clip_guided_diffusion_b200/losses.py).  fp32 throughout; every sum runs in a fixed order, with no atomics, so two runs give the
// same bits.  The fused step keeps its own kernels (guidance.cu: GUIDE_GRAD, SPHERICAL).
//
//   IMG_LOSS_FWD / _BWD   tv_loss, range_loss per image of [B, C, H, W]   cgd/losses.py:5-7, 17-22
//   SPH_DIST_FWD / _BWD   spherical_dist_loss over a list of row pairs    cgd/losses.py:10-14
#include <math.h>
#include <stdint.h>

#include <algorithm>

#include "common.cuh"
#include "ops.cuh"
#include "pdl.cuh"

namespace cgd {

static inline bool aligned4(const void* p) { return ((uintptr_t)p & 3u) == 0; }

// ---------------------------------------------------------------- tv / range
// KIND 1 = tv_loss: replicate pad, so the last column's x difference and the last row's y difference are 0; 2 = range_loss
template <int KIND>
__device__ __forceinline__ float img_loss_term(const float* __restrict__ xb, int64_t i, int64_t HW, int H, int W) {
  const float v = xb[i];
  if constexpr (KIND == 1) {
    const int64_t p = i % HW;
    const int h = (int)(p / W), w = (int)(p % W);
    const float xd = (w + 1 < W) ? xb[i + 1] - v : 0.f;
    const float yd = (h + 1 < H) ? xb[i + W] - v : 0.f;
    return xd * xd + yd * yd;
  } else {
    const float e = v - fminf(fmaxf(v, -1.f), 1.f);
    return e * e;
  }
}

// grid (nblk, B): CTA j of image b sums elements j * 256 + t + k * nblk * 256 (thread order, then the block_sum tree)
template <int KIND>
__global__ void __launch_bounds__(256) img_loss_partial_kernel(const float* __restrict__ x, float* __restrict__ partial, int C, int H, int W,
                                                               int nblk) {
  __shared__ float red[32];
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.y;
  const int64_t HW = (int64_t)H * W, per = (int64_t)C * HW;
  const float* xb = x + (int64_t)b * per;
  float s = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < per; i += (int64_t)nblk * blockDim.x) s += img_loss_term<KIND>(xb, i, HW, H, W);
  s = block_sum(s, red);
  if (threadIdx.x == 0) partial[(int64_t)b * nblk + blockIdx.x] = s;
}

// loss[b] = (partials of image b summed in CTA order) / (C H W): the reference's mean over dims 1..3
__global__ void img_loss_fold_kernel(const float* __restrict__ partial, float* __restrict__ loss, int B, int nblk, float n) {
  pdl_wait();
  pdl_launch_dependents();
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int j = 0; j < nblk; ++j) s += partial[(int64_t)b * nblk + j];
    loss[b] = s / n;
  }
}

// dx = d_loss[b] * d loss_b / d x: tv 2 / N (x[w] - x[w-1] + x[h] - x[h-1] - xd - yd), range 2 / N (x - clamp(x, -1, 1))
template <int KIND>
__global__ void img_loss_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dl, float* __restrict__ dx, int B, int C, int H, int W) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t HW = (int64_t)H * W, per = (int64_t)C * HW, total = (int64_t)B * per;
  const float two_n = 2.f / (float)per;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = idx / per;
    const float v = x[idx];
    float g;
    if constexpr (KIND == 1) {
      const int64_t p = idx % HW;
      const int h = (int)(p / W), w = (int)(p % W);
      const float xd = (w + 1 < W) ? x[idx + 1] - v : 0.f;
      const float yd = (h + 1 < H) ? x[idx + W] - v : 0.f;
      const float xdl = (w > 0) ? v - x[idx - 1] : 0.f;
      const float ydu = (h > 0) ? v - x[idx - W] : 0.f;
      g = (xdl + ydu) - (xd + yd);
    } else {
      g = v - fminf(fmaxf(v, -1.f), 1.f);
    }
    dx[idx] = dl[b] * two_n * g;
  }
}

static int img_loss_check(const CgdOp& op, const char* name) {
  const int64_t B = op.i[0], C = op.i[1], H = op.i[2], W = op.i[3];
  CGD_CHECK_ARG(op.flags == 1 || op.flags == 2, "%s: flags must be 1 (tv_loss) or 2 (range_loss), got %d", name, op.flags);
  CGD_CHECK_ARG(B > 0 && C > 0 && H > 0 && W > 0 && B <= 65535 && C <= 65535 && H <= (1 << 20) && W <= (1 << 20) && C * H * W <= ((int64_t)1 << 40),
                "%s: bad dims B=%lld C=%lld H=%lld W=%lld", name, (long long)B, (long long)C, (long long)H, (long long)W);
  return 0;
}

int launch_img_loss_fwd(const CgdOp& op, cudaStream_t st) {
  if (img_loss_check(op, "img_loss_fwd")) return -1;
  const int64_t B = op.i[0], C = op.i[1], H = op.i[2], W = op.i[3], nblk = op.i[4];
  CGD_CHECK_ARG(nblk >= 1 && nblk <= 4096, "img_loss_fwd: nblk must be in 1..4096, got %lld", (long long)nblk);
  CGD_CHECK_ARG(op.p[0] && op.p[1] && op.p[2] && aligned4(op.p[0]) && aligned4(op.p[1]) && aligned4(op.p[2]),
                "img_loss_fwd: null or misaligned pointer (x, partials, loss)");
  CGD_CUDA(launch_pdl(op.flags == 1 ? img_loss_partial_kernel<1> : img_loss_partial_kernel<2>, dim3((unsigned)nblk, (unsigned)B), dim3(256), 0, st,
                      (const float*)op.p[0], (float*)op.p[1], (int)C, (int)H, (int)W, (int)nblk));
  CGD_LAUNCH_CHECK();
  CGD_CUDA(launch_pdl(img_loss_fold_kernel, dim3((unsigned)ceil_div(B, 128)), dim3(128), 0, st, (const float*)op.p[1], (float*)op.p[2], (int)B,
                      (int)nblk, (float)(C * H * W)));
  CGD_LAUNCH_CHECK();
  return 0;
}

int launch_img_loss_bwd(const CgdOp& op, cudaStream_t st) {
  if (img_loss_check(op, "img_loss_bwd")) return -1;
  const int64_t B = op.i[0], C = op.i[1], H = op.i[2], W = op.i[3];
  CGD_CHECK_ARG(op.p[0] && op.p[1] && op.p[2] && aligned4(op.p[0]) && aligned4(op.p[1]) && aligned4(op.p[2]),
                "img_loss_bwd: null or misaligned pointer (x, d_loss, dx)");
  const int64_t blocks = std::min<int64_t>(ceil_div(B * C * H * W, 256), 132 * 8);
  CGD_CUDA(launch_pdl(op.flags == 1 ? img_loss_bwd_kernel<1> : img_loss_bwd_kernel<2>, dim3((unsigned)blocks), dim3(256), 0, st,
                      (const float*)op.p[0], (const float*)op.p[1], (float*)op.p[2], (int)B, (int)C, (int)H, (int)W));
  CGD_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------- spherical distance over row pairs
// F.normalize's max(||r||, 1e-12), one warp per row
__device__ __forceinline__ float sph_norm(const float* __restrict__ r, int D, int lane) {
  float s = 0.f;
  for (int d = lane; d < D; d += 32) s = fmaf(r[d], r[d], s);
  return fmaxf(sqrtf(warp_sum(s)), 1e-12f);
}

// |r / rn - o / on| of two rows, every lane gets it
__device__ __forceinline__ float sph_gap(const float* __restrict__ r, float rn, const float* __restrict__ o, float on, int D, int lane) {
  float s = 0.f;
  for (int d = lane; d < D; d += 32) {
    const float df = r[d] / rn - o[d] / on;
    s = fmaf(df, df, s);
  }
  return sqrtf(warp_sum(s));
}

constexpr int SPH_WARPS = 8;

// out[m] = 2 asin(min(|x^ - y^| / 2, 1))^2 for pair m = (x row, y row); a row index out of range gives NaN
__global__ void __launch_bounds__(32 * SPH_WARPS) sph_dist_fwd_kernel(const float* __restrict__ x, const float* __restrict__ y, const int* __restrict__ pairs,
                                                                      float* __restrict__ out, int M, int D, int Nx, int Ny) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int nw = gridDim.x * SPH_WARPS;
  for (int m = blockIdx.x * SPH_WARPS + (threadIdx.x >> 5); m < M; m += nw) {
    const int ix = pairs[2 * (int64_t)m], iy = pairs[2 * (int64_t)m + 1];
    float r = __int_as_float(0x7fc00000);
    if (ix >= 0 && ix < Nx && iy >= 0 && iy < Ny) {
      const float* xr = x + (int64_t)ix * D;
      const float* yr = y + (int64_t)iy * D;
      const float h = fminf(sph_gap(xr, sph_norm(xr, D, lane), yr, sph_norm(yr, D, lane), D, lane) * 0.5f, 1.f);
      const float a = asinf(h);
      r = 2.f * a * a;
    }
    if (lane == 0) out[m] = r;
  }
}

// One warp per output row s (x rows, then y rows), over the pairs that use it in CSR order (idx[ptr[s] .. ptr[s+1]), host-built):
//   G = sum_m d_out[m] * 2 asin(h) / sqrt(1 - h^2) / n * (s^ - o^),  n = |s^ - o^|, h = min(n / 2, 1)  (0 where n == 0, like torch's
//   norm backward), then back through F.normalize: (G - s^ (s^ . G)) / ||s|| (G / 1e-12 where ||s|| <= 1e-12).  G is accumulated in the
//   output row itself, each element by one lane in pair order.  A pair or row index out of range makes the row NaN.
__global__ void __launch_bounds__(32 * SPH_WARPS) sph_dist_bwd_kernel(const float* __restrict__ x, const float* __restrict__ y, const int* __restrict__ pairs,
                                                                      const float* __restrict__ dout, float* __restrict__ dx, float* __restrict__ dy,
                                                                      const int* __restrict__ xptr, const int* __restrict__ xidx,
                                                                      const int* __restrict__ yptr, const int* __restrict__ yidx, int M, int D, int Nx,
                                                                      int Ny) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int nw = gridDim.x * SPH_WARPS;
  for (int row = blockIdx.x * SPH_WARPS + (threadIdx.x >> 5); row < Nx + Ny; row += nw) {
    const int side = row < Nx ? 0 : 1, s = side ? row - Nx : row;
    float* G = side ? dy : dx;
    if (!G) continue;
    G += (int64_t)s * D;
    const float* S = (side ? y : x) + (int64_t)s * D;
    const float* O0 = side ? x : y;
    const int No = side ? Nx : Ny;
    const int* ptr = side ? yptr : xptr;
    const int* idx = side ? yidx : xidx;
    const float sn = sph_norm(S, D, lane);
    for (int d = lane; d < D; d += 32) G[d] = 0.f;
    int j0 = ptr[s], j1 = ptr[s + 1];
    bool bad = j0 < 0 || j1 > M || j0 > j1;
    for (int j = bad ? j1 : j0; j < j1; ++j) {
      const int m = idx[j];
      const int o = (m >= 0 && m < M) ? pairs[2 * (int64_t)m + 1 - side] : -1;
      if (o < 0 || o >= No || pairs[2 * (int64_t)m + side] != s) {
        bad = true;
        break;
      }
      const float* O = O0 + (int64_t)o * D;
      const float on = sph_norm(O, D, lane);
      const float n = sph_gap(S, sn, O, on, D, lane);
      const float h = fminf(n * 0.5f, 1.f);
      const float coef = n > 0.f ? dout[m] * (2.f * asinf(h) * rsqrtf(fmaxf(1.f - h * h, 1e-20f))) / n : 0.f;
      for (int d = lane; d < D; d += 32) G[d] = fmaf(coef, S[d] / sn - O[d] / on, G[d]);
    }
    __syncwarp();
    if (bad) {
      for (int d = lane; d < D; d += 32) G[d] = __int_as_float(0x7fc00000);
      continue;
    }
    float dot = 0.f;
    for (int d = lane; d < D; d += 32) dot = fmaf(S[d] / sn, G[d], dot);
    dot = warp_sum(dot);
    const bool clamped = sn <= 1e-12f;  // ||s|| below F.normalize's eps: s / 1e-12, no projection
    for (int d = lane; d < D; d += 32) G[d] = clamped ? G[d] / sn : (G[d] - S[d] / sn * dot) / sn;
  }
}

static int sph_check(const CgdOp& op, const char* name) {
  const int64_t M = op.i[0], D = op.i[1], Nx = op.i[2], Ny = op.i[3];
  CGD_CHECK_ARG(M > 0 && D > 0 && Nx > 0 && Ny > 0 && M <= (1 << 30) && D <= (1 << 20) && Nx <= (1 << 30) && Ny <= (1 << 30) && Nx + Ny <= (1 << 30),
                "%s: bad dims M=%lld D=%lld Nx=%lld Ny=%lld", name, (long long)M, (long long)D, (long long)Nx, (long long)Ny);
  CGD_CHECK_ARG(op.p[0] && op.p[1] && op.p[2] && aligned4(op.p[0]) && aligned4(op.p[1]) && aligned4(op.p[2]), "%s: null or misaligned pointer (x, y, pairs)",
                name);
  return 0;
}

static inline unsigned sph_blocks(int64_t warps) { return (unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div(warps, SPH_WARPS), 132 * 16)); }

int launch_sph_dist_fwd(const CgdOp& op, cudaStream_t st) {
  if (sph_check(op, "sph_dist_fwd")) return -1;
  CGD_CHECK_ARG(op.flags == 0, "sph_dist_fwd: flags must be 0, got %d", op.flags);
  CGD_CHECK_ARG(op.p[3] && aligned4(op.p[3]), "sph_dist_fwd: null or misaligned pointer (out)");
  CGD_CUDA(launch_pdl(sph_dist_fwd_kernel, dim3(sph_blocks(op.i[0])), dim3(32 * SPH_WARPS), 0, st, (const float*)op.p[0], (const float*)op.p[1],
                      (const int*)op.p[2], (float*)op.p[3], (int)op.i[0], (int)op.i[1], (int)op.i[2], (int)op.i[3]));
  CGD_LAUNCH_CHECK();
  return 0;
}

int launch_sph_dist_bwd(const CgdOp& op, cudaStream_t st) {
  if (sph_check(op, "sph_dist_bwd")) return -1;
  CGD_CHECK_ARG(op.flags >= 1 && op.flags <= 3, "sph_dist_bwd: flags must be 1 (d x), 2 (d y) or 3 (both), got %d", op.flags);
  CGD_CHECK_ARG(op.p[3] && aligned4(op.p[3]), "sph_dist_bwd: null or misaligned pointer (d_out)");
  for (int s = 0; s < 2; ++s) {
    const bool want = op.flags & (1 << s);
    const void* g = op.p[4 + s];
    const void* ptr = op.p[6 + 2 * s];
    const void* idx = op.p[7 + 2 * s];
    CGD_CHECK_ARG(want ? (g && ptr && idx && aligned4(g) && aligned4(ptr) && aligned4(idx)) : (!g && !ptr && !idx),
                  "sph_dist_bwd: the gradient and CSR pointers of side %d must be set (4-byte aligned) exactly when the flags select it", s);
  }
  CGD_CUDA(launch_pdl(sph_dist_bwd_kernel, dim3(sph_blocks(op.i[2] + op.i[3])), dim3(32 * SPH_WARPS), 0, st, (const float*)op.p[0],
                      (const float*)op.p[1], (const int*)op.p[2], (const float*)op.p[3], (float*)op.p[4], (float*)op.p[5], (const int*)op.p[6],
                      (const int*)op.p[7], (const int*)op.p[8], (const int*)op.p[9], (int)op.i[0], (int)op.i[1], (int)op.i[2], (int)op.i[3]));
  CGD_LAUNCH_CHECK();
  return 0;
}

}  // namespace cgd
