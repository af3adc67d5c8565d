// norm_stream.cu -- GroupNorm(32) (+SiLU, +scale/shift) forward and input gradient for LARGE activations as plain streaming
// kernels: the third engine behind the ops GN_FWD_GRID / GN_BWD_GRID / GN_APPLY_EPI (C % 256 == 0).
//
// Why: the persistent one-launch kernels (norm_grid.cu ring, norm_grid2.cu direct) run ONE 544- / 1024-thread CTA per SM whose
// threads move in lock-step through load -> compute phases, with a software grid barrier and a per-CTA fold between the two trips.
// That schedule, at 25 - 50 % occupancy, rather than the traffic can bound them; the elementwise kernels of this library
// (elementwise.cu: 256-thread CTAs, 8 per SM, grid-stride, one 16-byte vector per trip) are shaped for streaming, so: the same shape here.
//   forward :  [gn_stats_stream | conv-epilogue partials]  ->  gn_fold  ->  gn_apply_stream
//   backward:   gn_bwd_stats_stream                        ->  gn_fold  ->  gn_bwd_apply_stream
// Three short launches (PDL-chained) instead of one persistent one; every thread owns one 8-channel column for the whole kernel
// (per-channel coefficients in registers), partial sums are per CTA, folded in a fixed order in double precision (bit-reproducible).
//
// Replaces [3P] guided-diffusion GroupNorm32 + SiLU + scale-shift and their autograd (SURVEY.md K5, K6).
#include <algorithm>

#include "common.cuh"
#include "ops.cuh"
#include "pdl.cuh"

namespace cgd {

constexpr int kGsThreads = 256;
constexpr int kGsMaxCtas = 132 * 8;  // partial slots per launch (plan.py allocates N * kGsMaxCtas * 64 floats at most)

__device__ __forceinline__ uint4 gs_ld(const __half* p) {
  uint4 v;
  asm volatile("ld.global.nc.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ float2 gs_h2f(uint32_t w) { return __half22float2(*reinterpret_cast<const __half2*>(&w)); }
__device__ __forceinline__ uint32_t gs_f2h(float2 f) {
  const __half2 h = __floats2half2_rn(f.x, f.y);
  return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ void gs_unpack(const uint4& v, float2 (&f)[4]) {
  f[0] = gs_h2f(v.x);
  f[1] = gs_h2f(v.y);
  f[2] = gs_h2f(v.z);
  f[3] = gs_h2f(v.w);
}

// thread -> (row slot, column): V threads per pixel row, RP rows per CTA pass, the remaining threads of the CTA idle
struct GsMap {
  int V, RP, col, slot;
  bool active;
  __device__ __forceinline__ GsMap(int C) {
    V = C / 8;
    RP = kGsThreads / V;
    col = threadIdx.x % V;
    slot = threadIdx.x / V;
    active = slot < RP;
  }
};

// per-channel affine of this thread's 8 channels: v = x * A + B  (A = rstd * gamma * (1 + scale), B = (beta - mean * rstd * gamma) * (1 + scale) + shift)
__device__ __forceinline__ void gs_coef(int n, int col, int C, const float* __restrict__ gamma, const float* __restrict__ beta,
                                        const float* __restrict__ emb, float mu, float rs, float2 (&A)[4], float2 (&B)[4], float2 (&G)[4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float a[2], b[2], g[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = col * 8 + 2 * j + h;
      const float ga = gamma[c], be = beta[c];
      const float sc1 = emb ? 1.f + emb[(int64_t)n * 2 * C + c] : 1.f, sh = emb ? emb[(int64_t)n * 2 * C + C + c] : 0.f;
      g[h] = ga * sc1;
      a[h] = rs * ga * sc1;
      b[h] = (be - mu * rs * ga) * sc1 + sh;
    }
    A[j] = make_float2(a[0], a[1]);
    B[j] = make_float2(b[0], b[1]);
    G[j] = make_float2(g[0], g[1]);
  }
}

// (ts, tq) of every thread -> the CTA's 32 group sums -> partials[cta][32][2]; fixed order: row slots ascending, then columns ascending
__device__ __forceinline__ void gs_block_partials(const GsMap& m, int vpg, float ts, float tq, float* red, float* out) {
  // red: [kGsThreads][2]
  red[2 * threadIdx.x] = m.active ? ts : 0.f;
  red[2 * threadIdx.x + 1] = m.active ? tq : 0.f;
  __syncthreads();
  if (threadIdx.x < 32) {
    const int g = threadIdx.x;
    float s = 0.f, q = 0.f;
    for (int o = 0; o < vpg; ++o) {
      const int c = g * vpg + o;
      for (int r = 0; r < m.RP; ++r) {
        s += red[2 * (r * m.V + c)];
        q += red[2 * (r * m.V + c) + 1];
      }
    }
    out[2 * g] = s;
    out[2 * g + 1] = q;
  }
}

// ------------------------------------------------------------------------------------------------ fold
// sums[n][g][2] = sum over the partials of image n, group g.  mode 0: partials [n][G][32][2] (one row per CTA of a *_stats_stream
// launch); mode 1: conv-epilogue partials [n * tpi + tile][octs][2] (CONV flags 2), group g = octets [oct0 + g * vpg, + vpg) of each
// of the image's tpi tiles.  grid (32 groups, N), 256 threads: every thread takes a few partials with INDEPENDENT loads (a
// load -> add chain over all partials would wait for one L2 round trip per addend), then a fixed-order reduction: lanes by shuffle, the eight warps through shared memory.  Deterministic.
constexpr int kFoldThreads = 256;
__global__ void __launch_bounds__(kFoldThreads)
gn_fold_kernel(const float* __restrict__ partials, float* __restrict__ sums, int mode, int G, int tpi, int octs, int oct0, int vpg) {
  __shared__ float2 wsum[kFoldThreads / 32];
  pdl_wait();
  pdl_launch_dependents();
  const int g = blockIdx.x, n = blockIdx.y, t = threadIdx.x;
  const int cnt = mode == 0 ? G : tpi * vpg;
  auto addr = [&](int m) -> const float2* {
    if (mode == 0) return reinterpret_cast<const float2*>(partials + (((int64_t)n * G + m) * 32 + g) * 2);
    const int tile = m / vpg, o = m - tile * vpg;
    return reinterpret_cast<const float2*>(partials + (((int64_t)n * tpi + tile) * octs + oct0 + g * vpg + o) * 2);
  };
  float s = 0.f, q = 0.f;
  int m = t;
  for (; m + 3 * kFoldThreads < cnt; m += 4 * kFoldThreads) {
    const float2 v0 = __ldcg(addr(m)), v1 = __ldcg(addr(m + kFoldThreads)), v2 = __ldcg(addr(m + 2 * kFoldThreads)),
                 v3 = __ldcg(addr(m + 3 * kFoldThreads));
    s += (v0.x + v1.x) + (v2.x + v3.x);
    q += (v0.y + v1.y) + (v2.y + v3.y);
  }
  float2 r[3];
  int nr = 0;
  for (; m < cnt && nr < 3; m += kFoldThreads) r[nr++] = __ldcg(addr(m));
  for (int i = 0; i < nr; ++i) {
    s += r[i].x;
    q += r[i].y;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if ((t & 31) == 0) wsum[t >> 5] = make_float2(s, q);
  __syncthreads();
  if (t == 0) {
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int w = 0; w < kFoldThreads / 32; ++w) {
      a += wsum[w].x;
      b += wsum[w].y;
    }
    sums[((int64_t)n * 32 + g) * 2] = a;
    sums[((int64_t)n * 32 + g) * 2 + 1] = b;
  }
}

// ------------------------------------------------------------------------------------------------ forward
// partial sums of x and x^2 per (CTA, group).  grid (G, N)
__global__ void __launch_bounds__(kGsThreads)
gn_stats_stream_kernel(const __half* __restrict__ x, float* __restrict__ partials, int HW, int C, int64_t ldx) {
  __shared__ float red[2 * kGsThreads];
  const GsMap m(C);
  const int n = blockIdx.y, G = gridDim.x;
  pdl_wait();
  pdl_launch_dependents();
  const __half* xb = x + (int64_t)n * HW * ldx + m.col * 8;
  float2 s[4], q[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) s[j] = q[j] = make_float2(0.f, 0.f);
  auto acc = [&](const uint4& v) {
    float2 f[4];
    gs_unpack(v, f);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      s[j] = add2(s[j], f[j]);
      q[j] = fma2(f[j], f[j], q[j]);
    }
  };
  if (m.active) {  // four independent 16-byte loads in flight per thread: one per trip left the kernel at 3 TB/s (latency-bound)
    const int st = G * m.RP;
    int r = blockIdx.x * m.RP + m.slot;
    for (; r + 3 * st < HW; r += 4 * st) {
      const uint4 v0 = gs_ld(xb + (int64_t)r * ldx), v1 = gs_ld(xb + (int64_t)(r + st) * ldx), v2 = gs_ld(xb + (int64_t)(r + 2 * st) * ldx),
                  v3 = gs_ld(xb + (int64_t)(r + 3 * st) * ldx);
      acc(v0);
      acc(v1);
      acc(v2);
      acc(v3);
    }
    for (; r < HW; r += st) acc(gs_ld(xb + (int64_t)r * ldx));
  }
  const float ts = ((s[0].x + s[0].y) + (s[1].x + s[1].y)) + ((s[2].x + s[2].y) + (s[3].x + s[3].y));
  const float tq = ((q[0].x + q[0].y) + (q[1].x + q[1].y)) + ((q[2].x + q[2].y) + (q[3].x + q[3].y));
  gs_block_partials(m, C / 256, ts, tq, red, partials + ((int64_t)n * G + blockIdx.x) * 64);
}

// y = [silu](x * A + B); the CTA (0, n) also writes stats[n][g] = (mean, rstd) for the backward.  grid (G, N)
__global__ void __launch_bounds__(kGsThreads)
gn_apply_stream_kernel(const __half* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ emb,
                       __half* __restrict__ y, float* __restrict__ stats, const float* __restrict__ sums, int HW, int C, int64_t ldx, int64_t ldy,
                       float eps, int silu) {
  const GsMap m(C);
  const int n = blockIdx.y, G = gridDim.x, vpg = C / 256;
  pdl_wait();
  pdl_launch_dependents();
  const float inv_m = 1.f / ((float)(C / 32) * (float)HW);
  auto group_stats = [&](int g, float& mu, float& rs) {
    const float2 sq = __ldcg(reinterpret_cast<const float2*>(sums + ((int64_t)n * 32 + g) * 2));
    mu = sq.x * inv_m;
    const float var = fmaxf(fmaf(-mu, mu, sq.y * inv_m), 0.f);  // E[x^2] - mean^2 (sums folded in double)
    rs = 1.f / sqrtf(var + eps);
  };
  if (blockIdx.x == 0 && threadIdx.x < 32) {
    float mu, rs;
    group_stats(threadIdx.x, mu, rs);
    stats[((int64_t)n * 32 + threadIdx.x) * 2] = mu;
    stats[((int64_t)n * 32 + threadIdx.x) * 2 + 1] = rs;
  }
  if (!m.active) return;
  float mu, rs;
  group_stats(min(m.col / vpg, 31), mu, rs);
  float2 A[4], B[4], Gn[4];
  gs_coef(n, m.col, C, gamma, beta, emb, mu, rs, A, B, Gn);
  const __half* xb = x + (int64_t)n * HW * ldx + m.col * 8;
  __half* yb = y + (int64_t)n * HW * ldy + m.col * 8;
  auto apply = [&](const uint4& v, int r) {
    float2 f[4];
    gs_unpack(v, f);
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 t = fma2(f[j], A[j], B[j]);
      if (silu) t = silu2(t);
      ow[j] = gs_f2h(t);
    }
    *reinterpret_cast<uint4*>(yb + (int64_t)r * ldy) = o;
  };
  const int st = G * m.RP;
  int r = blockIdx.x * m.RP + m.slot;
  for (; r + 3 * st < HW; r += 4 * st) {
    const uint4 v0 = gs_ld(xb + (int64_t)r * ldx), v1 = gs_ld(xb + (int64_t)(r + st) * ldx), v2 = gs_ld(xb + (int64_t)(r + 2 * st) * ldx),
                v3 = gs_ld(xb + (int64_t)(r + 3 * st) * ldx);
    apply(v0, r);
    apply(v1, r + st);
    apply(v2, r + 2 * st);
    apply(v3, r + 3 * st);
  }
  for (; r < HW; r += st) apply(gs_ld(xb + (int64_t)r * ldx), r);
}

// ------------------------------------------------------------------------------------------------ backward
// v = x * A + B (pre-activation), e = dy * silu'(v), xhat = x * rs - mu * rs; partial sums of e * G and e * G * xhat per (CTA, group)
__global__ void __launch_bounds__(kGsThreads)
gn_bwd_stats_stream_kernel(const __half* __restrict__ dy, const __half* __restrict__ x, const float* __restrict__ stats,
                           const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ emb,
                           float* __restrict__ partials, int HW, int C, int64_t ld_dy, int64_t ldx, int silu) {
  __shared__ float red[2 * kGsThreads];
  const GsMap m(C);
  const int n = blockIdx.y, G = gridDim.x, vpg = C / 256;
  pdl_wait();
  pdl_launch_dependents();
  const int g = min(m.col / vpg, 31);
  const float mu = stats[((int64_t)n * 32 + g) * 2], rs = stats[((int64_t)n * 32 + g) * 2 + 1];
  float2 A[4], B[4], Gn[4];
  gs_coef(n, m.col, C, gamma, beta, emb, mu, rs, A, B, Gn);
  const float2 rs2 = make_float2(rs, rs), nmr2 = make_float2(-mu * rs, -mu * rs);
  const __half* db = dy + (int64_t)n * HW * ld_dy + m.col * 8;
  const __half* xb = x + (int64_t)n * HW * ldx + m.col * 8;
  float2 s[4], q[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) s[j] = q[j] = make_float2(0.f, 0.f);
  auto acc = [&](const uint4& vd, const uint4& vx) {
    float2 d[4], a[4];
    gs_unpack(vd, d);
    gs_unpack(vx, a);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 e = silu ? mul2(d[j], silu_grad2(fma2(a[j], A[j], B[j]))) : d[j];
      const float2 xh = fma2(a[j], rs2, nmr2);
      s[j] = add2(s[j], e);
      q[j] = fma2(e, xh, q[j]);
    }
  };
  if (m.active) {
    const int st = G * m.RP;
    int r = blockIdx.x * m.RP + m.slot;
    for (; r + 2 * st < HW; r += 3 * st) {  // six independent loads in flight
      const uint4 d0 = gs_ld(db + (int64_t)r * ld_dy), x0 = gs_ld(xb + (int64_t)r * ldx);
      const uint4 d1 = gs_ld(db + (int64_t)(r + st) * ld_dy), x1 = gs_ld(xb + (int64_t)(r + st) * ldx);
      const uint4 d2 = gs_ld(db + (int64_t)(r + 2 * st) * ld_dy), x2 = gs_ld(xb + (int64_t)(r + 2 * st) * ldx);
      acc(d0, x0);
      acc(d1, x1);
      acc(d2, x2);
    }
    for (; r < HW; r += st) acc(gs_ld(db + (int64_t)r * ld_dy), gs_ld(xb + (int64_t)r * ldx));
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {  // the channel gains are constant over pixels: applied once
    s[j] = mul2(s[j], Gn[j]);
    q[j] = mul2(q[j], Gn[j]);
  }
  const float ts = ((s[0].x + s[0].y) + (s[1].x + s[1].y)) + ((s[2].x + s[2].y) + (s[3].x + s[3].y));
  const float tq = ((q[0].x + q[0].y) + (q[1].x + q[1].y)) + ((q[2].x + q[2].y) + (q[3].x + q[3].y));
  gs_block_partials(m, vpg, ts, tq, red, partials + ((int64_t)n * G + blockIdx.x) * 64);
}

// dx (=|+=) rs * (e * G - m1 - xhat * m2) = e * A + x * k1 + k0 with m1 = mean(e G), m2 = mean(e G xhat) of the group
__global__ void __launch_bounds__(kGsThreads)
gn_bwd_apply_stream_kernel(const __half* __restrict__ dy, const __half* __restrict__ x, const float* __restrict__ stats,
                           const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ emb,
                           __half* __restrict__ dx, const float* __restrict__ sums, int HW, int C, int64_t ld_dy, int64_t ldx, int64_t ld_dx,
                           int silu, int accumulate) {
  const GsMap m(C);
  const int n = blockIdx.y, G = gridDim.x, vpg = C / 256;
  pdl_wait();
  pdl_launch_dependents();
  if (!m.active) return;
  const int g = min(m.col / vpg, 31);
  const float mu = stats[((int64_t)n * 32 + g) * 2], rs = stats[((int64_t)n * 32 + g) * 2 + 1];
  float2 A[4], B[4], Gn[4];
  gs_coef(n, m.col, C, gamma, beta, emb, mu, rs, A, B, Gn);
  const float2 sq = __ldcg(reinterpret_cast<const float2*>(sums + ((int64_t)n * 32 + g) * 2));
  const float inv_m = 1.f / ((float)(C / 32) * (float)HW);
  const float m1 = sq.x * inv_m, m2 = sq.y * inv_m;
  const float2 k1 = make_float2(-rs * rs * m2, -rs * rs * m2);
  const float k0s = -rs * m1 + mu * rs * rs * m2;
  const float2 k0 = make_float2(k0s, k0s);
  const __half* db = dy + (int64_t)n * HW * ld_dy + m.col * 8;
  const __half* xb = x + (int64_t)n * HW * ldx + m.col * 8;
  __half* ob = dx + (int64_t)n * HW * ld_dx + m.col * 8;
  auto apply = [&](const uint4& vd, const uint4& vx, uint4 o, int r) {
    float2 d[4], a[4];
    gs_unpack(vd, d);
    gs_unpack(vx, a);
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 e = silu ? mul2(d[j], silu_grad2(fma2(a[j], A[j], B[j]))) : d[j];
      float2 v = fma2(e, A[j], fma2(a[j], k1, k0));  // e * G * rs + x * k1 + k0
      if (accumulate) v = add2(v, gs_h2f(ow[j]));
      ow[j] = gs_f2h(v);
    }
    *reinterpret_cast<uint4*>(ob + (int64_t)r * ld_dx) = o;
  };
  const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
  auto ld_acc = [&](int r) { return accumulate ? *reinterpret_cast<const uint4*>(ob + (int64_t)r * ld_dx) : zero; };
  const int st = G * m.RP;
  int r = blockIdx.x * m.RP + m.slot;
  for (; r + st < HW; r += 2 * st) {  // four to six independent loads in flight
    const uint4 d0 = gs_ld(db + (int64_t)r * ld_dy), x0 = gs_ld(xb + (int64_t)r * ldx), o0 = ld_acc(r);
    const uint4 d1 = gs_ld(db + (int64_t)(r + st) * ld_dy), x1 = gs_ld(xb + (int64_t)(r + st) * ldx), o1 = ld_acc(r + st);
    apply(d0, x0, o0, r);
    apply(d1, x1, o1, r + st);
  }
  for (; r < HW; r += st) apply(gs_ld(db + (int64_t)r * ld_dy), gs_ld(xb + (int64_t)r * ldx), ld_acc(r), r);
}

// ------------------------------------------------------------------------------------------------ host
bool gn_stream_supports(int64_t C) { return C % 256 == 0 && C <= 2048; }

static inline int gs_ctas(int64_t N, int64_t HW, int64_t C) {  // CTAs per image: fill the machine, at least two passes of rows per CTA
  const int64_t RP = kGsThreads / (C / 8);
  int64_t g = std::min<int64_t>(kGsMaxCtas / N, ceil_div(HW, 2 * RP));
  return (int)std::max<int64_t>(1, g);
}

// ops GN_FWD_GRID (p6 partials sized >= N * gs_ctas * 64 floats; p7 barrier words: [0..63] reused here as the folded sums? no:
// the folded sums live in the TAIL of the partials buffer: floats [N * G * 64, + N * 64))
int launch_gn_fwd_stream(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], HW = op.i[1], C = op.i[2], ldx = op.i[3], ldy = op.i[4];
  const int G = gs_ctas(N, HW, C);
  float* partials = (float*)op.p[6];
  float* sums = partials + (int64_t)N * G * 64;
  CGD_CUDA(launch_pdl(gn_stats_stream_kernel, dim3(G, (unsigned)N), dim3(kGsThreads), 0, st, (const __half*)op.p[0], partials, (int)HW, (int)C, ldx));
  CGD_CUDA(launch_pdl(gn_fold_kernel, dim3(32, (unsigned)N), dim3(kFoldThreads), 0, st, (const float*)partials, sums, 0, G, 0, 0, 0, (int)(C / 256)));
  CGD_CUDA(launch_pdl(gn_apply_stream_kernel, dim3(G, (unsigned)N), dim3(kGsThreads), 0, st, (const __half*)op.p[0], (const float*)op.p[1],
                      (const float*)op.p[2], (const float*)op.p[3], (__half*)op.p[4], (float*)op.p[5], (const float*)sums, (int)HW, (int)C, ldx, ldy,
                      op.f[0], (int)(op.flags & 1)));
  CGD_LAUNCH_CHECK();
  return 0;
}

int launch_gn_bwd_stream(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], HW = op.i[1], C = op.i[2], ld_dy = op.i[3], ldx = op.i[4], ld_dx = op.i[5];
  const int G = gs_ctas(N, HW, C);
  float* partials = (float*)op.p[7];
  float* sums = partials + (int64_t)N * G * 64;
  const int silu = (int)(op.flags & 1), acc = (op.flags & 2) ? 1 : 0;
  CGD_CUDA(launch_pdl(gn_bwd_stats_stream_kernel, dim3(G, (unsigned)N), dim3(kGsThreads), 0, st, (const __half*)op.p[0], (const __half*)op.p[1],
                      (const float*)op.p[2], (const float*)op.p[3], (const float*)op.p[4], (const float*)op.p[5], partials, (int)HW, (int)C, ld_dy, ldx,
                      silu));
  CGD_CUDA(launch_pdl(gn_fold_kernel, dim3(32, (unsigned)N), dim3(kFoldThreads), 0, st, (const float*)partials, sums, 0, G, 0, 0, 0, (int)(C / 256)));
  CGD_CUDA(launch_pdl(gn_bwd_apply_stream_kernel, dim3(G, (unsigned)N), dim3(kGsThreads), 0, st, (const __half*)op.p[0], (const __half*)op.p[1],
                      (const float*)op.p[2], (const float*)op.p[3], (const float*)op.p[4], (const float*)op.p[5], (__half*)op.p[6], (const float*)sums,
                      (int)HW, (int)C, ld_dy, ldx, ld_dx, silu, acc));
  CGD_LAUNCH_CHECK();
  return 0;
}

// op GN_APPLY_EPI: conv-epilogue partials -> fold -> one streaming apply trip.  The folded sums go to the stats buffer's neighbour:
// p5 stats is [N][32][2]; the op's scratch for the sums is p7 (f [N * 64]) when given, else the tail of the partials cannot be
// used (owned by the conv) -- plan.py passes p7.
int launch_gn_apply_epi_stream(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], HW = op.i[1], C = op.i[2], ldx = op.i[3], ldy = op.i[4], octs = op.i[6], oct0 = op.i[7];
  CGD_CHECK_ARG(op.p[7] != nullptr, "gn_apply_epi (stream engine): p7 (scratch for the folded sums, N * 64 floats) missing");
  const int G = gs_ctas(N, HW, C);
  float* sums = (float*)op.p[7];
  CGD_CUDA(launch_pdl(gn_fold_kernel, dim3(32, (unsigned)N), dim3(kFoldThreads), 0, st, (const float*)op.p[6], sums, 1, 0, (int)(HW / 128), (int)octs, (int)oct0,
                      (int)(C / 256)));
  CGD_CUDA(launch_pdl(gn_apply_stream_kernel, dim3(G, (unsigned)N), dim3(kGsThreads), 0, st, (const __half*)op.p[0], (const float*)op.p[1],
                      (const float*)op.p[2], (const float*)op.p[3], (__half*)op.p[4], (float*)op.p[5], (const float*)sums, (int)HW, (int)C, ldx, ldy,
                      op.f[0], (int)(op.flags & 1)));
  CGD_LAUNCH_CHECK();
  return 0;
}

int gn_stream_partial_floats(int64_t N, int64_t HW, int64_t C) { return (int)(N * gs_ctas(N, HW, C) * 64 + N * 64); }

}  // namespace cgd
