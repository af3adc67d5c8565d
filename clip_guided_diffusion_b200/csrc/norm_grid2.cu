// norm_grid2.cu -- GroupNorm(32) (+SiLU, +scale/shift) forward and input-gradient for LARGE activations, second version of
// the single persistent launch of norm_grid.cu: same contract (ops GN_FWD_GRID / GN_BWD_GRID, same partials / barrier / stats
// buffers), different engine.
//
// Why: the ring kernel's consumers are a latency-bound instruction stream, not a memory-bound one: one 16-byte vector per loop trip with a serial
// HADD2 -> FFMA -> FMUL -> MUFU.EX2 -> FADD -> MUFU.RCP -> FMUL -> F2FP -> STG chain (85 SASS instructions per vector in
// the apply trip), generic-address LD from the shared-memory ring, mbarrier spin loops in every consumer warp.
// Here: 1024 threads per SM (32 warps) read global memory directly (the second trip finds much of the 8 - 67 MB tensor in the 50 MB L2), every thread owns ONE 8-channel column for the whole kernel, so the per-channel
// coefficients live in registers, and U vectors are in flight per thread per trip (U x 16 KB per SM).
// Requires C % 256 == 0 (a thread's 8 channels never straddle a group); other widths keep the ring kernels.
//
// Replaces [3P] guided-diffusion GroupNorm32 + SiLU + scale-shift and their autograd (SURVEY.md K5, K6).
#include "common.cuh"
#include "ops.cuh"
#include "pdl.cuh"

namespace cgd {

constexpr int kG2Threads = 1024;

__device__ __forceinline__ uint4 g2_ld(const __half* p) {
  uint4 v;
  asm volatile("ld.global.nc.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ float2 g2_h2f(uint32_t w) { return __half22float2(*reinterpret_cast<const __half2*>(&w)); }
__device__ __forceinline__ uint32_t g2_f2h(float2 f) {
  const __half2 h = __floats2half2_rn(f.x, f.y);
  return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ void g2_unpack(const uint4& v, float2 (&f)[4]) {
  f[0] = g2_h2f(v.x);
  f[1] = g2_h2f(v.y);
  f[2] = g2_h2f(v.z);
  f[3] = g2_h2f(v.w);
}

__device__ __forceinline__ void g2_grid_barrier(unsigned int* bar, unsigned int nblocks) {
  __syncthreads();  // every thread's partial-sum stores precede thread 0's release (cumulativity through the barrier)
  if (threadIdx.x == 0) global_barrier_arrive_wait(bar, nblocks);
  __syncthreads();
}

// one value pair per thread -> 32 group sums of this CTA (fixed order).  Thread (col, pl) belongs to group col / vpg; warp w
// gathers group w: its PP * vpg members, one or two per lane, then five shuffles.
__device__ __forceinline__ void g2_block_reduce(float ts, float tq, int V, int PP, int vpg, bool active, float* red_s, float* red_q,
                                                float* gs, float* gq) {
  red_s[threadIdx.x] = active ? ts : 0.f;
  red_q[threadIdx.x] = active ? tq : 0.f;
  __syncthreads();
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float as = 0.f, aq = 0.f;
  const int count = PP * vpg;
  for (int m = lane; m < count; m += 32) {
    const int pl = m / vpg, c = w * vpg + (m - pl * vpg);
    as += red_s[pl * V + c];
    aq += red_q[pl * V + c];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    as += __shfl_xor_sync(0xffffffffu, as, o);
    aq += __shfl_xor_sync(0xffffffffu, aq, o);
  }
  if (lane == 0) {
    gs[w] = as;
    gq[w] = aq;
  }
  __syncthreads();
}

// Fold the Gn per-CTA partials of image n (layout [Gn][32][2]) in a fixed order: warp g takes group g, lane j takes CTAs
// j, j + 32, ... with Neumaier-compensated fp32 sums, then five shuffles: bit-identical in every CTA.
__device__ __forceinline__ void g2_fold(const float* part_n, int Gn, float* out_a, float* out_b) {
  const int g = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float sa = 0.f, ca = 0.f, sb = 0.f, cb = 0.f;
  for (int j = lane; j < Gn; j += 32) {
    const float2 v = __ldcg(reinterpret_cast<const float2*>(part_n + ((int64_t)j * 32 + g) * 2));
    float t = sa + v.x;
    ca += fabsf(sa) >= fabsf(v.x) ? (sa - t) + v.x : (v.x - t) + sa;
    sa = t;
    t = sb + v.y;
    cb += fabsf(sb) >= fabsf(v.y) ? (sb - t) + v.y : (v.y - t) + sb;
    sb = t;
  }
  float da = sa + ca, db = sb + cb;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    da += __shfl_xor_sync(0xffffffffu, da, o);
    db += __shfl_xor_sync(0xffffffffu, db, o);
  }
  if (lane == 0) {
    out_a[g] = da;
    out_b[g] = db;
  }
  __syncthreads();
}

// f(pixel, slot) over this thread's pixels p0 + pl, p0 + pl + PP, ...: U of them per trip so U loads are in flight
template <int U, typename L, typename F>
__device__ __forceinline__ void g2_sweep(int p0, int p1, int pl, int PP, L&& load, F&& f) {
  int p = p0 + pl;
  for (; p + (U - 1) * PP < p1; p += U * PP) {
#pragma unroll
    for (int u = 0; u < U; ++u) load(p + u * PP, u);
#pragma unroll
    for (int u = 0; u < U; ++u) f(p + u * PP, u);
  }
  for (; p < p1; p += PP) {
    load(p, 0);
    f(p, 0);
  }
}

// ------------------------------------------------------------------------------------------------ forward
template <int U>
__global__ void __launch_bounds__(kG2Threads, 1)
gn_fwd_grid2_kernel(const __half* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                    const float* __restrict__ emb, __half* __restrict__ y, float* __restrict__ stats, float* __restrict__ partials,
                    unsigned int* __restrict__ bar, int HW, int C, int64_t ldx, int64_t ldy, int Gn, float eps, int silu) {
  __shared__ float red_s[kG2Threads], red_q[kG2Threads];
  __shared__ float gs[32], gq[32], fa[32], fb[32], s_mean[32], s_rstd[32];
  const int n = blockIdx.x / Gn, chunk = blockIdx.x % Gn;
  const int V = C / 8, PP = kG2Threads / V, cpg = C / 32, vpg = cpg / 8;
  const int ppc = (HW + Gn - 1) / Gn;
  const int p0 = min(HW, chunk * ppc), p1 = min(HW, p0 + ppc);
  const int col = threadIdx.x % V, pl = threadIdx.x / V;
  const bool active = pl < PP;
  const int pend = active ? p1 : p0;  // idle threads (1024 % V != 0) sweep an empty range
  pdl_wait();
  pdl_launch_dependents();
  const __half* xb = x + (int64_t)n * HW * ldx + col * 8;
  uint4 v[U];
  float2 s[4], q[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) s[j] = q[j] = make_float2(0.f, 0.f);
  g2_sweep<U>(
      p0, pend, pl, PP, [&](int p, int u) { v[u] = g2_ld(xb + (int64_t)p * ldx); },
      [&](int, int u) {
        float2 f[4];
        g2_unpack(v[u], f);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          s[j] = add2(s[j], f[j]);
          q[j] = fma2(f[j], f[j], q[j]);
        }
      });
  const float ts = ((s[0].x + s[0].y) + (s[1].x + s[1].y)) + ((s[2].x + s[2].y) + (s[3].x + s[3].y));
  const float tq = ((q[0].x + q[0].y) + (q[1].x + q[1].y)) + ((q[2].x + q[2].y) + (q[3].x + q[3].y));
  g2_block_reduce(ts, tq, V, PP, vpg, active, red_s, red_q, gs, gq);
  if (threadIdx.x < 32) {
    float* o = partials + (((int64_t)n * Gn + chunk) * 32 + threadIdx.x) * 2;
    o[0] = gs[threadIdx.x];
    o[1] = gq[threadIdx.x];
  }
  g2_grid_barrier(bar, gridDim.x);
  g2_fold(partials + (int64_t)n * Gn * 64, Gn, fa, fb);
  if (threadIdx.x < 32) {
    const float inv_m = 1.f / ((float)cpg * (float)HW);
    const float mu = fa[threadIdx.x] * inv_m;
    const float var = fmaxf(fmaf(-mu, mu, fb[threadIdx.x] * inv_m), 0.f);  // E[x^2] - mean^2: relative error ~ 6e-8 * mean^2 / var
    const float rs = 1.f / sqrtf(var + eps);
    s_mean[threadIdx.x] = mu;
    s_rstd[threadIdx.x] = rs;
    if (chunk == 0) {
      stats[((int64_t)n * 32 + threadIdx.x) * 2 + 0] = mu;
      stats[((int64_t)n * 32 + threadIdx.x) * 2 + 1] = rs;
    }
  }
  __syncthreads();
  float2 A[4], Bc[4];
  {
    const int g = min(col / vpg, 31);
    const float mu = s_mean[g], rs = s_rstd[g];
    float a[8], b[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = col * 8 + j;
      const float ga = gamma[c], be = beta[c];
      float sc1 = 1.f, sh = 0.f;
      if (emb) {
        sc1 = 1.f + emb[(int64_t)n * 2 * C + c];
        sh = emb[(int64_t)n * 2 * C + C + c];
      }
      a[j] = rs * ga * sc1;
      b[j] = (be - mu * rs * ga) * sc1 + sh;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      A[j] = make_float2(a[2 * j], a[2 * j + 1]);
      Bc[j] = make_float2(b[2 * j], b[2 * j + 1]);
    }
  }
  __half* yb = y + (int64_t)n * HW * ldy + col * 8;
  g2_sweep<U>(
      p0, pend, pl, PP, [&](int p, int u) { v[u] = g2_ld(xb + (int64_t)p * ldx); },
      [&](int p, int u) {
        float2 f[4];
        g2_unpack(v[u], f);
        uint4 o;
        uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float2 t = fma2(f[j], A[j], Bc[j]);
          if (silu) t = silu2(t);
          ow[j] = g2_f2h(t);
        }
        *reinterpret_cast<uint4*>(yb + (int64_t)p * ldy) = o;
      });
}

// ------------------------------------------------------------------------------------------------ forward from conv-epilogue statistics
// GN_APPLY_EPI: the conv that produced x already reduced it to per (128-pixel tile, 8-channel octet) sums (CONV flags 2,
// conv_tc.cu, CONV flags 2), so the forward is ONE streaming trip: every CTA folds the partial sums of its image (warp g = group g, fixed
// order, compensated fp32 -- bit-identical in every CTA, no grid barrier), then applies.  partials: [N * tpi][octs][2], tpi = HW / 128.
template <int U>
__global__ void __launch_bounds__(kG2Threads, 1)
gn_apply_epi_kernel(const __half* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ emb,
                    __half* __restrict__ y, float* __restrict__ stats, const float* __restrict__ partials, int HW, int C, int64_t ldx, int64_t ldy,
                    int Gn, int octs, int oct0, float eps, int silu) {
  __shared__ float s_mean[32], s_rstd[32];
  const int n = blockIdx.x / Gn, chunk = blockIdx.x % Gn;
  const int V = C / 8, PP = kG2Threads / V, cpg = C / 32, vpg = cpg / 8;
  const int ppc = (HW + Gn - 1) / Gn;
  const int p0 = min(HW, chunk * ppc), p1 = min(HW, p0 + ppc);
  const int col = threadIdx.x % V, pl = threadIdx.x / V;
  const bool active = pl < PP;
  const int pend = active ? p1 : p0;
  pdl_wait();
  pdl_launch_dependents();
  {
    const int g = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tpi = HW / 128, cnt = tpi * vpg;  // group g: octets [oct0 + g * vpg, + vpg) of every tile of image n
    float sa = 0.f, ca = 0.f, sb = 0.f, cb = 0.f;
    for (int m = lane; m < cnt; m += 32) {
      const int tile = m / vpg, o = m - tile * vpg;
      const float2 v = __ldcg(reinterpret_cast<const float2*>(partials + (((int64_t)n * tpi + tile) * octs + oct0 + g * vpg + o) * 2));
      float t = sa + v.x;
      ca += fabsf(sa) >= fabsf(v.x) ? (sa - t) + v.x : (v.x - t) + sa;
      sa = t;
      t = sb + v.y;
      cb += fabsf(sb) >= fabsf(v.y) ? (sb - t) + v.y : (v.y - t) + sb;
      sb = t;
    }
    float da = sa + ca, db = sb + cb;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      da += __shfl_xor_sync(0xffffffffu, da, o);
      db += __shfl_xor_sync(0xffffffffu, db, o);
    }
    if (lane == 0) {
      const float inv_m = 1.f / ((float)cpg * (float)HW);
      const float mu = da * inv_m;
      const float var = fmaxf(fmaf(-mu, mu, db * inv_m), 0.f);
      const float rs = 1.f / sqrtf(var + eps);
      s_mean[g] = mu;
      s_rstd[g] = rs;
      if (chunk == 0) {
        stats[((int64_t)n * 32 + g) * 2 + 0] = mu;
        stats[((int64_t)n * 32 + g) * 2 + 1] = rs;
      }
    }
  }
  __syncthreads();
  float2 A[4], Bc[4];
  {
    const int g = min(col / vpg, 31);
    const float mu = s_mean[g], rs = s_rstd[g];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float a[2], b[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = col * 8 + 2 * j + h;
        const float ga = gamma[c], be = beta[c];
        const float sc1 = emb ? 1.f + emb[(int64_t)n * 2 * C + c] : 1.f, sh = emb ? emb[(int64_t)n * 2 * C + C + c] : 0.f;
        a[h] = rs * ga * sc1;
        b[h] = (be - mu * rs * ga) * sc1 + sh;
      }
      A[j] = make_float2(a[0], a[1]);
      Bc[j] = make_float2(b[0], b[1]);
    }
  }
  const __half* xb = x + (int64_t)n * HW * ldx + col * 8;
  __half* yb = y + (int64_t)n * HW * ldy + col * 8;
  uint4 v[U];
  g2_sweep<U>(
      p0, pend, pl, PP, [&](int p, int u) { v[u] = g2_ld(xb + (int64_t)p * ldx); },
      [&](int p, int u) {
        float2 f[4];
        g2_unpack(v[u], f);
        uint4 o;
        uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float2 t = fma2(f[j], A[j], Bc[j]);
          if (silu) t = silu2(t);
          ow[j] = g2_f2h(t);
        }
        *reinterpret_cast<uint4*>(yb + (int64_t)p * ldy) = o;
      });
}

// ------------------------------------------------------------------------------------------------ backward
template <int U>
__global__ void __launch_bounds__(kG2Threads, 1)
gn_bwd_grid2_kernel(const __half* __restrict__ dy, const __half* __restrict__ x, const float* __restrict__ stats,
                    const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ emb,
                    __half* __restrict__ dx, float* __restrict__ partials, unsigned int* __restrict__ bar, int HW, int C, int64_t ld_dy,
                    int64_t ldx, int64_t ld_dx, int Gn, int silu, int accumulate) {
  __shared__ float red_s[kG2Threads], red_q[kG2Threads];
  __shared__ float gs[32], gq[32], fa[32], fb[32];
  const int n = blockIdx.x / Gn, chunk = blockIdx.x % Gn;
  const int V = C / 8, PP = kG2Threads / V, cpg = C / 32, vpg = cpg / 8;
  const int ppc = (HW + Gn - 1) / Gn;
  const int p0 = min(HW, chunk * ppc), p1 = min(HW, p0 + ppc);
  const int col = threadIdx.x % V, pl = threadIdx.x / V;
  const bool active = pl < PP;
  const int pend = active ? p1 : p0;
  pdl_wait();
  pdl_launch_dependents();
  // v = x * RG + Bc (the pre-activation), xhat = x * rs + nmr, e = dy * silu'(v), d xhat = e * G (G = gamma * (1 + scale))
  const int g = min(col / vpg, 31);
  const float mu = stats[((int64_t)n * 32 + g) * 2], rs = stats[((int64_t)n * 32 + g) * 2 + 1];
  const float2 rs2 = make_float2(rs, rs), nmr2 = make_float2(-mu * rs, -mu * rs);
  auto gain = [&](int c) { return gamma[c] * (emb ? 1.f + emb[(int64_t)n * 2 * C + c] : 1.f); };
  float2 RG[4], Bc[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float a[2], b[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = col * 8 + 2 * j + h;
      const float sc1 = emb ? 1.f + emb[(int64_t)n * 2 * C + c] : 1.f, sh = emb ? emb[(int64_t)n * 2 * C + C + c] : 0.f;
      a[h] = rs * gamma[c] * sc1;
      b[h] = (beta[c] - mu * rs * gamma[c]) * sc1 + sh;
    }
    RG[j] = make_float2(a[0], a[1]);
    Bc[j] = make_float2(b[0], b[1]);
  }
  const __half* db = dy + (int64_t)n * HW * ld_dy + col * 8;
  const __half* xb = x + (int64_t)n * HW * ldx + col * 8;
  uint4 vd[U], vx[U];
  auto load = [&](int p, int u) {
    vd[u] = g2_ld(db + (int64_t)p * ld_dy);
    vx[u] = g2_ld(xb + (int64_t)p * ldx);
  };
  auto egrad = [&](float2 d, float2 a, int j) { return silu ? mul2(d, silu_grad2(fma2(a, RG[j], Bc[j]))) : d; };
  // per-channel sums of e and e * xhat; the channel gains are applied once at the end (they are constant over pixels)
  float2 s[4], q[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) s[j] = q[j] = make_float2(0.f, 0.f);
  g2_sweep<U>(p0, pend, pl, PP, load, [&](int, int u) {
    float2 d[4], a[4];
    g2_unpack(vd[u], d);
    g2_unpack(vx[u], a);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 e = egrad(d[j], a[j], j);
      const float2 xh = fma2(a[j], rs2, nmr2);
      s[j] = add2(s[j], e);
      q[j] = fma2(e, xh, q[j]);
    }
  });
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 G = make_float2(gain(col * 8 + 2 * j), gain(col * 8 + 2 * j + 1));
    s[j] = mul2(s[j], G);
    q[j] = mul2(q[j], G);
  }
  const float ts = ((s[0].x + s[0].y) + (s[1].x + s[1].y)) + ((s[2].x + s[2].y) + (s[3].x + s[3].y));
  const float tq = ((q[0].x + q[0].y) + (q[1].x + q[1].y)) + ((q[2].x + q[2].y) + (q[3].x + q[3].y));
  g2_block_reduce(ts, tq, V, PP, vpg, active, red_s, red_q, gs, gq);
  if (threadIdx.x < 32) {
    float* o = partials + (((int64_t)n * Gn + chunk) * 32 + threadIdx.x) * 2;
    o[0] = gs[threadIdx.x];
    o[1] = gq[threadIdx.x];
  }
  g2_grid_barrier(bar, gridDim.x);
  g2_fold(partials + (int64_t)n * Gn * 64, Gn, fa, fb);
  const float inv_m = 1.f / ((float)cpg * (float)HW);
  const float m1 = fa[g] * inv_m, m2 = fb[g] * inv_m;  // mean(d xhat), mean(d xhat * xhat)
  // dx = rs * (d xhat - m1 - xhat * m2) = d xhat * rs + x * k1 + k0
  const float2 k1 = make_float2(-rs * rs * m2, -rs * rs * m2);
  const float k0s = -rs * m1 + mu * rs * rs * m2;
  const float2 k0 = make_float2(k0s, k0s);
  __half* ob = dx + (int64_t)n * HW * ld_dx + col * 8;
  g2_sweep<U>(p0, pend, pl, PP, load, [&](int p, int u) {
    float2 d[4], a[4];
    g2_unpack(vd[u], d);
    g2_unpack(vx[u], a);
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
    if (accumulate) o = *reinterpret_cast<const uint4*>(ob + (int64_t)p * ld_dx);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 r = fma2(egrad(d[j], a[j], j), RG[j], fma2(a[j], k1, k0));  // e * G * rs + x * k1 + k0
      if (accumulate) r = add2(r, g2_h2f(ow[j]));
      ow[j] = g2_f2h(r);
    }
    *reinterpret_cast<uint4*>(ob + (int64_t)p * ld_dx) = o;
  });
}

// ------------------------------------------------------------------------------------------------ host
constexpr int kG2FwdU = 4, kG2BwdU = 2;

bool gn_grid2_supports(int64_t C) { return C % 256 == 0 && C <= 2048; }

int launch_gn_apply_epi_stream(const CgdOp& op, cudaStream_t st);  // norm_stream.cu: fold launch + streaming apply launch
static bool epi_use_stream(const CgdOp& op) {
  static int off = -1;
  if (off < 0) {
    const char* e = getenv("CGD_GN_GRID_ENGINE");
    off = (e && e[0] == 's') ? 0 : 1;  // streaming engine opt-in
  }
  return !off && op.p[7] != nullptr;
}
int gn_apply_epi_num_launches(const CgdOp& op) { return epi_use_stream(op) ? 2 : 1; }

int launch_gn_apply_epi(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], HW = op.i[1], C = op.i[2], ldx = op.i[3], ldy = op.i[4], Gn = op.i[5], octs = op.i[6], oct0 = op.i[7];
  CGD_CHECK_ARG(N > 0 && HW > 0 && HW % 128 == 0 && gn_grid2_supports(C) && Gn >= 1 && ldx % 8 == 0 && ldy % 8 == 0 && octs >= oct0 + C / 8 && oct0 >= 0,
                "gn_apply_epi: bad dims (HW %% 128, C %% 256, octets)");
  CGD_CHECK_ARG(op.p[0] && op.p[1] && op.p[2] && op.p[4] && op.p[5] && op.p[6], "gn_apply_epi: null pointer");
  if (epi_use_stream(op)) return launch_gn_apply_epi_stream(op, st);
  CGD_CUDA(launch_pdl(gn_apply_epi_kernel<kG2FwdU>, dim3((unsigned)(N * Gn)), dim3(kG2Threads), 0, st, (const __half*)op.p[0], (const float*)op.p[1],
                      (const float*)op.p[2], (const float*)op.p[3], (__half*)op.p[4], (float*)op.p[5], (const float*)op.p[6], (int)HW, (int)C, ldx, ldy,
                      (int)Gn, (int)octs, (int)oct0, op.f[0], (int)(op.flags & 1)));
  return 0;
}

int launch_gn_fwd_grid2(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], HW = op.i[1], C = op.i[2], ldx = op.i[3], ldy = op.i[4], Gn = op.i[5];
  static DeviceOnce checked;
  if (checked.needed()) {
    int occ = 0;
    CGD_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gn_fwd_grid2_kernel<kG2FwdU>, kG2Threads, 0));
    CGD_CHECK_ARG(occ >= 1, "gn_fwd_grid2: the 1024-thread CTA does not fit an SM (occupancy %d)", occ);
    checked.mark();
  }
  CGD_CUDA(launch_pdl(gn_fwd_grid2_kernel<kG2FwdU>, dim3((unsigned)(N * Gn)), dim3(kG2Threads), 0, st, (const __half*)op.p[0],
                      (const float*)op.p[1], (const float*)op.p[2], (const float*)op.p[3], (__half*)op.p[4], (float*)op.p[5], (float*)op.p[6],
                      (unsigned int*)op.p[7], (int)HW, (int)C, ldx, ldy, (int)Gn, op.f[0], (int)(op.flags & 1)));
  return 0;
}

int launch_gn_bwd_grid2(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], HW = op.i[1], C = op.i[2], ld_dy = op.i[3], ldx = op.i[4], ld_dx = op.i[5], Gn = op.i[6];
  static DeviceOnce checked;
  if (checked.needed()) {
    int occ = 0;
    CGD_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gn_bwd_grid2_kernel<kG2BwdU>, kG2Threads, 0));
    CGD_CHECK_ARG(occ >= 1, "gn_bwd_grid2: the 1024-thread CTA does not fit an SM (occupancy %d)", occ);
    checked.mark();
  }
  CGD_CUDA(launch_pdl(gn_bwd_grid2_kernel<kG2BwdU>, dim3((unsigned)(N * Gn)), dim3(kG2Threads), 0, st, (const __half*)op.p[0],
                      (const __half*)op.p[1], (const float*)op.p[2], (const float*)op.p[3], (const float*)op.p[4], (const float*)op.p[5],
                      (__half*)op.p[6], (float*)op.p[7], (unsigned int*)op.p[8], (int)HW, (int)C, ld_dy, ldx, ld_dx, (int)Gn,
                      (int)(op.flags & 1), (int)((op.flags & 2) ? 1 : 0)));
  return 0;
}

}  // namespace cgd
