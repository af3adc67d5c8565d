// norm_grid.cu -- GroupNorm(32) (+SiLU, +scale/shift) forward and input-gradient for LARGE activations as ONE persistent
// launch: statistics pass, grid-wide barrier, apply pass, both passes fed by a bulk-async-copy (TMA) ring.
//
// Why: at the 128x128 / 256x256 levels the two-launch kernels of
// norm.cu keep too few bytes in flight (two blocks of 256 threads per SM), their grids end in half-empty waves and the second
// launch waits for a last-block fold; a single-launch version whose threads load a few 16-byte vectors each is bounded by the
// registers that hold the bytes in flight.  Here one CTA per SM owns a
// contiguous pixel range of one image across ALL channels; a producer warp streams it through an 8-stage shared-memory
// ring with cp.async.bulk (16 KB per stage, 128 KB in flight per SM, independent of the consumers'
// registers); 512 consumer threads reduce each stage from shared memory, write per-group partial sums, meet the other CTAs
// at a generation-counted grid barrier (every CTA is resident: grid <= SM count, one CTA per SM), fold the partials
// themselves (fixed order, compensated fp32: bit-identical in every CTA) and normalise the same pixel range from a second trip through
// the ring, whose loads are largely L2 hits (the tensors are 8 - 67 MB, the L2 is 50 MB) and start while the barrier is still
// being crossed.  HBM traffic: x once + y once (forward), dy + x once + dx (backward).
//
// The large backward launches of widths C % 256 == 0 run on the direct-load kernel of norm_grid2.cu instead (gn_bwd_direct below).
//
// Replaces [3P] guided-diffusion GroupNorm32 + SiLU + scale-shift and their autograd (SURVEY.md K5, K6).
#include "common.cuh"
#include "ops.cuh"
#include "pdl.cuh"
#include "tc_ptx.cuh"

namespace cgd {

constexpr int kGngConsumers = 512;             // warps 0..15
constexpr int kGngThreads = kGngConsumers + 32; // + producer warp 16
constexpr int kGngStages = 8;                  // x 16 KB = 128 KB of bulk copies in flight per SM
constexpr int kGngStageBytes = 16384;          // upper bound; the used part is NT * R * C * 2
constexpr int kGngBarId = 1;                   // named barrier of the consumer threads

__device__ __forceinline__ void gng_sync() { named_bar_sync(kGngBarId, kGngConsumers); }

// Generation-counted barrier over all CTAs of the grid (consumer threads only).  bar[0] = arrival count (returns to 0),
// bar[1] = generation (only ever incremented), so the buffer needs no reset between launches or CUDA-graph replays.
__device__ __forceinline__ void grid_barrier(unsigned int* bar, unsigned int nblocks) {
  gng_sync();  // every consumer's partial-sum stores precede thread 0's release below (cumulativity through the barrier)
  if (threadIdx.x == 0) global_barrier_arrive_wait(bar, nblocks);
  gng_sync();
}

// 8 channel sums per thread -> 32 group sums of this CTA.  Shared layout [pixel lane][channel]; thread (g = t/16, part = t%16)
// adds elements part, part+16, ... of group g's PP * cpg values, then the 16 parts are folded by shuffles (fixed order).
__device__ __forceinline__ void gng_block_reduce(const float* s, const float* q, int C, int col, int pl, int PP, bool active,
                                                 float* red_s, float* red_q, float* gs, float* gq) {
  gng_sync();
  if (active) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      red_s[pl * C + col * 8 + j] = s[j];
      red_q[pl * C + col * 8 + j] = q[j];
    }
  }
  gng_sync();
  const int cpg = C / 32, g = threadIdx.x >> 4, part = threadIdx.x & 15;
  float as = 0.f, aq = 0.f;
  const int n = PP * cpg;
  for (int e = part; e < n; e += 16) {
    const int l = e / cpg, c = e - l * cpg;
    as += red_s[l * C + g * cpg + c];
    aq += red_q[l * C + g * cpg + c];
  }
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) {
    as += __shfl_xor_sync(0xffffffffu, as, o);
    aq += __shfl_xor_sync(0xffffffffu, aq, o);
  }
  if (part == 0) {
    gs[g] = as;
    gq[g] = aq;
  }
  gng_sync();
}

// Fold the Gn per-CTA partials of image n (layout [Gn][32][2]) in a fixed order: thread (g, part) takes CTAs part, part+16, ...
// with Neumaier-compensated fp32 sums (exact to ~1 ulp for <= 10 terms), the 16 parts are folded by shuffles.  No fp64: the
// F2F.F64 / DADD sequence of a double-precision fold stalls on the narrow fp64 pipe for a reduction of one number per SM.  Results for all 32 groups land in shared memory.
__device__ __forceinline__ void gng_fold(const float* part_n, int Gn, float* out_a, float* out_b) {
  const int g = threadIdx.x >> 4, part = threadIdx.x & 15;
  float sa = 0.f, ca = 0.f, sb = 0.f, cb = 0.f;
  for (int j = part; j < Gn; j += 16) {
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
  for (int o = 8; o > 0; o >>= 1) {
    da += __shfl_xor_sync(0xffffffffu, da, o);
    db += __shfl_xor_sync(0xffffffffu, db, o);
  }
  if (part == 0) {
    out_a[g] = da;
    out_b[g] = db;
  }
  gng_sync();
}

// ---- the ring: NT tensors (1: x; 2: dy, x), R pixel rows of C channels per stage and tensor
struct GngRing {
  uint8_t* buf;
  uint64_t *full, *empty;
  int R, row_bytes, tensor_bytes;  // rows per stage, C * 2, R * C * 2
};

// Producer warp: `passes` trips over pixels [p0, p1) of the NT source tensors (row strides ld[t] elements).
template <int NT>
__device__ __forceinline__ void gng_produce(const GngRing& rg, const __half* const (&src)[NT], const int64_t (&ld)[NT], int C, int p0, int p1,
                                            int passes, uint32_t& cnt) {
  const int lane = threadIdx.x & 31;
  const int n_it = (p1 - p0 + rg.R - 1) / rg.R;
  for (int pass = 0; pass < passes; ++pass) {
    for (int it = 0; it < n_it; ++it, ++cnt) {
      const int stage = cnt % kGngStages;
      const uint32_t parity = (cnt / kGngStages) & 1u;
      if (lane == 0) mbar_wait(&rg.empty[stage], parity ^ 1u);
      __syncwarp();
      const int p = p0 + it * rg.R;
      const int rows = min(rg.R, p1 - p);
      if (lane == 0) mbar_expect_tx(&rg.full[stage], (uint32_t)(NT * rows * rg.row_bytes));
      __syncwarp();
      uint8_t* dst = rg.buf + stage * kGngStageBytes;
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        if (ld[t] == C) {  // the pixel range is one contiguous block
          if (lane == t) bulk_load_1d(dst + t * rg.tensor_bytes, src[t] + (int64_t)p * C, (uint32_t)(rows * rg.row_bytes), &rg.full[stage]);
        } else {           // channel slice of a wider tensor: one copy per pixel row
          for (int r = lane; r < rows; r += 32)
            bulk_load_1d(dst + t * rg.tensor_bytes + r * rg.row_bytes, src[t] + (int64_t)(p + r) * ld[t], (uint32_t)rg.row_bytes, &rg.full[stage]);
        }
      }
    }
  }
}

// Consumer side of one trip: f(p, v[NT]) for every (pixel row p, 8-channel vector) this thread owns.
template <int NT, typename F>
__device__ __forceinline__ void gng_consume(const GngRing& rg, uint32_t& cnt, int p0, int p1, int col, int pl, int PP, bool active, F&& f) {
  const int lane = threadIdx.x & 31;
  const int n_it = (p1 - p0 + rg.R - 1) / rg.R;
  for (int it = 0; it < n_it; ++it, ++cnt) {
    const int stage = cnt % kGngStages;
    const uint32_t parity = (cnt / kGngStages) & 1u;
    mbar_wait(&rg.full[stage], parity);
    const int p = p0 + it * rg.R;
    const int rows = min(rg.R, p1 - p);
    const uint8_t* base = rg.buf + stage * kGngStageBytes + col * 16;
    if (active) {
      for (int r = pl; r < rows; r += PP) {
        half8 v[NT];
#pragma unroll
        for (int t = 0; t < NT; ++t) v[t] = ld8(reinterpret_cast<const __half*>(base + t * rg.tensor_bytes + r * rg.row_bytes));
        f(p + r, v);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&rg.empty[stage]);
  }
}

__device__ __forceinline__ void gng_ring_init(GngRing& rg, uint8_t* dyn_smem, uint64_t* bars, int C, int NT) {
  rg.buf = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(dyn_smem) + 127) & ~uintptr_t(127));
  rg.full = bars;
  rg.empty = bars + kGngStages;
  rg.row_bytes = C * 2;
  const int V = C / 8, PP = kGngConsumers / V;
  rg.R = (NT == 1 ? 2 : 1) * PP;  // 16 KB (one tensor) or 2 x 8 KB per stage when C / 8 divides 512
  rg.tensor_bytes = rg.R * rg.row_bytes;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kGngStages; ++s) {
      mbar_init(&rg.full[s], 1);
      mbar_init(&rg.empty[s], kGngConsumers / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
}

// ------------------------------------------------------------------------------------------------ forward
__global__ void __launch_bounds__(kGngThreads, 1)
gn_fwd_grid_kernel(const __half* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                   const float* __restrict__ emb, __half* __restrict__ y, float* __restrict__ stats, float* __restrict__ partials,
                   unsigned int* __restrict__ bar, int HW, int C, int64_t ldx, int64_t ldy, int Gn, float eps, int silu) {
  extern __shared__ uint8_t gng_dyn[];
  __shared__ float red_s[kGngConsumers * 8], red_q[kGngConsumers * 8];
  __shared__ float gs[32], gq[32];
  __shared__ float fa[32], fb[32];
  __shared__ float s_mean[32], s_rstd[32];
  __shared__ __align__(8) uint64_t bars[2 * kGngStages];
  const int n = blockIdx.x / Gn, chunk = blockIdx.x % Gn;
  const int V = C / 8, PP = kGngConsumers / V;
  const int cpg = C / 32;
  const int ppc = (HW + Gn - 1) / Gn;
  const int p0 = min(HW, chunk * ppc), p1 = min(HW, p0 + ppc);
  GngRing rg;
  gng_ring_init(rg, gng_dyn, bars, C, 1);
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();
  const __half* xn = x + (int64_t)n * HW * ldx;
  if (threadIdx.x >= kGngConsumers) {
    const __half* const src[1] = {xn};
    const int64_t ld[1] = {ldx};
    uint32_t pcnt = 0;
    gng_produce<1>(rg, src, ld, C, p0, p1, 2, pcnt);
    return;
  }
  const int col = threadIdx.x % V, pl = threadIdx.x / V;
  const bool active = pl < PP;
  // The sums are taken about a per-group pivot -- the group's first element, the same in every CTA -- so that E[x^2] - mean^2 below
  // cancels only over the spread of x around it, not over the group's mean: without it the variance of a group whose |mean| is
  // 64 std loses ~12 of fp32's 24 bits.  The gain assumes the pivot (pixel 0, an image corner) lies within a few std of the group's
  // mean: a pivot k std away loses ~log2(1 + k^2) bits again, as a mean of k std did without it.  |mean - pivot| / std has not been
  // measured on real activations.
  float s[8], q[8], piv[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    s[j] = q[j] = 0.f;
    piv[j] = __half2float(xn[(col * 8 + j) / cpg * cpg]);
  }
  uint32_t cnt = 0;
  gng_consume<1>(rg, cnt, p0, p1, col, pl, PP, active, [&](int, const half8(&v)[1]) {
    float f[8];
    unpack8(v[0], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float d = f[j] - piv[j];
      s[j] += d;
      q[j] = fmaf(d, d, q[j]);
    }
  });
  gng_block_reduce(s, q, C, col, pl, PP, active, red_s, red_q, gs, gq);
  if (threadIdx.x < 32) {
    float* o = partials + (((int64_t)n * Gn + chunk) * 32 + threadIdx.x) * 2;
    o[0] = gs[threadIdx.x];
    o[1] = gq[threadIdx.x];
  }
  grid_barrier(bar, gridDim.x);
  gng_fold(partials + (int64_t)n * Gn * 64, Gn, fa, fb);
  if (threadIdx.x < 32) {
    const float inv_m = 1.f / ((float)cpg * (float)HW);
    const float dm = fa[threadIdx.x] * inv_m;  // mean - pivot
    const float mu = __half2float(xn[threadIdx.x * cpg]) + dm;
    const float var = fmaxf(fmaf(-dm, dm, fb[threadIdx.x] * inv_m), 0.f);  // relative error ~ 6e-8 * (mean - pivot)^2 / var
    const float rs = 1.f / sqrtf(var + eps);
    s_mean[threadIdx.x] = mu;
    s_rstd[threadIdx.x] = rs;
    if (chunk == 0) {
      stats[((int64_t)n * 32 + threadIdx.x) * 2 + 0] = mu;
      stats[((int64_t)n * 32 + threadIdx.x) * 2 + 1] = rs;
    }
  }
  gng_sync();
  float A[8], Bc[8];
  if (active) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = col * 8 + j, g = c / cpg;
      const float mu = s_mean[g], rs = s_rstd[g];
      const float ga = gamma[c], be = beta[c];
      float sc1 = 1.f, sh = 0.f;
      if (emb) {
        sc1 = 1.f + emb[(int64_t)n * 2 * C + c];
        sh = emb[(int64_t)n * 2 * C + C + c];
      }
      A[j] = rs * ga * sc1;
      Bc[j] = (be - mu * rs * ga) * sc1 + sh;
    }
  }
  __half* yb = y + (int64_t)n * HW * ldy + col * 8;
  gng_consume<1>(rg, cnt, p0, p1, col, pl, PP, active, [&](int p, const half8(&v)[1]) {
    float f[8];
    unpack8(v[0], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float t = fmaf(f[j], A[j], Bc[j]);
      f[j] = silu ? silu_f(t) : t;
    }
    st8(yb + (int64_t)p * ldy, pack8(f));
  });
}

// ------------------------------------------------------------------------------------------------ backward
__global__ void __launch_bounds__(kGngThreads, 1)
gn_bwd_grid_kernel(const __half* __restrict__ dy, const __half* __restrict__ x, const float* __restrict__ stats,
                   const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ emb,
                   __half* __restrict__ dx, float* __restrict__ partials, unsigned int* __restrict__ bar, __half* __restrict__ tmp, int HW,
                   int C, int64_t ld_dy, int64_t ldx, int64_t ld_dx, int Gn, int silu, int accumulate) {
  // `tmp` (optional scratch, dense [N, HW, C] fp16): the first trip stores d xhat = dy * silu'(v) * d v / d xhat once -- the fp16
  // tensor the reference's autograd holds between SiLU.backward and GroupNorm.backward -- and the second trip streams it back
  // instead of dy, so SiLU' (2 MUFU + ~10 FP32 ops per element) is not recomputed.  Each CTA re-reads only what it wrote.
  extern __shared__ uint8_t gng_dyn[];
  __shared__ float red_s[kGngConsumers * 8], red_q[kGngConsumers * 8];
  __shared__ float gs[32], gq[32];
  __shared__ float fa[32], fb[32];
  __shared__ float s_m1[32], s_m2[32];
  __shared__ __align__(8) uint64_t bars[2 * kGngStages + 1];
  uint64_t* trip1_done = &bars[2 * kGngStages];
  const int n = blockIdx.x / Gn, chunk = blockIdx.x % Gn;
  const int V = C / 8, PP = kGngConsumers / V;
  const int cpg = C / 32;
  const int ppc = (HW + Gn - 1) / Gn;
  const int p0 = min(HW, chunk * ppc), p1 = min(HW, p0 + ppc);
  GngRing rg;
  gng_ring_init(rg, gng_dyn, bars, C, 2);
  if (threadIdx.x == 0) {
    mbar_init(trip1_done, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();
  __half* tmp_n = tmp ? tmp + (int64_t)n * HW * C : nullptr;
  if (threadIdx.x >= kGngConsumers) {
    const __half* const src[2] = {dy + (int64_t)n * HW * ld_dy, x + (int64_t)n * HW * ldx};
    const int64_t ld[2] = {ld_dy, ldx};
    uint32_t pcnt = 0;
    if (!tmp) {
      gng_produce<2>(rg, src, ld, C, p0, p1, 2, pcnt);
    } else {
      gng_produce<2>(rg, src, ld, C, p0, p1, 1, pcnt);
      if ((threadIdx.x & 31) == 0) mbar_wait(trip1_done, 0);  // the consumers' d xhat stores of this CTA's range are visible
      __syncwarp();
      const __half* const src2[2] = {tmp_n, x + (int64_t)n * HW * ldx};
      const int64_t ld2[2] = {C, ldx};
      gng_produce<2>(rg, src2, ld2, C, p0, p1, 1, pcnt);
    }
    return;
  }
  const int col = threadIdx.x % V, pl = threadIdx.x / V;
  const bool active = pl < PP;
  float G[8], Bc[8], mu[8], rs[8];
  if (active) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = col * 8 + j, g = c / cpg;
      mu[j] = stats[((int64_t)n * 32 + g) * 2];
      rs[j] = stats[((int64_t)n * 32 + g) * 2 + 1];
      float sc1 = 1.f, sh = 0.f;
      if (emb) {
        sc1 = 1.f + emb[(int64_t)n * 2 * C + c];
        sh = emb[(int64_t)n * 2 * C + C + c];
      }
      const float ga = gamma[c];
      G[j] = ga * sc1;                                   // d v / d xhat
      Bc[j] = (beta[c] - mu[j] * rs[j] * ga) * sc1 + sh;  // v = x * (rs * G) + Bc
    }
  }
  float s[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
  uint32_t cnt = 0;
  gng_consume<2>(rg, cnt, p0, p1, col, pl, PP, active, [&](int p, const half8(&v)[2]) {
    float d[8], a[8];
    unpack8(v[0], d);
    unpack8(v[1], a);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float dv = d[j];
      if (silu) dv *= silu_grad_f(fmaf(a[j], rs[j] * G[j], Bc[j]));
      const float dxh = dv * G[j];
      const float xh = (a[j] - mu[j]) * rs[j];
      d[j] = dxh;
      q[j] = fmaf(dxh, xh, q[j]);
    }
    if (tmp_n) {
      const half8 h = pack8(d);
      st8(tmp_n + (int64_t)p * C + col * 8, h);
      unpack8(h, d);  // the statistics use the rounded values the second trip will read
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] += d[j];
  });
  if (tmp_n) {  // generic-proxy global stores -> async-proxy (cp.async.bulk) reads by this CTA's producer warp
    asm volatile("fence.proxy.async;" ::: "memory");
    __threadfence();
  }
  gng_block_reduce(s, q, C, col, pl, PP, active, red_s, red_q, gs, gq);
  if (tmp_n && threadIdx.x == 0) mbar_arrive(trip1_done);  // after the barriers inside the reduce: every consumer has fenced
  if (threadIdx.x < 32) {
    float* o = partials + (((int64_t)n * Gn + chunk) * 32 + threadIdx.x) * 2;
    o[0] = gs[threadIdx.x];
    o[1] = gq[threadIdx.x];
  }
  grid_barrier(bar, gridDim.x);
  gng_fold(partials + (int64_t)n * Gn * 64, Gn, fa, fb);
  if (threadIdx.x < 32) {
    const float inv_m = 1.f / ((float)cpg * (float)HW);
    s_m1[threadIdx.x] = fa[threadIdx.x] * inv_m;  // mean(dxhat)
    s_m2[threadIdx.x] = fb[threadIdx.x] * inv_m;  // mean(dxhat * xhat)
  }
  gng_sync();
  float m1[8], m2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int g = min((col * 8 + j) / cpg, 31);
    m1[j] = s_m1[g];
    m2[j] = s_m2[g];
  }
  __half* ob = dx + (int64_t)n * HW * ld_dx + col * 8;
  gng_consume<2>(rg, cnt, p0, p1, col, pl, PP, active, [&](int p, const half8(&v)[2]) {
    float d[8], a[8], o[8];
    if (accumulate) unpack8(ld8(ob + (int64_t)p * ld_dx), o);
    unpack8(v[0], d);
    unpack8(v[1], a);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float dxh = d[j];  // with `tmp`: d xhat itself
      if (!tmp_n) {
        if (silu) dxh *= silu_grad_f(fmaf(a[j], rs[j] * G[j], Bc[j]));
        dxh *= G[j];
      }
      const float xh = (a[j] - mu[j]) * rs[j];
      const float r = rs[j] * (dxh - m1[j] - xh * m2[j]);
      o[j] = accumulate ? o[j] + r : r;
    }
    st8(ob + (int64_t)p * ld_dx, pack8(o));
  });
}

// ------------------------------------------------------------------------------------------------ host
constexpr int kGngDynSmem = kGngStages * kGngStageBytes + 128;
constexpr int kGngCtasPerSm = 1;  // measured: two CTAs per SM (56 registers, 4 stages) ran 1.4 - 1.9x SLOWER (296-way barrier, spills)

static int gng_check(const char* what, int64_t N, int64_t HW, int64_t C, int64_t Gn) {
  CGD_CHECK_ARG(N > 0 && HW > 0, "%s: bad dims", what);
  CGD_CHECK_ARG(C >= 64 && C % 64 == 0 && C <= 2048, "%s: C=%lld must be a multiple of 64 in [64, 2048]", what, (long long)C);
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    CGD_CUDA(cudaGetDevice(&dev));
    CGD_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  }
  // the grid barrier needs every CTA resident: one 544-thread CTA per SM
  CGD_CHECK_ARG(Gn >= 1 && N * Gn <= kGngCtasPerSm * sms, "%s: %lld x %lld CTAs exceed %d per SM x %d SMs (grid barrier needs a resident grid)",
                what, (long long)N, (long long)Gn, kGngCtasPerSm, sms);
  return 0;
}
// norm_grid2.cu: the direct-load backward (C % 256 == 0)
bool gn_grid2_supports(int64_t C);
int launch_gn_bwd_grid2(const CgdOp& op, cudaStream_t st);
// Every forward runs on the ring kernels of this file.  A backward of a large activation (HW * C >= 2^23) whose width the direct-load
// kernel takes runs on that kernel, which keeps more bytes in flight; smaller ones stay on the ring.
static bool gn_bwd_direct(int64_t HW, int64_t C) { return gn_grid2_supports(C) && HW * C >= (int64_t(1) << 23); }

template <typename K>
static int gng_prepare(K kernel) {
  CGD_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kGngDynSmem));
  int occ = 0;
  CGD_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, kGngThreads, kGngDynSmem));
  CGD_CHECK_ARG(occ >= kGngCtasPerSm, "groupnorm grid kernel: only %d CTA(s) per SM fit, the grid barrier assumes %d", occ, kGngCtasPerSm);
  return 0;
}

int launch_gn_fwd_grid(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], HW = op.i[1], C = op.i[2], ldx = op.i[3], ldy = op.i[4], Gn = op.i[5];
  if (int rc = gng_check("gn_fwd_grid", N, HW, C, Gn)) return rc;
  CGD_CHECK_ARG(ldx % 8 == 0 && ldy % 8 == 0 && op.p[0] && op.p[1] && op.p[2] && op.p[4] && op.p[5] && op.p[6] && op.p[7], "gn_fwd_grid: bad args");
  static DeviceOnce set;
  if (set.needed()) {
    if (int rc = gng_prepare(gn_fwd_grid_kernel)) return rc;
    set.mark();
  }
  CGD_CUDA(launch_pdl(gn_fwd_grid_kernel, dim3((unsigned)(N * Gn)), dim3(kGngThreads), kGngDynSmem, st, (const __half*)op.p[0], (const float*)op.p[1],
                      (const float*)op.p[2], (const float*)op.p[3], (__half*)op.p[4], (float*)op.p[5], (float*)op.p[6], (unsigned int*)op.p[7],
                      (int)HW, (int)C, ldx, ldy, (int)Gn, op.f[0], (int)(op.flags & 1)));
  return 0;
}

int launch_gn_bwd_grid(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], HW = op.i[1], C = op.i[2], ld_dy = op.i[3], ldx = op.i[4], ld_dx = op.i[5], Gn = op.i[6];
  if (int rc = gng_check("gn_bwd_grid", N, HW, C, Gn)) return rc;
  CGD_CHECK_ARG(ld_dy % 8 == 0 && ldx % 8 == 0 && ld_dx % 8 == 0 && op.p[0] && op.p[1] && op.p[2] && op.p[3] && op.p[4] && op.p[6] && op.p[7] &&
                    op.p[8],
                "gn_bwd_grid: bad args");
  if (gn_bwd_direct(HW, C)) return launch_gn_bwd_grid2(op, st);
  static DeviceOnce set;
  if (set.needed()) {
    if (int rc = gng_prepare(gn_bwd_grid_kernel)) return rc;
    set.mark();
  }
  CGD_CUDA(launch_pdl(gn_bwd_grid_kernel, dim3((unsigned)(N * Gn)), dim3(kGngThreads), kGngDynSmem, st, (const __half*)op.p[0], (const __half*)op.p[1],
                      (const float*)op.p[2], (const float*)op.p[3], (const float*)op.p[4], (const float*)op.p[5], (__half*)op.p[6],
                      (float*)op.p[7], (unsigned int*)op.p[8], (__half*)op.p[9], (int)HW, (int)C, ld_dy, ldx, ld_dx, (int)Gn, (int)(op.flags & 1),
                      (int)((op.flags & 2) ? 1 : 0)));
  return 0;
}

}  // namespace cgd
