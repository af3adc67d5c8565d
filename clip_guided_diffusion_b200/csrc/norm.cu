// norm.cu -- GroupNorm(32) and LayerNorm, forward and input-gradient, on pixel-major fp16 activations.
//
// Replaces [3P] guided-diffusion GroupNorm32 (+ the SiLU / scale-shift elementwise work around it) and
// [3P] CLIP LayerNorm that the reference runs as unfused ATen kernels with fp32 up-casts
// (SURVEY.md K5, K6, K15).  All reductions are fp32 (final combination in fp64), deterministic
// (per-chunk partials combined in a fixed order by the last block to finish, no float atomics in
// global memory), 128-bit vectorised and coalesced along the channel dimension.
#include "common.cuh"
#include "pdl.cuh"
#include "ops.cuh"

namespace cgd {

// Thread mapping shared by all GroupNorm kernels: blockDim.x = V * PP with V = C/8 vector columns;
// a thread owns 8 consecutive channels (col*8 ..) and walks pixels pl, pl+PP, ...
struct GnGeom {
  int V, PP, threads;
};
static GnGeom gn_geom(int C) {
  GnGeom g;
  g.V = C / 8;
  g.PP = 256 / g.V;
  if (g.PP < 1) g.PP = 1;
  g.threads = g.V * g.PP;
  return g;
}

// Deterministic block reduction of per-thread channel sums into the 32 groups: every thread parks its 8 channel sums in
// shared memory ([pixel lane][channel], PP * C <= 2048 floats), then thread g adds the PP * (C/32) = 64 values of group g in
// a fixed order.  (Shared float atomics would make the statistics -- and everything downstream -- run-to-run different.)
__device__ __forceinline__ void block_group_reduce(const float* s, const float* q, int C, int col, int pl, int PP, float* red_s,
                                                   float* red_q, float* gs, float* gq) {
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    red_s[pl * C + col * 8 + j] = s[j];
    red_q[pl * C + col * 8 + j] = q[j];
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    const int cpg = C / 32, g = threadIdx.x;
    float as = 0.f, aq = 0.f;
    for (int l = 0; l < PP; ++l)
      for (int c = 0; c < cpg; ++c) {
        as += red_s[l * C + g * cpg + c];
        aq += red_q[l * C + g * cpg + c];
      }
    gs[g] = as;
    gq[g] = aq;
  }
  __syncthreads();
}

// Fixed-order (deterministic) fold of [nchunk][32][2] partials by the whole block: thread t sums chunks t/32, t/32 + nthr/32, ...
// for group t%32 in fp64, then the per-part sums are combined in ascending part order.
__device__ __forceinline__ void fold_partials(const float* part, int nchunk, double* out_s, double* out_q) {
  __shared__ double ps[8][32], pq[8][32];
  const int g = threadIdx.x & 31, part_id = threadIdx.x >> 5;
  const int nparts = min((int)(blockDim.x >> 5), 8);
  if (part_id < nparts) {
    double ds = 0.0, dq = 0.0;
    int c = part_id;
    // 8 independent (sum, sumsq) pairs in flight per thread: the loop is latency-bound (L2), not bandwidth-bound
    for (; c + 7 * nparts < nchunk; c += 8 * nparts) {
      float2 v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = __ldcg(reinterpret_cast<const float2*>(part + ((int64_t)(c + u * nparts) * 32 + g) * 2));
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        ds += (double)v[u].x;
        dq += (double)v[u].y;
      }
    }
    for (; c < nchunk; c += nparts) {
      const float2 v = __ldcg(reinterpret_cast<const float2*>(part + ((int64_t)c * 32 + g) * 2));
      ds += (double)v.x;
      dq += (double)v.y;
    }
    ps[part_id][g] = ds;
    pq[part_id][g] = dq;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    double ds = 0.0, dq = 0.0;
    for (int k = 0; k < nparts; ++k) {
      ds += ps[k][g];
      dq += pq[k][g];
    }
    out_s[g] = ds;
    out_q[g] = dq;
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// pass 1: per-(image, chunk, group) sum and sum of squares; last block per image folds the chunks.
__global__ void gn_stats_kernel(const __half* __restrict__ x, float* __restrict__ partials, float* __restrict__ stats,
                                unsigned int* __restrict__ counters, int HW, int C, int64_t ld, int nchunk, float eps) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float gs[32], gq[32];
  __shared__ float red_s[2048], red_q[2048];
  __shared__ double fold_s[32], fold_q[32];
  __shared__ int is_last;
  const int n = blockIdx.y, chunk = blockIdx.x;
  const int V = C / 8, col = threadIdx.x % V, pl = threadIdx.x / V, PP = blockDim.x / V;
  const int cpg = C / 32;
  const int ppc = (HW + nchunk - 1) / nchunk;
  const int p0 = chunk * ppc, p1 = min(HW, p0 + ppc);
  // sums about a per-group pivot (the group's first element, the same in every block): the fold's E[x^2] - mean^2 then cancels only
  // over the spread of x around it, not over the group's mean.  That assumes the pivot (pixel 0, an image corner) lies within a few
  // std of the mean: k std away costs ~log2(1 + k^2) bits, as before; not measured on real activations.
  float s[8], q[8], piv[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    s[j] = q[j] = 0.f;
    piv[j] = __half2float(x[(int64_t)n * HW * ld + (col * 8 + j) / cpg * cpg]);
  }
  const __half* xb = x + (int64_t)n * HW * ld + col * 8;
  for (int p = p0 + pl; p < p1; p += 4 * PP) {  // 4 independent 128-bit loads in flight per thread
    half8 raw[4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (p + u * PP < p1) raw[u] = ld8(xb + (int64_t)(p + u * PP) * ld);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (p + u * PP < p1) {
        float v[8];
        unpack8(raw[u], v);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[j] - piv[j];
          s[j] += d;
          q[j] = fmaf(d, d, q[j]);
        }
      }
    }
  }
  __syncthreads();
  block_group_reduce(s, q, C, col, pl, PP, red_s, red_q, gs, gq);
  if (threadIdx.x < 32) {
    float* o = partials + (((int64_t)n * nchunk + chunk) * 32 + threadIdx.x) * 2;
    o[0] = gs[threadIdx.x];
    o[1] = gq[threadIdx.x];
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(&counters[n], 1u) == (unsigned)(nchunk - 1));
  __syncthreads();
  if (is_last) {
    __threadfence();
    fold_partials(partials + (int64_t)n * nchunk * 64, nchunk, fold_s, fold_q);
    if (threadIdx.x < 32) {
      const double ds = fold_s[threadIdx.x], dq = fold_q[threadIdx.x];
      const double m = (double)cpg * (double)HW;
      const double dm = ds / m;  // mean - pivot
      double var = dq / m - dm * dm;
      if (var < 0.0) var = 0.0;
      const double mean = (double)__half2float(x[(int64_t)n * HW * ld + threadIdx.x * cpg]) + dm;
      stats[((int64_t)n * 32 + threadIdx.x) * 2 + 0] = (float)mean;
      stats[((int64_t)n * 32 + threadIdx.x) * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
    }
    if (threadIdx.x == 0) counters[n] = 0u;  // self-reset for the next launch / graph replay
  }
}

// per-thread affine of the normalisation: v = x*A + B (v = pre-activation), G = d v / d xhat
__device__ __forceinline__ void gn_coeffs(const float* stats, const float* gamma, const float* beta, const float* emb, int n,
                                          int C, int col, float* A, float* Bc, float* G, float* mean, float* rstd) {
  const int cpg = C / 32;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = col * 8 + j, g = c / cpg;
    const float mu = stats[((int64_t)n * 32 + g) * 2], rs = stats[((int64_t)n * 32 + g) * 2 + 1];
    float ga = gamma[c], be = beta[c];
    float sc1 = 1.f, sh = 0.f;
    if (emb) {
      sc1 = 1.f + emb[(int64_t)n * 2 * C + c];
      sh = emb[(int64_t)n * 2 * C + C + c];
    }
    A[j] = rs * ga * sc1;
    Bc[j] = (be - mu * rs * ga) * sc1 + sh;
    G[j] = ga * sc1;
    mean[j] = mu;
    rstd[j] = rs;
  }
}

__global__ void gn_apply_kernel(const __half* __restrict__ x, const float* __restrict__ stats, const float* __restrict__ gamma,
                                const float* __restrict__ beta, const float* __restrict__ emb, __half* __restrict__ y, int HW,
                                int C, int64_t ldx, int64_t ldy, int silu) {
  pdl_wait();
  pdl_launch_dependents();
  const int n = blockIdx.y;
  const int V = C / 8, col = threadIdx.x % V, pl = threadIdx.x / V, PP = blockDim.x / V;
  float A[8], Bc[8], G[8], mu[8], rs[8];
  gn_coeffs(stats, gamma, beta, emb, n, C, col, A, Bc, G, mu, rs);
  const __half* xb = x + (int64_t)n * HW * ldx + col * 8;
  __half* yb = y + (int64_t)n * HW * ldy + col * 8;
  const int stride = gridDim.x * PP;
  for (int p = blockIdx.x * PP + pl; p < HW; p += 4 * stride) {
    half8 raw[4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (p + u * stride < HW) raw[u] = ld8(xb + (int64_t)(p + u * stride) * ldx);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (p + u * stride < HW) {
        float v[8];
        unpack8(raw[u], v);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float t = fmaf(v[j], A[j], Bc[j]);
          v[j] = silu ? silu_f(t) : t;
        }
        st8(yb + (int64_t)(p + u * stride) * ldy, pack8(v));
      }
    }
  }
}

// backward pass 1: s1 = sum dxhat, s2 = sum dxhat * xhat per (image, group)
__global__ void gn_bwd_stats_kernel(const __half* __restrict__ dy, const __half* __restrict__ x, const float* __restrict__ stats,
                                    const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ emb,
                                    float* __restrict__ partials, float* __restrict__ sums, unsigned int* __restrict__ counters,
                                    int HW, int C, int64_t ld_dy, int64_t ldx, int nchunk, int silu) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float gs[32], gq[32];
  __shared__ float red_s[2048], red_q[2048];
  __shared__ double fold_s[32], fold_q[32];
  __shared__ int is_last;
  const int n = blockIdx.y, chunk = blockIdx.x;
  const int V = C / 8, col = threadIdx.x % V, pl = threadIdx.x / V, PP = blockDim.x / V;
  const int cpg = C / 32;
  const int ppc = (HW + nchunk - 1) / nchunk;
  const int p0 = chunk * ppc, p1 = min(HW, p0 + ppc);
  float A[8], Bc[8], G[8], mu[8], rs[8];
  gn_coeffs(stats, gamma, beta, emb, n, C, col, A, Bc, G, mu, rs);
  float s[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
  const __half* xb = x + (int64_t)n * HW * ldx + col * 8;
  const __half* db = dy + (int64_t)n * HW * ld_dy + col * 8;
  for (int p = p0 + pl; p < p1; p += 2 * PP) {  // 4 independent 128-bit loads in flight per thread
    half8 rx[2], rd[2];
#pragma unroll
    for (int u = 0; u < 2; ++u)
      if (p + u * PP < p1) {
        rx[u] = ld8(xb + (int64_t)(p + u * PP) * ldx);
        rd[u] = ld8(db + (int64_t)(p + u * PP) * ld_dy);
      }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (p + u * PP < p1) {
        float v[8], d[8];
        unpack8(rx[u], v);
        unpack8(rd[u], d);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float dv = d[j];
          if (silu) dv *= silu_grad_f(fmaf(v[j], A[j], Bc[j]));
          const float dxh = dv * G[j];
          const float xh = (v[j] - mu[j]) * rs[j];
          s[j] += dxh;
          q[j] = fmaf(dxh, xh, q[j]);
        }
      }
    }
  }
  __syncthreads();
  block_group_reduce(s, q, C, col, pl, PP, red_s, red_q, gs, gq);
  if (threadIdx.x < 32) {
    float* o = partials + (((int64_t)n * nchunk + chunk) * 32 + threadIdx.x) * 2;
    o[0] = gs[threadIdx.x];
    o[1] = gq[threadIdx.x];
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(&counters[n], 1u) == (unsigned)(nchunk - 1));
  __syncthreads();
  if (is_last) {
    __threadfence();
    fold_partials(partials + (int64_t)n * nchunk * 64, nchunk, fold_s, fold_q);
    if (threadIdx.x < 32) {
      const double ds = fold_s[threadIdx.x], dq = fold_q[threadIdx.x];
      const double m = (double)cpg * (double)HW;
      sums[((int64_t)n * 32 + threadIdx.x) * 2 + 0] = (float)(ds / m);  // mean(dxhat)
      sums[((int64_t)n * 32 + threadIdx.x) * 2 + 1] = (float)(dq / m);  // mean(dxhat * xhat)
    }
    if (threadIdx.x == 0) counters[n] = 0u;
  }
}

__global__ void gn_bwd_apply_kernel(const __half* __restrict__ dy, const __half* __restrict__ x, const float* __restrict__ stats,
                                    const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ emb,
                                    const float* __restrict__ sums, __half* __restrict__ dx, int HW, int C, int64_t ld_dy,
                                    int64_t ldx, int64_t ld_dx, int silu, int accumulate) {
  pdl_wait();
  pdl_launch_dependents();
  const int n = blockIdx.y;
  const int V = C / 8, col = threadIdx.x % V, pl = threadIdx.x / V, PP = blockDim.x / V;
  const int cpg = C / 32;
  float A[8], Bc[8], G[8], mu[8], rs[8], m1[8], m2[8];
  gn_coeffs(stats, gamma, beta, emb, n, C, col, A, Bc, G, mu, rs);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int g = (col * 8 + j) / cpg;
    m1[j] = sums[((int64_t)n * 32 + g) * 2];
    m2[j] = sums[((int64_t)n * 32 + g) * 2 + 1];
  }
  const __half* xb = x + (int64_t)n * HW * ldx + col * 8;
  const __half* db = dy + (int64_t)n * HW * ld_dy + col * 8;
  __half* ob = dx + (int64_t)n * HW * ld_dx + col * 8;
  const int stride = gridDim.x * PP;
  for (int p = blockIdx.x * PP + pl; p < HW; p += 2 * stride) {
    half8 rx[2], rd[2], ro[2];
#pragma unroll
    for (int u = 0; u < 2; ++u)
      if (p + u * stride < HW) {
        rx[u] = ld8(xb + (int64_t)(p + u * stride) * ldx);
        rd[u] = ld8(db + (int64_t)(p + u * stride) * ld_dy);
        if (accumulate) ro[u] = ld8(ob + (int64_t)(p + u * stride) * ld_dx);
      }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (p + u * stride < HW) {
        float v[8], d[8], o[8];
        unpack8(rx[u], v);
        unpack8(rd[u], d);
        if (accumulate) unpack8(ro[u], o);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float dv = d[j];
          if (silu) dv *= silu_grad_f(fmaf(v[j], A[j], Bc[j]));
          const float dxh = dv * G[j];
          const float xh = (v[j] - mu[j]) * rs[j];
          const float r = rs[j] * (dxh - m1[j] - xh * m2[j]);
          o[j] = accumulate ? o[j] + r : r;
        }
        st8(ob + (int64_t)(p + u * stride) * ld_dx, pack8(o));
      }
    }
  }
}

static int gn_check(const CgdOp& op, int64_t C, int64_t HW, int64_t N) {
  CGD_CHECK_ARG(N > 0 && HW > 0, "groupnorm: bad dims");
  CGD_CHECK_ARG(C >= 64 && C % 64 == 0 && C <= 2048, "groupnorm: C=%lld must be a multiple of 64 in [64, 2048]", (long long)C);
  return 0;
}
static int gn_apply_chunks(int64_t HW, int64_t N, int PP) {
  int64_t c = ceil_div(HW, (int64_t)PP * 8);
  const int64_t cap = ceil_div(132 * 3, N);
  if (c > cap) c = cap;
  if (c < 1) c = 1;
  return (int)c;
}

int launch_gn_stats(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], HW = op.i[1], C = op.i[2], ld = op.i[3], nchunk = op.i[4];
  if (int rc = gn_check(op, C, HW, N)) return rc;
  CGD_CHECK_ARG(nchunk >= 1 && ld % 8 == 0 && op.p[0] && op.p[1] && op.p[2] && op.p[3], "gn_stats: bad args");
  const GnGeom g = gn_geom((int)C);
  CGD_CUDA(launch_pdl(gn_stats_kernel, dim3((unsigned)nchunk, (unsigned)N), dim3(g.threads), 0, st, 
      (const __half*)op.p[0], (float*)op.p[1], (float*)op.p[2], (unsigned int*)op.p[3], (int)HW, (int)C, ld, (int)nchunk, op.f[0]));
  CGD_LAUNCH_CHECK();
  return 0;
}

int launch_gn_apply(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], HW = op.i[1], C = op.i[2], ldx = op.i[3], ldy = op.i[5];
  if (int rc = gn_check(op, C, HW, N)) return rc;
  CGD_CHECK_ARG(ldx % 8 == 0 && ldy % 8 == 0 && op.p[0] && op.p[1] && op.p[2] && op.p[3] && op.p[5], "gn_apply: bad args");
  const GnGeom g = gn_geom((int)C);
  CGD_CUDA(launch_pdl(gn_apply_kernel, dim3(gn_apply_chunks(HW, N, g.PP), (unsigned)N), dim3(g.threads), 0, st, 
      (const __half*)op.p[0], (const float*)op.p[1], (const float*)op.p[2], (const float*)op.p[3], (const float*)op.p[4],
      (__half*)op.p[5], (int)HW, (int)C, ldx, ldy, op.flags & 1));
  CGD_LAUNCH_CHECK();
  return 0;
}

int launch_gn_bwd_stats(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], HW = op.i[1], C = op.i[2], ld_dy = op.i[3], ldx = op.i[4], nchunk = op.i[5];
  if (int rc = gn_check(op, C, HW, N)) return rc;
  CGD_CHECK_ARG(nchunk >= 1 && ld_dy % 8 == 0 && ldx % 8 == 0 && op.p[0] && op.p[1] && op.p[2] && op.p[6] && op.p[7] && op.p[8],
                "gn_bwd_stats: bad args");
  const GnGeom g = gn_geom((int)C);
  CGD_CUDA(launch_pdl(gn_bwd_stats_kernel, dim3((unsigned)nchunk, (unsigned)N), dim3(g.threads), 0, st, 
      (const __half*)op.p[0], (const __half*)op.p[1], (const float*)op.p[2], (const float*)op.p[3], (const float*)op.p[4],
      (const float*)op.p[5], (float*)op.p[6], (float*)op.p[7], (unsigned int*)op.p[8], (int)HW, (int)C, ld_dy, ldx, (int)nchunk,
      op.flags & 1));
  CGD_LAUNCH_CHECK();
  return 0;
}

int launch_gn_bwd_apply(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], HW = op.i[1], C = op.i[2], ld_dy = op.i[3], ldx = op.i[4], ld_dx = op.i[6];
  if (int rc = gn_check(op, C, HW, N)) return rc;
  CGD_CHECK_ARG(ld_dy % 8 == 0 && ldx % 8 == 0 && ld_dx % 8 == 0 && op.p[0] && op.p[1] && op.p[2] && op.p[6] && op.p[7],
                "gn_bwd_apply: bad args");
  const GnGeom g = gn_geom((int)C);
  CGD_CUDA(launch_pdl(gn_bwd_apply_kernel, dim3(gn_apply_chunks(HW, N, g.PP), (unsigned)N), dim3(g.threads), 0, st, 
      (const __half*)op.p[0], (const __half*)op.p[1], (const float*)op.p[2], (const float*)op.p[3], (const float*)op.p[4],
      (const float*)op.p[5], (const float*)op.p[6], (__half*)op.p[7], (int)HW, (int)C, ld_dy, ldx, ld_dx, op.flags & 1,
      (op.flags & 2) ? 1 : 0));
  CGD_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, row held in registers (w <= 2048), exact two-pass statistics.
constexpr int LN_MAXV = 8;  // 8 vectors of 8 halves per lane -> w <= 2048

__global__ void ln_fwd_kernel(const __half* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                              __half* __restrict__ y, float* __restrict__ stats, int rows, int w, int64_t ldx, int64_t ldy, float eps) {
  pdl_wait();
  pdl_launch_dependents();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int nv = w / 8;
  float v[LN_MAXV][8];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < LN_MAXV; ++k) {
    const int vi = lane + k * 32;
    if (vi < nv) {
      unpack8(ld8(x + (int64_t)row * ldx + vi * 8), v[k]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[k][j];
    }
  }
  const float mean = warp_sum(s) / (float)w;
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < LN_MAXV; ++k) {
    const int vi = lane + k * 32;
    if (vi < nv) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[k][j] - mean;
        q = fmaf(d, d, q);
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)w + eps);
  if (lane == 0 && stats) {
    stats[(int64_t)row * 2] = mean;
    stats[(int64_t)row * 2 + 1] = rstd;
  }
#pragma unroll
  for (int k = 0; k < LN_MAXV; ++k) {
    const int vi = lane + k * 32;
    if (vi < nv) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = fmaf((v[k][j] - mean) * rstd, gamma[vi * 8 + j], beta[vi * 8 + j]);
      st8(y + (int64_t)row * ldy + vi * 8, pack8(o));
    }
  }
}

__global__ void ln_bwd_kernel(const __half* __restrict__ dy, const __half* __restrict__ x, const float* __restrict__ gamma,
                              const float* __restrict__ stats, __half* __restrict__ dx, int rows, int w, int64_t ld_dy, int64_t ldx,
                              int64_t ld_dx, int accumulate) {
  pdl_wait();
  pdl_launch_dependents();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int nv = w / 8;
  const float mean = stats[(int64_t)row * 2], rstd = stats[(int64_t)row * 2 + 1];
  float xh[LN_MAXV][8], dh[LN_MAXV][8];
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int k = 0; k < LN_MAXV; ++k) {
    const int vi = lane + k * 32;
    if (vi < nv) {
      float a[8], d[8];
      unpack8(ld8(x + (int64_t)row * ldx + vi * 8), a);
      unpack8(ld8(dy + (int64_t)row * ld_dy + vi * 8), d);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        xh[k][j] = (a[j] - mean) * rstd;
        dh[k][j] = d[j] * gamma[vi * 8 + j];
        s1 += dh[k][j];
        s2 = fmaf(dh[k][j], xh[k][j], s2);
      }
    }
  }
  s1 = warp_sum(s1) / (float)w;
  s2 = warp_sum(s2) / (float)w;
#pragma unroll
  for (int k = 0; k < LN_MAXV; ++k) {
    const int vi = lane + k * 32;
    if (vi < nv) {
      float o[8];
      if (accumulate) unpack8(ld8(dx + (int64_t)row * ld_dx + vi * 8), o);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float r = rstd * (dh[k][j] - s1 - xh[k][j] * s2);
        o[j] = accumulate ? o[j] + r : r;
      }
      st8(dx + (int64_t)row * ld_dx + vi * 8, pack8(o));
    }
  }
}

int launch_ln_fwd(const CgdOp& op, cudaStream_t st) {
  const int64_t rows = op.i[0], w = op.i[1], ldx = op.i[2], ldy = op.i[3];
  CGD_CHECK_ARG(rows > 0 && w % 8 == 0 && w <= 8 * 32 * LN_MAXV && ldx % 8 == 0 && ldy % 8 == 0, "layernorm: unsupported shape rows=%lld w=%lld",
                (long long)rows, (long long)w);
  CGD_CHECK_ARG(op.p[0] && op.p[1] && op.p[2] && op.p[3], "layernorm: null pointer");
  CGD_CUDA(launch_pdl(ln_fwd_kernel, dim3((unsigned)ceil_div(rows, 8)), dim3(256), 0, st, (const __half*)op.p[0], (const float*)op.p[1], (const float*)op.p[2],
                                                           (__half*)op.p[3], (float*)op.p[4], (int)rows, (int)w, ldx, ldy, op.f[0]));
  CGD_LAUNCH_CHECK();
  return 0;
}
int launch_ln_bwd(const CgdOp& op, cudaStream_t st) {
  const int64_t rows = op.i[0], w = op.i[1], ld_dy = op.i[2], ldx = op.i[3], ld_dx = op.i[4];
  CGD_CHECK_ARG(rows > 0 && w % 8 == 0 && w <= 8 * 32 * LN_MAXV && ld_dy % 8 == 0 && ldx % 8 == 0 && ld_dx % 8 == 0,
                "layernorm bwd: unsupported shape");
  CGD_CHECK_ARG(op.p[0] && op.p[1] && op.p[2] && op.p[3] && op.p[4], "layernorm bwd: null pointer");
  CGD_CUDA(launch_pdl(ln_bwd_kernel, dim3((unsigned)ceil_div(rows, 8)), dim3(256), 0, st, (const __half*)op.p[0], (const __half*)op.p[1], (const float*)op.p[2],
                                                           (const float*)op.p[3], (__half*)op.p[4], (int)rows, (int)w, ld_dy, ldx,
                                                           ld_dx, (op.flags & 2) ? 1 : 0));
  CGD_LAUNCH_CHECK();
  return 0;
}

}  // namespace cgd
