// norm_fused.cu -- single-launch GroupNorm(32) (+SiLU, +scale/shift) forward and input-gradient for activations whose
// per-(image, group) slab fits the registers of one thread-block cluster.
//
// Why: the two-pass kernels of norm.cu cost two launches per layer *independently of size* at the 8x8 .. 64x64 levels of the
// UNet -- a chain of load -> block reduce -> partials -> fence -> atomic -> last-block fold -> second launch -> reload -- while the data is
// 0.1 .. 8 MB.  Here one cluster of CS CTAs owns `gpc` consecutive groups of one image: the slab is read ONCE into
// registers, statistics are exact two-pass (mean, then sum (x - mean)^2) and are exchanged between the CTAs of the cluster
// through distributed shared memory in a fixed order (deterministic), then the slab is normalised from registers and written.
// HBM traffic: 4 B / element forward (two-pass kernels: 6), 6 - 8 B / element backward (10 - 12).
//
// Replaces [3P] guided-diffusion GroupNorm32 + SiLU + scale-shift (SURVEY.md K5, K6) for C % 256 == 0.
#include <cuda.h>

#include "common.cuh"
#include "ops.cuh"
#include "pdl.cuh"

namespace cgd {

constexpr int kGnfThreads = 512;

__device__ __forceinline__ uint32_t gnf_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void gnf_cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void gnf_cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ float2 gnf_ld_remote(const float2* p, uint32_t cta) {
  uint32_t a;
  float2 v;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(gnf_smem_u32(p)), "r"(cta));
  asm volatile("ld.shared::cluster.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a) : "memory");
  return v;
}

struct GnfGeom {
  int cpg, gpc, vpp, PP;  // channels per group, groups per CTA, 16-byte vectors per pixel per CTA, pixel lanes
};
__host__ __device__ inline GnfGeom gnf_geom(int C) {
  GnfGeom g;
  g.cpg = C / 32;
  g.gpc = g.cpg < 16 ? 16 / g.cpg : 1;  // >= 32 contiguous bytes per pixel per CTA
  g.vpp = g.gpc * g.cpg / 8;
  g.PP = kGnfThreads / g.vpp;
  return g;
}

// Deterministic reduction of one (a, b) pair per thread into per-group sums of this CTA, then over the cluster.
// `red` = kGnfThreads float2, `cl` = this phase's exchange slot [2 groups].  Returns the cluster-wide sums of group `gi`.
__device__ __forceinline__ float2 gnf_reduce(float a, float b, bool active, int gi, const GnfGeom& g, int CS, float2* red, float2* cl,
                                             float2* bcast) {
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  red[t] = active ? make_float2(a, b) : make_float2(0.f, 0.f);
  __syncthreads();
  if (warp < g.gpc) {
    float sa = 0.f, sb = 0.f;
    const int vpg = g.cpg / 8;  // vectors per group
    for (int i = lane; i < g.PP * g.vpp; i += 32) {
      if ((i % g.vpp) / vpg == warp) {
        const float2 v = red[i];
        sa += v.x;
        sb += v.y;
      }
    }
    sa = warp_sum(sa);
    sb = warp_sum(sb);
    if (lane == 0) cl[warp] = make_float2(sa, sb);
  }
  // publish to the cluster, then every CTA folds the CS partials in rank order (bit-identical in all CTAs)
  gnf_cluster_arrive();
  gnf_cluster_wait();
  if (t < g.gpc) {
    float sa = 0.f, sb = 0.f;
    for (int r = 0; r < CS; ++r) {
      const float2 v = gnf_ld_remote(&cl[t], (uint32_t)r);
      sa += v.x;
      sb += v.y;
    }
    bcast[t] = make_float2(sa, sb);
  }
  __syncthreads();
  return bcast[gi];
}

// ------------------------------------------------------------------------------------------------ forward
template <int MAXV>
__global__ void __launch_bounds__(kGnfThreads, 1)
gn_fwd_fused_kernel(const __half* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                    const float* __restrict__ emb, __half* __restrict__ y, float* __restrict__ stats, int HW, int C, int64_t ldx,
                    int64_t ldy, int CS, float eps, int silu) {
  __shared__ float2 red[kGnfThreads];
  __shared__ float2 cl[2][2];
  __shared__ float2 bcast[2][2];
  const GnfGeom g = gnf_geom(C);
  const int n = blockIdx.y, crank = blockIdx.x % CS, gblk = blockIdx.x / CS;
  const int t = threadIdx.x;
  const bool active = t < g.PP * g.vpp;
  const int v = t % g.vpp, pl = t / g.vpp;
  const int gi = (v * 8) / g.cpg;
  const int ch = gblk * g.gpc * g.cpg + v * 8;
  const int HWc = (HW + CS - 1) / CS;
  const int p0 = crank * HWc, p1 = min(HW, p0 + HWc);

  // parameters do not depend on the previous kernel: fetch them before the grid dependency resolves
  float G[8], Bc[8];
  if (active) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      G[j] = gamma[ch + j];
      Bc[j] = beta[ch + j];
    }
  }
  pdl_wait();
  pdl_launch_dependents();
  if (active) {  // G <- gamma * (1 + scale), Bc <- beta * (1 + scale) + shift; the statistics enter after the reductions
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sc1 = emb ? 1.f + emb[(int64_t)n * 2 * C + ch + j] : 1.f;
      const float sh = emb ? emb[(int64_t)n * 2 * C + C + ch + j] : 0.f;
      G[j] *= sc1;
      Bc[j] = fmaf(Bc[j], sc1, sh);
    }
  }
  const __half* xb = x + (int64_t)n * HW * ldx + ch;
  half8 raw[MAXV];
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int p = p0 + pl + k * g.PP;
    if (active && p < p1) raw[k] = ld8(xb + (int64_t)p * ldx);
  }
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int p = p0 + pl + k * g.PP;
    if (active && p < p1) {
      float f[8];
      unpack8(raw[k], f);
      s += ((f[0] + f[1]) + (f[2] + f[3])) + ((f[4] + f[5]) + (f[6] + f[7]));
    }
  }
  const float inv_m = 1.f / ((float)g.cpg * (float)HW);
  const float mean = gnf_reduce(s, 0.f, active, gi, g, CS, red, cl[0], bcast[0]).x * inv_m;
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int p = p0 + pl + k * g.PP;
    if (active && p < p1) {
      float f[8];
      unpack8(raw[k], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = f[j] - mean;
        q = fmaf(d, d, q);
      }
    }
  }
  const float var = gnf_reduce(q, 0.f, active, gi, g, CS, red, cl[1], bcast[1]).x * inv_m;
  gnf_cluster_arrive();  // this CTA has finished reading its peers' shared memory (waited for before exit)
  const float rstd = rsqrtf(var + eps);
  if (crank == 0 && active && pl == 0 && (v * 8) % g.cpg == 0) {
    const int grp = gblk * g.gpc + gi;
    stats[((int64_t)n * 32 + grp) * 2 + 0] = mean;
    stats[((int64_t)n * 32 + grp) * 2 + 1] = rstd;
  }
  if (active) {
    float A[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      A[j] = rstd * G[j];
      Bc[j] = fmaf(-mean, A[j], Bc[j]);
    }
    __half* yb = y + (int64_t)n * HW * ldy + ch;
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
      const int p = p0 + pl + k * g.PP;
      if (p < p1) {
        float f[8];
        unpack8(raw[k], f);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float u = fmaf(f[j], A[j], Bc[j]);
          f[j] = silu ? silu_f(u) : u;
        }
        st8(yb + (int64_t)p * ldy, pack8(f));
      }
    }
  }
  gnf_cluster_wait();
}

// ------------------------------------------------------------------------------------------------ backward
template <int MAXV>
__global__ void __launch_bounds__(kGnfThreads, 1)
gn_bwd_fused_kernel(const __half* __restrict__ dy, const __half* __restrict__ x, const float* __restrict__ stats,
                    const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ emb,
                    __half* __restrict__ dx, int HW, int C, int64_t ld_dy, int64_t ldx, int64_t ld_dx, int CS, int silu,
                    int accumulate) {
  __shared__ float2 red[kGnfThreads];
  __shared__ float2 cl[2];
  __shared__ float2 bcast[2];
  const GnfGeom g = gnf_geom(C);
  const int n = blockIdx.y, crank = blockIdx.x % CS, gblk = blockIdx.x / CS;
  const int t = threadIdx.x;
  const bool active = t < g.PP * g.vpp;
  const int v = t % g.vpp, pl = t / g.vpp;
  const int gi = (v * 8) / g.cpg;
  const int ch = gblk * g.gpc * g.cpg + v * 8;
  const int HWc = (HW + CS - 1) / CS;
  const int p0 = crank * HWc, p1 = min(HW, p0 + HWc);

  float G[8], Bc[8];
  if (active) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      G[j] = gamma[ch + j];
      Bc[j] = beta[ch + j];
    }
  }
  pdl_wait();
  pdl_launch_dependents();
  float mu = 0.f, rs = 0.f;
  if (active) {
    const int grp = gblk * g.gpc + gi;
    mu = stats[((int64_t)n * 32 + grp) * 2];
    rs = stats[((int64_t)n * 32 + grp) * 2 + 1];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sc1 = emb ? 1.f + emb[(int64_t)n * 2 * C + ch + j] : 1.f;
      const float sh = emb ? emb[(int64_t)n * 2 * C + C + ch + j] : 0.f;
      const float ga = G[j];
      G[j] = ga * sc1;                               // d v / d xhat
      Bc[j] = (Bc[j] - mu * rs * ga) * sc1 + sh;     // v = x * (rs * G) + Bc
    }
  }
  const __half* xb = x + (int64_t)n * HW * ldx + ch;
  const __half* db = dy + (int64_t)n * HW * ld_dy + ch;
  half8 rx[MAXV], rd[MAXV];
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int p = p0 + pl + k * g.PP;
    if (active && p < p1) {
      rx[k] = ld8(xb + (int64_t)p * ldx);
      rd[k] = ld8(db + (int64_t)p * ld_dy);
    }
  }
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int p = p0 + pl + k * g.PP;
    if (active && p < p1) {
      float a[8], d[8];
      unpack8(rx[k], a);
      unpack8(rd[k], d);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float dv = d[j];
        if (silu) dv *= silu_grad_f(fmaf(a[j], rs * G[j], Bc[j]));
        const float dxh = dv * G[j];
        const float xh = (a[j] - mu) * rs;
        s1 += dxh;
        s2 = fmaf(dxh, xh, s2);
      }
    }
  }
  const float inv_m = 1.f / ((float)g.cpg * (float)HW);
  const float2 tot = gnf_reduce(s1, s2, active, gi, g, CS, red, cl, bcast);
  gnf_cluster_arrive();
  const float m1 = tot.x * inv_m, m2 = tot.y * inv_m;
  if (active) {
    __half* ob = dx + (int64_t)n * HW * ld_dx + ch;
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
      const int p = p0 + pl + k * g.PP;
      if (p < p1) {
        float a[8], d[8], o[8];
        unpack8(rx[k], a);
        unpack8(rd[k], d);
        if (accumulate) unpack8(ld8(ob + (int64_t)p * ld_dx), o);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float dv = d[j];
          if (silu) dv *= silu_grad_f(fmaf(a[j], rs * G[j], Bc[j]));
          const float dxh = dv * G[j];
          const float xh = (a[j] - mu) * rs;
          const float r = rs * (dxh - m1 - xh * m2);
          o[j] = accumulate ? o[j] + r : r;
        }
        st8(ob + (int64_t)p * ld_dx, pack8(o));
      }
    }
  }
  gnf_cluster_wait();
}

// ------------------------------------------------------------------------------------------------ host
// Largest number of pixels per CTA = MAXV * PP; CS must make HW / CS fit (checked), grid = (32 / gpc) * CS x N.
static int gnf_check(const char* what, int64_t N, int64_t HW, int64_t C, int64_t CS, int maxv) {
  CGD_CHECK_ARG(N > 0 && HW > 0, "%s: bad dims", what);
  CGD_CHECK_ARG(C >= 256 && C % 256 == 0 && C <= 4096, "%s: C=%lld must be a multiple of 256 (whole 16-byte vectors per group)", what,
                (long long)C);
  CGD_CHECK_ARG(CS == 1 || CS == 2 || CS == 4 || CS == 8, "%s: cluster size %lld must be 1, 2, 4 or 8", what, (long long)CS);
  const GnfGeom g = gnf_geom((int)C);
  CGD_CHECK_ARG(ceil_div(HW, CS) <= (int64_t)maxv * g.PP, "%s: %lld pixels per CTA exceed the register slab (%d)", what,
                (long long)ceil_div(HW, CS), maxv * g.PP);
  return 0;
}

template <typename K, typename... Args>
static int gnf_launch(K kernel, dim3 grid, int CS, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(kGnfThreads);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = st;
  cudaLaunchAttribute at[2];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = (unsigned)CS;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  int na = 1;
  if (pdl_enabled()) {
    at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[1].val.programmaticStreamSerializationAllowed = 1;
    na = 2;
  }
  cfg.attrs = at;
  cfg.numAttrs = na;
  CGD_CUDA(cudaLaunchKernelEx(&cfg, kernel, args...));
  return 0;
}

int launch_gn_fwd_fused(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], HW = op.i[1], C = op.i[2], ldx = op.i[3], ldy = op.i[4], CS = op.i[5];
  if (int rc = gnf_check("gn_fwd_fused", N, HW, C, CS, 16)) return rc;
  CGD_CHECK_ARG(ldx % 8 == 0 && ldy % 8 == 0 && op.p[0] && op.p[1] && op.p[2] && op.p[4] && op.p[5], "gn_fwd_fused: bad args");
  const GnfGeom g = gnf_geom((int)C);
  const dim3 grid((unsigned)((32 / g.gpc) * CS), (unsigned)N);
  const bool small = ceil_div(HW, CS) <= 4 * g.PP;
  auto kern = small ? gn_fwd_fused_kernel<4> : gn_fwd_fused_kernel<16>;
  return gnf_launch(kern, grid, (int)CS, st, (const __half*)op.p[0], (const float*)op.p[1], (const float*)op.p[2], (const float*)op.p[3],
                    (__half*)op.p[4], (float*)op.p[5], (int)HW, (int)C, ldx, ldy, (int)CS, op.f[0], (int)(op.flags & 1));
}

int launch_gn_bwd_fused(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], HW = op.i[1], C = op.i[2], ld_dy = op.i[3], ldx = op.i[4], ld_dx = op.i[5], CS = op.i[6];
  if (int rc = gnf_check("gn_bwd_fused", N, HW, C, CS, 8)) return rc;
  CGD_CHECK_ARG(ld_dy % 8 == 0 && ldx % 8 == 0 && ld_dx % 8 == 0 && op.p[0] && op.p[1] && op.p[2] && op.p[3] && op.p[4] && op.p[6],
                "gn_bwd_fused: bad args");
  const GnfGeom g = gnf_geom((int)C);
  const dim3 grid((unsigned)((32 / g.gpc) * CS), (unsigned)N);
  const bool small = ceil_div(HW, CS) <= 2 * g.PP;
  auto kern = small ? gn_bwd_fused_kernel<2> : gn_bwd_fused_kernel<8>;
  return gnf_launch(kern, grid, (int)CS, st, (const __half*)op.p[0], (const __half*)op.p[1], (const float*)op.p[2], (const float*)op.p[3],
                    (const float*)op.p[4], (const float*)op.p[5], (__half*)op.p[6], (int)HW, (int)C, ld_dy, ldx, ld_dx, (int)CS,
                    (int)(op.flags & 1), (int)((op.flags & 2) ? 1 : 0));
}

}  // namespace cgd
