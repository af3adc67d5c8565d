// attention_mma.cu -- flash attention (any sequence length, head dim 64), forward and backward, on warp-level tensor-core
// MMAs (mma.sync m16n8k16, fp16 operands, fp32 accumulate / softmax), K/V (or Q/dO) tiles double-buffered with cp.async.
//
// Replaces [3P] guided-diffusion QKVAttention(Legacy) at the 32x32 / 16x16 UNet levels (T = 1024 / 256) and [3P] CLIP
// nn.MultiheadAttention's core for ViT-B/16, L/14 (T = 197, 257) (SURVEY.md K4, K14).  Nothing T x T touches HBM.
// The alternative, batched tensor-core GEMMs (plan.tc_attention: S and P materialised, K = 64 per GEMM, explicit transposes, row
// softmax kernels), needs ~110 launches per step and a T x T round trip through memory.  Structure of the backward (as in attention.cu): delta = rowsum(dO * O); one kernel per key
// tile accumulates dK, dV over the query tiles, one CTA per query tile accumulates dQ over the key tiles (same launch).
#include <cuda_fp16.h>

#include "attn_mma.cuh"
#include "common.cuh"
#include "ops.cuh"
#include "pdl.cuh"

namespace cgd {

struct AttnMmaArgs {
  const __half *q, *k, *v, *o, *dout;
  __half *out, *dq, *dk, *dv;
  float *lse, *delta;
  int B, heads, T;
  int64_t qbs, qrs, qhs;  // qkv batch / row / head strides (elements)
  int64_t obs, ors, ohs;  // out / dout strides
  float scale;
};

constexpr int AM_TILE = AS_T * AS_LD;  // halfs per shared tile

// 64 x 64 fp16 tile, rows r0 .. r0+63 of a [T, 64] matrix, global -> shared with cp.async (rows >= T zero-filled)
__device__ __forceinline__ void am_load_async(__half* s, const __half* g, int64_t rs, int r0, int T) {
  for (int v = threadIdx.x; v < AS_T * 8; v += blockDim.x) {
    const int r = v >> 3, c = (v & 7) * 8;
    const int row = r0 + r;
    const __half* src = g + (int64_t)min(row, T - 1) * rs + c;
    const uint32_t sz = row < T ? 16u : 0u;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(as_smem(s + r * AS_LD + c)), "l"(src), "r"(sz) : "memory");
  }
}
__device__ __forceinline__ void am_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void am_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ------------------------------------------------------------------------------------------------ forward
__global__ void __launch_bounds__(128) attn_mma_fwd_kernel(const AttnMmaArgs a) {
  __shared__ __align__(16) __half sm[5 * AM_TILE];  // Q | K0 | K1 | V0 | V1
  __half* Qs = sm;
  __half* Ks = sm + AM_TILE;
  __half* Vs = sm + 3 * AM_TILE;
  pdl_wait();
  pdl_launch_dependents();
  const int q0 = blockIdx.x * AS_T, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t qoff = (int64_t)b * a.qbs + (int64_t)h * a.qhs;
  const int n_kt = (a.T + AS_T - 1) / AS_T;
  am_load_async(Qs, a.q + qoff, a.qrs, q0, a.T);
  am_load_async(Ks, a.k + qoff, a.qrs, 0, a.T);
  am_load_async(Vs, a.v + qoff, a.qrs, 0, a.T);
  am_commit();
  const int r0 = warp * 16;
  const int cb = (lane & 3) * 2;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float o[8][4];
  as_zero(o);
  for (int kt = 0; kt < n_kt; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < n_kt) {  // prefetch the next K / V tile into the other buffer (its last readers finished at the barrier below)
      am_load_async(Ks + (buf ^ 1) * AM_TILE, a.k + qoff, a.qrs, (kt + 1) * AS_T, a.T);
      am_load_async(Vs + (buf ^ 1) * AM_TILE, a.v + qoff, a.qrs, (kt + 1) * AS_T, a.T);
      am_commit();
      am_wait<1>();
    } else {
      am_wait<0>();
    }
    __syncthreads();
    float s[8][4];
    as_mm_nk(s, Qs, Ks + buf * AM_TILE, r0, lane);
    const int k0 = kt * AS_T;
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const bool ok = k0 + j * 8 + cb + e < a.T;
        s[j][e] = ok ? s[j][e] * a.scale : -INFINITY;
        s[j][2 + e] = ok ? s[j][2 + e] * a.scale : -INFINITY;
        mx0 = fmaxf(mx0, s[j][e]);
        mx1 = fmaxf(mx1, s[j][2 + e]);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);  // finite: every key tile holds at least one valid key
    const float al0 = __expf(m0 - mn0), al1 = __expf(m1 - mn1);
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        s[j][e] = __expf(s[j][e] - mn0);
        s[j][2 + e] = __expf(s[j][2 + e] - mn1);
        rs0 += s[j][e];
        rs1 += s[j][2 + e];
      }
    }
    rs0 += __shfl_xor_sync(0xffffffffu, rs0, 1);
    rs0 += __shfl_xor_sync(0xffffffffu, rs0, 2);
    rs1 += __shfl_xor_sync(0xffffffffu, rs1, 1);
    rs1 += __shfl_xor_sync(0xffffffffu, rs1, 2);
    l0 = l0 * al0 + rs0;
    l1 = l1 * al1 + rs1;
    m0 = mn0;
    m1 = mn1;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[j][0] *= al0;
      o[j][1] *= al0;
      o[j][2] *= al1;
      o[j][3] *= al1;
    }
    uint32_t pa[4][4];
    as_c_to_a(s, pa);
    as_mm_reg_kn<false>(o, pa, Vs + buf * AM_TILE, lane);
    __syncthreads();  // all warps are done with buffer `buf` before the next iteration's prefetch overwrites it
  }
  const float i0 = 1.f / l0, i1 = 1.f / l1;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    o[j][0] *= i0;
    o[j][1] *= i0;
    o[j][2] *= i1;
    o[j][3] *= i1;
  }
  as_store_c(o, a.out + (int64_t)b * a.obs + (int64_t)h * a.ohs + (int64_t)q0 * a.ors, a.ors, r0, a.T - q0, lane);
  if ((lane & 3) == 0) {
    const int ra = q0 + r0 + (lane >> 2);
    float* lse = a.lse + ((int64_t)b * a.heads + h) * a.T;
    if (ra < a.T) lse[ra] = m0 + __logf(l0);
    if (ra + 8 < a.T) lse[ra + 8] = m1 + __logf(l1);
  }
}

// delta[b,h,q] = sum_d dO[q,d] * O[q,d]; one warp per row
__global__ void attn_mma_delta_kernel(const AttnMmaArgs a) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int64_t total = (int64_t)a.B * a.heads * a.T;
  if (row >= total) return;
  const int q = (int)(row % a.T);
  const int h = (int)((row / a.T) % a.heads);
  const int b = (int)(row / ((int64_t)a.T * a.heads));
  const int64_t off = (int64_t)b * a.obs + (int64_t)q * a.ors + (int64_t)h * a.ohs + lane * 2;
  const float2 x = __half22float2(*reinterpret_cast<const __half2*>(a.o + off));
  const float2 y = __half22float2(*reinterpret_cast<const __half2*>(a.dout + off));
  const float s = warp_sum(x.x * y.x + x.y * y.y);
  if (lane == 0) a.delta[row] = s;
}

// P and dS fragments of the warp's 16 query rows against 64 keys: s <- P = exp(S * scale - lse), dp <- dS = P * (dP - delta) * scale
__device__ __forceinline__ void am_p_ds(float (&s)[8][4], float (&dp)[8][4], float ls0, float ls1, float de0, float de1, bool q0ok, bool q1ok,
                                        int k0, int T, float scale, int lane) {
  const int cb = (lane & 3) * 2;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const bool kok = k0 + j * 8 + cb + e < T;
      const float p0 = (kok && q0ok) ? __expf(s[j][e] * scale - ls0) : 0.f;
      const float p1 = (kok && q1ok) ? __expf(s[j][2 + e] * scale - ls1) : 0.f;
      s[j][e] = p0;
      s[j][2 + e] = p1;
      dp[j][e] = p0 * (dp[j][e] - de0) * scale;
      dp[j][2 + e] = p1 * (dp[j][2 + e] - de1) * scale;
    }
  }
}

// ------------------------------------------------------------------------------------------------ backward: dK, dV per key tile
__device__ __forceinline__ void attn_mma_bwd_dkv_body(const AttnMmaArgs& a, __half* am_dyn, int tile_x) {
  // shared: K | V | Q0 | Q1 | dO0 | dO1 | P | dS
  __half* Ks = am_dyn;
  __half* Vs = am_dyn + AM_TILE;
  __half* Qs = am_dyn + 2 * AM_TILE;
  __half* dOs = am_dyn + 4 * AM_TILE;
  __half* Ps = am_dyn + 6 * AM_TILE;
  __half* dSs = am_dyn + 7 * AM_TILE;
  const int k0 = tile_x * AS_T, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t qoff = (int64_t)b * a.qbs + (int64_t)h * a.qhs;
  const int64_t ooff = (int64_t)b * a.obs + (int64_t)h * a.ohs;
  const float* lse = a.lse + ((int64_t)b * a.heads + h) * a.T;
  const float* delta = a.delta + ((int64_t)b * a.heads + h) * a.T;
  const int n_qt = (a.T + AS_T - 1) / AS_T;
  am_load_async(Ks, a.k + qoff, a.qrs, k0, a.T);
  am_load_async(Vs, a.v + qoff, a.qrs, k0, a.T);
  am_load_async(Qs, a.q + qoff, a.qrs, 0, a.T);
  am_load_async(dOs, a.dout + ooff, a.ors, 0, a.T);
  am_commit();
  const int r0 = warp * 16;
  float dk[8][4], dv[8][4];
  as_zero(dk);
  as_zero(dv);
  for (int qt = 0; qt < n_qt; ++qt) {
    const int buf = qt & 1;
    if (qt + 1 < n_qt) {
      am_load_async(Qs + (buf ^ 1) * AM_TILE, a.q + qoff, a.qrs, (qt + 1) * AS_T, a.T);
      am_load_async(dOs + (buf ^ 1) * AM_TILE, a.dout + ooff, a.ors, (qt + 1) * AS_T, a.T);
      am_commit();
      am_wait<1>();
    } else {
      am_wait<0>();
    }
    __syncthreads();
    const __half* Qb = Qs + buf * AM_TILE;
    const __half* dOb = dOs + buf * AM_TILE;
    {
      float s[8][4], dp[8][4];
      as_mm_nk(s, Qb, Ks, r0, lane);    // S rows = this warp's 16 queries of the tile
      as_mm_nk(dp, dOb, Vs, r0, lane);  // dP = dO V^T
      const int qa = qt * AS_T + r0 + (lane >> 2), qb = qa + 8;
      const bool okA = qa < a.T, okB = qb < a.T;
      am_p_ds(s, dp, okA ? lse[qa] : 0.f, okB ? lse[qb] : 0.f, okA ? delta[qa] : 0.f, okB ? delta[qb] : 0.f, okA, okB, k0, a.T, a.scale, lane);
      const int ra = r0 + (lane >> 2), cb = (lane & 3) * 2;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        *reinterpret_cast<__half2*>(Ps + ra * AS_LD + j * 8 + cb) = __floats2half2_rn(s[j][0], s[j][1]);
        *reinterpret_cast<__half2*>(Ps + (ra + 8) * AS_LD + j * 8 + cb) = __floats2half2_rn(s[j][2], s[j][3]);
        *reinterpret_cast<__half2*>(dSs + ra * AS_LD + j * 8 + cb) = __floats2half2_rn(dp[j][0], dp[j][1]);
        *reinterpret_cast<__half2*>(dSs + (ra + 8) * AS_LD + j * 8 + cb) = __floats2half2_rn(dp[j][2], dp[j][3]);
      }
    }
    __syncthreads();
    as_mm_t_kn<false>(dv, Ps, dOb, r0, lane);  // dV[keys r0..] += P^T dO
    as_mm_t_kn<false>(dk, dSs, Qb, r0, lane);  // dK[keys r0..] += dS^T Q
    __syncthreads();  // P / dS and buffer `buf` are free again
  }
  as_store_c(dk, a.dk + qoff + (int64_t)k0 * a.qrs, a.qrs, r0, a.T - k0, lane);
  as_store_c(dv, a.dv + qoff + (int64_t)k0 * a.qrs, a.qrs, r0, a.T - k0, lane);
}

// ------------------------------------------------------------------------------------------------ backward: dQ per query tile
__device__ __forceinline__ void attn_mma_bwd_dq_body(const AttnMmaArgs& a, __half* am_dyn, int tile_x) {
  // shared: Q | dO | K0 | K1 | V0 | V1
  __half* Qs = am_dyn;
  __half* dOs = am_dyn + AM_TILE;
  __half* Ks = am_dyn + 2 * AM_TILE;
  __half* Vs = am_dyn + 4 * AM_TILE;
  const int q0 = tile_x * AS_T, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t qoff = (int64_t)b * a.qbs + (int64_t)h * a.qhs;
  const int64_t ooff = (int64_t)b * a.obs + (int64_t)h * a.ohs;
  const int n_kt = (a.T + AS_T - 1) / AS_T;
  am_load_async(Qs, a.q + qoff, a.qrs, q0, a.T);
  am_load_async(dOs, a.dout + ooff, a.ors, q0, a.T);
  am_load_async(Ks, a.k + qoff, a.qrs, 0, a.T);
  am_load_async(Vs, a.v + qoff, a.qrs, 0, a.T);
  am_commit();
  const int r0 = warp * 16;
  const int qa = q0 + r0 + (lane >> 2), qb = qa + 8;
  const bool okA = qa < a.T, okB = qb < a.T;
  const float* lse = a.lse + ((int64_t)b * a.heads + h) * a.T;
  const float* delta = a.delta + ((int64_t)b * a.heads + h) * a.T;
  const float lsA = okA ? lse[qa] : 0.f, lsB = okB ? lse[qb] : 0.f, deA = okA ? delta[qa] : 0.f, deB = okB ? delta[qb] : 0.f;
  float dq[8][4];
  as_zero(dq);
  for (int kt = 0; kt < n_kt; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < n_kt) {
      am_load_async(Ks + (buf ^ 1) * AM_TILE, a.k + qoff, a.qrs, (kt + 1) * AS_T, a.T);
      am_load_async(Vs + (buf ^ 1) * AM_TILE, a.v + qoff, a.qrs, (kt + 1) * AS_T, a.T);
      am_commit();
      am_wait<1>();
    } else {
      am_wait<0>();
    }
    __syncthreads();
    float s[8][4], dp[8][4];
    as_mm_nk(s, Qs, Ks + buf * AM_TILE, r0, lane);
    as_mm_nk(dp, dOs, Vs + buf * AM_TILE, r0, lane);
    am_p_ds(s, dp, lsA, lsB, deA, deB, okA, okB, kt * AS_T, a.T, a.scale, lane);
    uint32_t dsa[4][4];
    as_c_to_a(dp, dsa);
    as_mm_reg_kn<false>(dq, dsa, Ks + buf * AM_TILE, lane);  // dQ += dS K
    __syncthreads();
  }
  as_store_c(dq, a.dq + qoff + (int64_t)q0 * a.qrs, a.qrs, r0, a.T - q0, lane);
}

// One launch for both: blocks [0, tiles) accumulate dK / dV of a key tile, blocks [tiles, 2 * tiles) dQ of a query tile.  The
// two halves are independent and each runs four warps per CTA, so side by side they fill the SMs twice as well as back to back.
__global__ void __launch_bounds__(128) attn_mma_bwd_kernel(const AttnMmaArgs a, int tiles) {
  extern __shared__ __align__(16) __half am_dyn[];
  pdl_wait();
  pdl_launch_dependents();
  if ((int)blockIdx.x < tiles) attn_mma_bwd_dkv_body(a, am_dyn, (int)blockIdx.x);
  else attn_mma_bwd_dq_body(a, am_dyn, (int)blockIdx.x - tiles);
}

// ------------------------------------------------------------------------------------------------ host
static void am_args(const CgdOp& op, AttnMmaArgs& a, bool bwd) {
  a.B = (int)op.i[0]; a.heads = (int)op.i[1]; a.T = (int)op.i[2];
  a.qbs = op.i[4]; a.qrs = op.i[5]; a.qhs = op.i[6]; a.obs = op.i[7]; a.ors = op.i[8]; a.ohs = op.i[9];
  a.scale = op.f[0];
  a.q = (const __half*)op.p[0]; a.k = (const __half*)op.p[1]; a.v = (const __half*)op.p[2];
  if (!bwd) {
    a.out = (__half*)op.p[3]; a.lse = (float*)op.p[4];
  } else {
    a.o = (const __half*)op.p[3]; a.dout = (const __half*)op.p[4]; a.lse = (float*)op.p[5];
    a.dq = (__half*)op.p[6]; a.dk = (__half*)op.p[7]; a.dv = (__half*)op.p[8]; a.delta = (float*)op.p[9];
  }
}

int launch_attn_mma_fwd(const CgdOp& op, cudaStream_t st) {
  AttnMmaArgs a{};
  am_args(op, a, false);
  CGD_CUDA(launch_pdl(attn_mma_fwd_kernel, dim3((unsigned)ceil_div(a.T, AS_T), a.heads, a.B), dim3(128), 0, st, a));
  return 0;
}

int launch_attn_mma_bwd(const CgdOp& op, cudaStream_t st) {
  AttnMmaArgs a{};
  am_args(op, a, true);
  constexpr int smem = 8 * AM_TILE * (int)sizeof(__half);  // the dK / dV half needs 8 tiles, the dQ half 6
  static DeviceOnce set;
  if (set.needed()) {
    CGD_CUDA(cudaFuncSetAttribute(attn_mma_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    set.mark();
  }
  const int64_t rows = (int64_t)a.B * a.heads * a.T;
  CGD_CUDA(launch_pdl(attn_mma_delta_kernel, dim3((unsigned)ceil_div(rows, 8)), dim3(256), 0, st, a));
  const int tiles = (int)ceil_div(a.T, AS_T);
  CGD_CUDA(launch_pdl(attn_mma_bwd_kernel, dim3((unsigned)(2 * tiles), a.heads, a.B), dim3(128), smem, st, a, tiles));
  return 0;
}

}  // namespace cgd
