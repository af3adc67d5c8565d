// attention_small.cu -- single-tile softmax attention (T <= 64 keys, head dim 64), forward and backward, one CTA per
// (image, head), all five / seven products on warp-level tensor-core MMAs (mma.sync m16n8k16, fp16 operands, fp32 accumulate).
//
// Replaces [3P] CLIP nn.MultiheadAttention's core for ViT-B/32 (50 tokens) and [3P] guided-diffusion QKVAttention(Legacy) at the
// 8x8 UNet level (64 tokens) (SURVEY.md K4, K14).  Why a separate kernel: these problems are one 64x64 tile per head -- the
// wgmma conv kernel wants 128-row tiles (conv_tc.cu) and the fp32 CUDA-core flash kernels of attention.cu need three launches
// for the backward of such tiles.  Here the
// whole backward -- S, P, dP, dS, dQ, dK, dV -- is one launch; P and dS go through shared memory once (fp16, like the
// reference's fp16 attention weights) to feed the transposed products.
#include <cuda_fp16.h>

#include "attn_mma.cuh"
#include "common.cuh"
#include "ops.cuh"
#include "pdl.cuh"

namespace cgd {

struct AttnSmallArgs {
  const __half *q, *k, *v, *dout;
  __half *out, *dq, *dk, *dv;
  float* lse;
  int B, heads, T;
  int64_t qbs, qrs, qhs;  // qkv batch / row / head strides (elements)
  int64_t obs, ors, ohs;  // out / dout strides
  float scale;
};

__global__ void __launch_bounds__(128) attn_small_fwd_kernel(const AttnSmallArgs a) {
  __shared__ __align__(16) __half Qs[AS_T * AS_LD], Ks[AS_T * AS_LD], Vs[AS_T * AS_LD];
  pdl_wait();
  pdl_launch_dependents();
  const int h = blockIdx.x, b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t qoff = (int64_t)b * a.qbs + (int64_t)h * a.qhs;
  as_load_tile(Qs, a.q + qoff, a.qrs, a.T);
  as_load_tile(Ks, a.k + qoff, a.qrs, a.T);
  as_load_tile(Vs, a.v + qoff, a.qrs, a.T);
  __syncthreads();
  const int r0 = warp * 16;
  if (r0 >= a.T) return;
  float s[8][4], lse0, lse1;
  as_mm_nk(s, Qs, Ks, r0, lane);
  as_softmax(s, a.T, a.scale, lane, lse0, lse1);
  if (a.lse && (lane & 3) == 0) {
    const int ra = r0 + (lane >> 2);
    float* l = a.lse + ((int64_t)b * a.heads + h) * a.T;
    if (ra < a.T) l[ra] = lse0;
    if (ra + 8 < a.T) l[ra + 8] = lse1;
  }
  uint32_t pa[4][4];
  as_c_to_a(s, pa);
  float o[8][4];
  as_mm_reg_kn(o, pa, Vs, lane);
  as_store_c(o, a.out + (int64_t)b * a.obs + (int64_t)h * a.ohs, a.ors, r0, a.T, lane);
}

__global__ void __launch_bounds__(128) attn_small_bwd_kernel(const AttnSmallArgs a) {
  extern __shared__ __align__(16) __half as_dyn[];
  __half *Qs = as_dyn, *Ks = Qs + AS_T * AS_LD, *Vs = Ks + AS_T * AS_LD, *dOs = Vs + AS_T * AS_LD, *Ps = dOs + AS_T * AS_LD, *dSs = Ps + AS_T * AS_LD;
  pdl_wait();
  pdl_launch_dependents();
  const int h = blockIdx.x, b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t qoff = (int64_t)b * a.qbs + (int64_t)h * a.qhs;
  const int64_t ooff = (int64_t)b * a.obs + (int64_t)h * a.ohs;
  as_load_tile(Qs, a.q + qoff, a.qrs, a.T);
  as_load_tile(Ks, a.k + qoff, a.qrs, a.T);
  as_load_tile(Vs, a.v + qoff, a.qrs, a.T);
  as_load_tile(dOs, a.dout + ooff, a.ors, a.T);
  __syncthreads();
  const int r0 = warp * 16;
  {
    // ---- rows r0 .. r0+15 of the queries: P, dP, dS, dQ
    float s[8][4], dp[8][4], lse0, lse1;
    as_mm_nk(s, Qs, Ks, r0, lane);
    as_softmax(s, a.T, a.scale, lane, lse0, lse1);   // s = P (rows of padded queries are harmless: their dO rows are zero)
    as_mm_nk(dp, dOs, Vs, r0, lane);     // dP = dO V^T
    float d0 = 0.f, d1 = 0.f;            // delta = rowsum(P * dP) (= rowsum(dO * O))
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      d0 += s[j][0] * dp[j][0] + s[j][1] * dp[j][1];
      d1 += s[j][2] * dp[j][2] + s[j][3] * dp[j][3];
    }
    d0 += __shfl_xor_sync(0xffffffffu, d0, 1);
    d0 += __shfl_xor_sync(0xffffffffu, d0, 2);
    d1 += __shfl_xor_sync(0xffffffffu, d1, 1);
    d1 += __shfl_xor_sync(0xffffffffu, d1, 2);
#pragma unroll
    for (int j = 0; j < 8; ++j) {  // dp <- dS = P * (dP - delta) * scale
      dp[j][0] = s[j][0] * (dp[j][0] - d0) * a.scale;
      dp[j][1] = s[j][1] * (dp[j][1] - d0) * a.scale;
      dp[j][2] = s[j][2] * (dp[j][2] - d1) * a.scale;
      dp[j][3] = s[j][3] * (dp[j][3] - d1) * a.scale;
    }
    // P and dS to shared memory (fp16, [q][key]) for the transposed products
    const int ra = r0 + (lane >> 2), cb = (lane & 3) * 2;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<__half2*>(Ps + ra * AS_LD + j * 8 + cb) = __floats2half2_rn(s[j][0], s[j][1]);
      *reinterpret_cast<__half2*>(Ps + (ra + 8) * AS_LD + j * 8 + cb) = __floats2half2_rn(s[j][2], s[j][3]);
      *reinterpret_cast<__half2*>(dSs + ra * AS_LD + j * 8 + cb) = __floats2half2_rn(dp[j][0], dp[j][1]);
      *reinterpret_cast<__half2*>(dSs + (ra + 8) * AS_LD + j * 8 + cb) = __floats2half2_rn(dp[j][2], dp[j][3]);
    }
    uint32_t dsa[4][4];
    as_c_to_a(dp, dsa);
    float dq[8][4];
    as_mm_reg_kn(dq, dsa, Ks, lane);     // dQ = dS K
    as_store_c(dq, a.dq + qoff, a.qrs, r0, a.T, lane);
  }
  __syncthreads();
  {
    // ---- rows r0 .. r0+15 of the keys: dV = P^T dO, dK = dS^T Q
    float acc[8][4];
    as_mm_t_kn(acc, Ps, dOs, r0, lane);
    as_store_c(acc, a.dv + qoff, a.qrs, r0, a.T, lane);
    as_mm_t_kn(acc, dSs, Qs, r0, lane);
    as_store_c(acc, a.dk + qoff, a.qrs, r0, a.T, lane);
  }
}

int attn_small_supported(int64_t T) { return T >= 1 && T <= AS_T; }

static int attn_small_args(const CgdOp& op, AttnSmallArgs& a, bool bwd) {
  a.B = (int)op.i[0]; a.heads = (int)op.i[1]; a.T = (int)op.i[2];
  a.qbs = op.i[4]; a.qrs = op.i[5]; a.qhs = op.i[6]; a.obs = op.i[7]; a.ors = op.i[8]; a.ohs = op.i[9];
  a.scale = op.f[0];
  a.q = (const __half*)op.p[0]; a.k = (const __half*)op.p[1]; a.v = (const __half*)op.p[2];
  if (!bwd) {
    a.out = (__half*)op.p[3];
    a.lse = (float*)op.p[4];
  } else {
    a.dout = (const __half*)op.p[4];
    a.dq = (__half*)op.p[6]; a.dk = (__half*)op.p[7]; a.dv = (__half*)op.p[8];
  }
  return 0;
}

int launch_attn_small_fwd(const CgdOp& op, cudaStream_t st) {
  AttnSmallArgs a{};
  attn_small_args(op, a, false);
  CGD_CUDA(launch_pdl(attn_small_fwd_kernel, dim3(a.heads, a.B), dim3(128), 0, st, a));
  return 0;
}
int launch_attn_small_bwd(const CgdOp& op, cudaStream_t st) {
  AttnSmallArgs a{};
  attn_small_args(op, a, true);
  constexpr int smem = 6 * AS_T * AS_LD * (int)sizeof(__half);
  static DeviceOnce set;
  if (set.needed()) {
    CGD_CUDA(cudaFuncSetAttribute(attn_small_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    set.mark();
  }
  CGD_CUDA(launch_pdl(attn_small_bwd_kernel, dim3(a.heads, a.B), dim3(128), smem, st, a));
  return 0;
}

}  // namespace cgd
