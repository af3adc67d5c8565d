// attention.cu -- multi-head softmax attention (head dim 64), forward and backward, flash-style.
//
// Replaces [3P] guided-diffusion QKVAttention / QKVAttentionLegacy (einsum -> cuBLAS bmm + ATen softmax,
// fp32 softmax) and [3P] CLIP nn.MultiheadAttention's core (SURVEY.md K4, K14): 0.5 % of the UNet FLOPs at
// 256^2 and ~1 % of ViT-B/32, so this first version is a register-tiled CUDA-core kernel (fp32 math on fp16
// operands staged through shared memory, online softmax, nothing T x T ever touches HBM).  The q/k/v
// operands are addressed by (batch, row, head) strides so both the legacy per-head [q|k|v] interleave and the
// [q..|k..|v..] order read straight out of the fused qkv GEMM output.
#include <stdlib.h>

#include "common.cuh"
#include "pdl.cuh"
#include "ops.cuh"

namespace cgd {

constexpr int AT = 64;       // tile edge (queries, keys, head dim)
constexpr int ALD = AT + 4;  // padded leading dimension (floats); 68*4 B keeps float4 alignment

struct AttnArgs {
  const __half *q, *k, *v, *o, *dout;
  __half *out, *dq, *dk, *dv;
  float *lse, *delta;
  int B, heads, T;
  int64_t qbs, qrs, qhs;  // qkv batch / row / head strides (elements)
  int64_t obs, ors, ohs;  // out strides
  float scale;
};

// 64x64 fp16 tile (rows r0.., 64 contiguous columns) -> shared fp32, row-major [r][c]
__device__ __forceinline__ void load_tile_rm(float* s, const __half* g, int64_t rs, int r0, int T) {
  for (int vid = threadIdx.x; vid < AT * 8; vid += blockDim.x) {
    const int r = vid >> 3, dv = vid & 7;
    float f[8];
    if (r0 + r < T) unpack8(ld8(g + (int64_t)(r0 + r) * rs + dv * 8), f);
    else {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = 0.f;
    }
    float4* d = reinterpret_cast<float4*>(s + r * ALD + dv * 8);
    d[0] = make_float4(f[0], f[1], f[2], f[3]);
    d[1] = make_float4(f[4], f[5], f[6], f[7]);
  }
}
// same tile -> shared fp32 transposed [c][r]
__device__ __forceinline__ void load_tile_tr(float* s, const __half* g, int64_t rs, int r0, int T) {
  for (int vid = threadIdx.x; vid < AT * 8; vid += blockDim.x) {
    const int r = vid & 63, dv = vid >> 6;
    float f[8];
    if (r0 + r < T) unpack8(ld8(g + (int64_t)(r0 + r) * rs + dv * 8), f);
    else {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) s[(dv * 8 + j) * ALD + r] = f[j];
  }
}
// acc[i][j] += sum_r At[r][ty*4+i] * Bt[r][tx*4+j]   (both operands reduction-major in shared memory)
__device__ __forceinline__ void mm64(const float* At, const float* Bt, int ty, int tx, float acc[4][4]) {
#pragma unroll 8
  for (int r = 0; r < AT; ++r) {
    const float4 a = *reinterpret_cast<const float4*>(At + r * ALD + ty * 4);
    const float4 b = *reinterpret_cast<const float4*>(Bt + r * ALD + tx * 4);
    const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
  }
}
__device__ __forceinline__ float row16_max(float v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float row16_sum(float v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(256) attn_fwd_kernel(const AttnArgs a) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ float sm[];
  float* QsT = sm;
  float* KsT = QsT + AT * ALD;
  float* Vs = KsT + AT * ALD;
  float* Pt = Vs + AT * ALD;
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * AT;
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  const __half* qg = a.q + (int64_t)b * a.qbs + (int64_t)h * a.qhs;
  const __half* kg = a.k + (int64_t)b * a.qbs + (int64_t)h * a.qhs;
  const __half* vg = a.v + (int64_t)b * a.qbs + (int64_t)h * a.qhs;
  load_tile_tr(QsT, qg, a.qrs, q0, a.T);
  float m[4], l[4], acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m[i] = -INFINITY;
    l[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  }
  for (int k0 = 0; k0 < a.T; k0 += AT) {
    __syncthreads();
    load_tile_tr(KsT, kg, a.qrs, k0, a.T);
    load_tile_rm(Vs, vg, a.qrs, k0, a.T);
    __syncthreads();
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
    mm64(QsT, KsT, ty, tx, s);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s[i][j] = (k0 + tx * 4 + j < a.T) ? s[i][j] * a.scale : -INFINITY;
        mx = fmaxf(mx, s[i][j]);
      }
      mx = row16_max(mx);
      const float m_new = fmaxf(m[i], mx);  // finite: every key tile holds at least one valid key
      const float alpha = __expf(m[i] - m_new);
      float rs = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s[i][j] = __expf(s[i][j] - m_new);
        rs += s[i][j];
      }
      rs = row16_sum(rs);
      l[i] = l[i] * alpha + rs;
      m[i] = m_new;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        acc[i][j] *= alpha;
        Pt[(tx * 4 + j) * ALD + ty * 4 + i] = s[i][j];
      }
    }
    __syncthreads();
    mm64(Pt, Vs, ty, tx, acc);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int q = q0 + ty * 4 + i;
    if (q >= a.T) continue;
    const float inv = 1.f / l[i];
    __half2* o = reinterpret_cast<__half2*>(a.out + (int64_t)b * a.obs + (int64_t)q * a.ors + (int64_t)h * a.ohs + tx * 4);
    o[0] = __floats2half2_rn(acc[i][0] * inv, acc[i][1] * inv);
    o[1] = __floats2half2_rn(acc[i][2] * inv, acc[i][3] * inv);
    if (tx == 0) a.lse[((int64_t)b * a.heads + h) * a.T + q] = m[i] + __logf(l[i]);
  }
}

// delta[b,h,q] = sum_d dO[q,d] * O[q,d]; one warp per row
__global__ void attn_delta_kernel(const AttnArgs a) {
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

// dK, dV for one key tile: loop over query tiles
__global__ void __launch_bounds__(256) attn_bwd_dkv_kernel(const AttnArgs a) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ float sm[];
  float* KsT = sm;
  float* VsT = KsT + AT * ALD;
  float* QsT = VsT + AT * ALD;
  float* Qs = QsT + AT * ALD;
  float* dOT = Qs + AT * ALD;
  float* dOs = dOT + AT * ALD;
  float* Ps = dOs + AT * ALD;
  float* dSs = Ps + AT * ALD;
  const int b = blockIdx.z, h = blockIdx.y, k0 = blockIdx.x * AT;
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  const int64_t qoff = (int64_t)b * a.qbs + (int64_t)h * a.qhs;
  const int64_t ooff = (int64_t)b * a.obs + (int64_t)h * a.ohs;
  load_tile_tr(KsT, a.k + qoff, a.qrs, k0, a.T);
  load_tile_tr(VsT, a.v + qoff, a.qrs, k0, a.T);
  float accK[4][4], accV[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) accK[i][j] = accV[i][j] = 0.f;
  const float* lse = a.lse + ((int64_t)b * a.heads + h) * a.T;
  const float* delta = a.delta + ((int64_t)b * a.heads + h) * a.T;
  for (int q0 = 0; q0 < a.T; q0 += AT) {
    __syncthreads();
    load_tile_tr(QsT, a.q + qoff, a.qrs, q0, a.T);
    load_tile_rm(Qs, a.q + qoff, a.qrs, q0, a.T);
    load_tile_tr(dOT, a.dout + ooff, a.ors, q0, a.T);
    load_tile_rm(dOs, a.dout + ooff, a.ors, q0, a.T);
    __syncthreads();
    float s[4][4], dp[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = dp[i][j] = 0.f;
    mm64(QsT, KsT, ty, tx, s);    // rows q (ty), cols k (tx)
    mm64(dOT, VsT, ty, tx, dp);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int q = q0 + ty * 4 + i;
      const bool qok = q < a.T;
      const float ls = qok ? lse[q] : 0.f, de = qok ? delta[q] : 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const bool ok = qok && (k0 + tx * 4 + j < a.T);
        const float p = ok ? __expf(s[i][j] * a.scale - ls) : 0.f;
        Ps[(ty * 4 + i) * ALD + tx * 4 + j] = p;
        dSs[(ty * 4 + i) * ALD + tx * 4 + j] = p * (dp[i][j] - de) * a.scale;
      }
    }
    __syncthreads();
    mm64(Ps, dOs, ty, tx, accV);   // rows k (ty), cols d (tx): sum_q P[q][k] dO[q][d]
    mm64(dSs, Qs, ty, tx, accK);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int k = k0 + ty * 4 + i;
    if (k >= a.T) continue;
    const int64_t off = qoff + (int64_t)k * a.qrs + tx * 4;
    __half2* dk = reinterpret_cast<__half2*>(a.dk + off);
    __half2* dv = reinterpret_cast<__half2*>(a.dv + off);
    dk[0] = __floats2half2_rn(accK[i][0], accK[i][1]);
    dk[1] = __floats2half2_rn(accK[i][2], accK[i][3]);
    dv[0] = __floats2half2_rn(accV[i][0], accV[i][1]);
    dv[1] = __floats2half2_rn(accV[i][2], accV[i][3]);
  }
}

// dQ for one query tile: loop over key tiles
__global__ void __launch_bounds__(256) attn_bwd_dq_kernel(const AttnArgs a) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ float sm[];
  float* QsT = sm;
  float* dOT = QsT + AT * ALD;
  float* KsT = dOT + AT * ALD;
  float* Ks = KsT + AT * ALD;
  float* VsT = Ks + AT * ALD;
  float* dSt = VsT + AT * ALD;
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * AT;
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  const int64_t qoff = (int64_t)b * a.qbs + (int64_t)h * a.qhs;
  const int64_t ooff = (int64_t)b * a.obs + (int64_t)h * a.ohs;
  load_tile_tr(QsT, a.q + qoff, a.qrs, q0, a.T);
  load_tile_tr(dOT, a.dout + ooff, a.ors, q0, a.T);
  float ls[4], de[4], acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int q = q0 + ty * 4 + i;
    ls[i] = q < a.T ? a.lse[((int64_t)b * a.heads + h) * a.T + q] : 0.f;
    de[i] = q < a.T ? a.delta[((int64_t)b * a.heads + h) * a.T + q] : 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  }
  for (int k0 = 0; k0 < a.T; k0 += AT) {
    __syncthreads();
    load_tile_tr(KsT, a.k + qoff, a.qrs, k0, a.T);
    load_tile_rm(Ks, a.k + qoff, a.qrs, k0, a.T);
    load_tile_tr(VsT, a.v + qoff, a.qrs, k0, a.T);
    __syncthreads();
    float s[4][4], dp[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = dp[i][j] = 0.f;
    mm64(QsT, KsT, ty, tx, s);
    mm64(dOT, VsT, ty, tx, dp);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const bool qok = (q0 + ty * 4 + i) < a.T;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const bool ok = qok && (k0 + tx * 4 + j < a.T);
        const float p = ok ? __expf(s[i][j] * a.scale - ls[i]) : 0.f;
        dSt[(tx * 4 + j) * ALD + ty * 4 + i] = p * (dp[i][j] - de[i]) * a.scale;
      }
    }
    __syncthreads();
    mm64(dSt, Ks, ty, tx, acc);  // rows q (ty), cols d (tx): sum_k dS[q][k] K[k][d]
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int q = q0 + ty * 4 + i;
    if (q >= a.T) continue;
    __half2* dq = reinterpret_cast<__half2*>(a.dq + qoff + (int64_t)q * a.qrs + tx * 4);
    dq[0] = __floats2half2_rn(acc[i][0], acc[i][1]);
    dq[1] = __floats2half2_rn(acc[i][2], acc[i][3]);
  }
}

int attn_wide_supported(int64_t d);                          // attention_wide.cu: head dims 128 / 192 / 256 (the 128x128 checkpoint's 4 heads)
int launch_attn_wide_fwd(const CgdOp& op, cudaStream_t st);
int launch_attn_wide_bwd(const CgdOp& op, cudaStream_t st);

static int attn_args(const CgdOp& op, AttnArgs& a, bool bwd) {
  a.B = (int)op.i[0]; a.heads = (int)op.i[1]; a.T = (int)op.i[2];
  CGD_CHECK_ARG(op.i[3] == 64 || attn_wide_supported(op.i[3]), "attention: head dim %lld unsupported (64, 128, 192, 256)", (long long)op.i[3]);
  CGD_CHECK_ARG(a.B > 0 && a.heads > 0 && a.T > 0, "attention: bad dims");
  a.qbs = op.i[4]; a.qrs = op.i[5]; a.qhs = op.i[6]; a.obs = op.i[7]; a.ors = op.i[8]; a.ohs = op.i[9];
  CGD_CHECK_ARG(a.qrs % 8 == 0 && a.qhs % 8 == 0 && a.qbs % 8 == 0 && a.ors % 8 == 0 && a.ohs % 8 == 0 && a.obs % 8 == 0,
                "attention: strides must be multiples of 8 elements");
  a.scale = op.f[0];
  a.q = (const __half*)op.p[0]; a.k = (const __half*)op.p[1]; a.v = (const __half*)op.p[2];
  for (int k = 0; k < 3; ++k) CGD_CHECK_ARG(op.p[k] && ((uintptr_t)op.p[k] % 16) == 0, "attention: q/k/v must be non-null and 16-byte aligned");
  if (!bwd) {
    a.out = (__half*)op.p[3]; a.lse = (float*)op.p[4];
    CGD_CHECK_ARG(a.out && a.lse, "attention: null out / lse");
  } else {
    a.o = (const __half*)op.p[3]; a.dout = (const __half*)op.p[4]; a.lse = (float*)op.p[5];
    a.dq = (__half*)op.p[6]; a.dk = (__half*)op.p[7]; a.dv = (__half*)op.p[8]; a.delta = (float*)op.p[9];
    CGD_CHECK_ARG(a.o && a.dout && a.lse && a.dq && a.dk && a.dv && a.delta, "attention bwd: null pointer");
  }
  return 0;
}

int attn_small_supported(int64_t T);                            // attention_small.cu: one 64-key tile per head on warp MMAs
int launch_attn_small_fwd(const CgdOp& op, cudaStream_t st);
int launch_attn_small_bwd(const CgdOp& op, cudaStream_t st);
static bool attn_use_small(int64_t T) {
  static int off = -1;
  if (off < 0) {
    const char* e = getenv("CGD_ATTN_SMALL");
    off = (e && e[0] == '0') ? 1 : 0;
  }
  return !off && attn_small_supported(T);
}

int launch_attn_mma_fwd(const CgdOp& op, cudaStream_t st);  // attention_mma.cu: flash attention on warp MMAs (any T)
int launch_attn_mma_bwd(const CgdOp& op, cudaStream_t st);
static bool attn_use_mma() {
  static int off = -1;
  if (off < 0) {
    const char* e = getenv("CGD_ATTN_MMA");
    off = (e && e[0] == '0') ? 1 : 0;
  }
  return !off;
}
int attn_bwd_num_launches(const CgdOp& op) {
  if (op.i[3] != 64) return 2;
  return attn_use_small(op.i[2]) ? 1 : (attn_use_mma() ? 2 : 3);
}

int launch_attn_fwd(const CgdOp& op, cudaStream_t st) {
  AttnArgs a{};
  if (int rc = attn_args(op, a, false)) return rc;
  if (op.i[3] != 64) return launch_attn_wide_fwd(op, st);
  if (attn_use_small(a.T)) return launch_attn_small_fwd(op, st);
  if (attn_use_mma()) return launch_attn_mma_fwd(op, st);
  const int smem = 4 * AT * ALD * (int)sizeof(float);
  static DeviceOnce set;
  if (set.needed()) {
    CGD_CUDA(cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    set.mark();
  }
  CGD_CUDA(launch_pdl(attn_fwd_kernel, dim3((unsigned)ceil_div(a.T, AT), a.heads, a.B), dim3(256), smem, st, a));
  CGD_LAUNCH_CHECK();
  return 0;
}

int launch_attn_bwd(const CgdOp& op, cudaStream_t st) {
  AttnArgs a{};
  if (int rc = attn_args(op, a, true)) return rc;
  if (op.i[3] != 64) return launch_attn_wide_bwd(op, st);
  if (attn_use_small(a.T)) return launch_attn_small_bwd(op, st);
  if (attn_use_mma()) return launch_attn_mma_bwd(op, st);
  const int smem_kv = 8 * AT * ALD * (int)sizeof(float), smem_q = 6 * AT * ALD * (int)sizeof(float);
  static DeviceOnce set;
  if (set.needed()) {
    CGD_CUDA(cudaFuncSetAttribute(attn_bwd_dkv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_kv));
    CGD_CUDA(cudaFuncSetAttribute(attn_bwd_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_q));
    set.mark();
  }
  const int64_t rows = (int64_t)a.B * a.heads * a.T;
  CGD_CUDA(launch_pdl(attn_delta_kernel, dim3((unsigned)ceil_div(rows, 8)), dim3(256), 0, st, a));
  CGD_LAUNCH_CHECK();
  const dim3 grid((unsigned)ceil_div(a.T, AT), a.heads, a.B);
  CGD_CUDA(launch_pdl(attn_bwd_dkv_kernel, dim3(grid), dim3(256), smem_kv, st, a));
  CGD_LAUNCH_CHECK();
  CGD_CUDA(launch_pdl(attn_bwd_dq_kernel, dim3(grid), dim3(256), smem_q, st, a));
  CGD_LAUNCH_CHECK();
  return 0;
}

// ================================================================================================
// Tensor-core attention for long sequences (T % 256 == 0: the 32x32 and 16x16 UNet levels).
// S = Q K^T, O = P V and the four backward products run as batched GEMMs on the wgmma conv kernel (conv_tc.cu,
// CGD_OP_CONV with a batched B operand); the kernels below are the glue: batched fp16 transposes (so that every GEMM
// operand is K-major), the fp32 row softmax (fp16 in/out like the reference's `softmax(w.float()).type(w.dtype)`), and
// its backward dS = P * (dP - rowsum(P * dP)) * scale.
// ================================================================================================

struct TransposeArgs {
  const __half* src[3];
  __half* dst[3];
  int64_t sb1[3], sb2[3], sr[3];
  int npairs, nb1, nb2, R, C;
  int64_t Rp;
};
// dst[b1][b2][c][r] = src[b1][b2][r][c]; 32x32 tiles through shared memory, coalesced both ways
__global__ void transpose_kernel(const TransposeArgs a) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ __half tile[32][34];
  int z = blockIdx.z;
  const int pair = z % a.npairs;
  z /= a.npairs;
  const int b2 = z % a.nb2, b1 = z / a.nb2;
  const __half* src = a.src[pair] + (int64_t)b1 * a.sb1[pair] + (int64_t)b2 * a.sb2[pair];
  __half* dst = a.dst[pair] + ((int64_t)b1 * a.nb2 + b2) * a.C * a.Rp;
  const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int r = r0 + j, c = c0 + threadIdx.x;
    tile[j][threadIdx.x] = (r < a.R && c < a.C) ? src[(int64_t)r * a.sr[pair] + c] : __float2half(0.f);
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    if (c < a.C && r < a.R) dst[(int64_t)c * a.Rp + r] = tile[threadIdx.x][j];
  }
}
int launch_transpose(const CgdOp& op, cudaStream_t st) {
  TransposeArgs a{};
  a.nb1 = (int)op.i[0]; a.nb2 = (int)op.i[1]; a.R = (int)op.i[2]; a.C = (int)op.i[3]; a.Rp = op.i[13];
  CGD_CHECK_ARG(a.nb1 > 0 && a.nb2 > 0 && a.R > 0 && a.C > 0 && a.Rp >= a.R, "transpose: bad dims");
  for (int k = 0; k < 3; ++k) {
    if (!op.p[2 * k]) break;
    CGD_CHECK_ARG(op.p[2 * k + 1] != nullptr, "transpose: null destination");
    a.src[k] = (const __half*)op.p[2 * k];
    a.dst[k] = (__half*)op.p[2 * k + 1];
    a.sb1[k] = op.i[4 + 3 * k]; a.sb2[k] = op.i[5 + 3 * k]; a.sr[k] = op.i[6 + 3 * k];
    a.npairs = k + 1;
  }
  CGD_CHECK_ARG(a.npairs > 0, "transpose: no operands");
  dim3 grid((unsigned)ceil_div(a.R, 32), (unsigned)ceil_div(a.C, 32), (unsigned)(a.nb1 * a.nb2 * a.npairs));
  CGD_CUDA(launch_pdl(transpose_kernel, dim3(grid), dim3(32, 8), 0, st, a));
  CGD_LAUNCH_CHECK();
  return 0;
}

constexpr int SM_MAXV = 8;  // 8 x half8 per lane -> T <= 2048
// in place: S[row, :T] (fp16 logits, un-scaled) -> P = softmax(scale * S) ; lse[row] = logsumexp(scale * S)
__global__ void softmax_fwd_kernel(__half* __restrict__ S, float* __restrict__ lse, int64_t rows, int T, int64_t Tp, float scale) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  __half* s = S + row * Tp;
  const int nv = T / 8;
  float v[SM_MAXV][8];
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < SM_MAXV; ++k) {
    const int vi = lane + k * 32;
    if (vi < nv) {
      unpack8(ld8(s + vi * 8), v[k]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        v[k][j] *= scale;
        mx = fmaxf(mx, v[k][j]);
      }
    }
  }
  mx = warp_max(mx);
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < SM_MAXV; ++k) {
    const int vi = lane + k * 32;
    if (vi < nv) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        v[k][j] = __expf(v[k][j] - mx);
        sum += v[k][j];
      }
    }
  }
  sum = warp_sum(sum);
  const float inv = 1.f / sum;
  if (lane == 0 && lse) lse[row] = mx + __logf(sum);
#pragma unroll
  for (int k = 0; k < SM_MAXV; ++k) {
    const int vi = lane + k * 32;
    if (vi < nv) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[k][j] *= inv;
      st8(s + vi * 8, pack8(v[k]));
    }
  }
}
// in place on dP: dS = P * (dP - sum_k P*dP) * scale
__global__ void softmax_bwd_kernel(const __half* __restrict__ P, __half* __restrict__ dP, int64_t rows, int T, int64_t Tp, float scale) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const __half* p = P + row * Tp;
  __half* d = dP + row * Tp;
  const int nv = T / 8;
  float pv[SM_MAXV][8], dv[SM_MAXV][8];
  float dot = 0.f;
#pragma unroll
  for (int k = 0; k < SM_MAXV; ++k) {
    const int vi = lane + k * 32;
    if (vi < nv) {
      unpack8(ld8(p + vi * 8), pv[k]);
      unpack8(ld8(d + vi * 8), dv[k]);
#pragma unroll
      for (int j = 0; j < 8; ++j) dot = fmaf(pv[k][j], dv[k][j], dot);
    }
  }
  dot = warp_sum(dot);
#pragma unroll
  for (int k = 0; k < SM_MAXV; ++k) {
    const int vi = lane + k * 32;
    if (vi < nv) {
#pragma unroll
      for (int j = 0; j < 8; ++j) dv[k][j] = pv[k][j] * (dv[k][j] - dot) * scale;
      st8(d + vi * 8, pack8(dv[k]));
    }
  }
}
int launch_softmax_fwd(const CgdOp& op, cudaStream_t st) {
  const int64_t rows = op.i[0], T = op.i[1], Tp = op.i[2];
  CGD_CHECK_ARG(rows > 0 && T > 0 && T % 8 == 0 && T <= 8 * 32 * SM_MAXV && Tp >= T && Tp % 8 == 0 && op.p[0], "softmax: unsupported shape");
  CGD_CUDA(launch_pdl(softmax_fwd_kernel, dim3((unsigned)ceil_div(rows, 8)), dim3(256), 0, st, (__half*)op.p[0], (float*)op.p[1], rows, (int)T, Tp, op.f[0]));
  CGD_LAUNCH_CHECK();
  return 0;
}
int launch_softmax_bwd(const CgdOp& op, cudaStream_t st) {
  const int64_t rows = op.i[0], T = op.i[1], Tp = op.i[2];
  CGD_CHECK_ARG(rows > 0 && T > 0 && T % 8 == 0 && T <= 8 * 32 * SM_MAXV && Tp >= T && Tp % 8 == 0 && op.p[0] && op.p[1], "softmax bwd: unsupported shape");
  CGD_CUDA(launch_pdl(softmax_bwd_kernel, dim3((unsigned)ceil_div(rows, 8)), dim3(256), 0, st, (const __half*)op.p[0], (__half*)op.p[1], rows, (int)T, Tp, op.f[0]));
  CGD_LAUNCH_CHECK();
  return 0;
}

}  // namespace cgd
