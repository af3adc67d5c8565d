// attention_flash.cu -- flash attention for head dims 64 / 128 / 192 / 256 (any sequence length), forward and backward, on
// warp-level tensor-core MMAs (mma.sync m16n8k16, ldmatrix, fp16 operands, fp32 accumulate / softmax).  Nothing T x T touches HBM.
//
// Replaces [3P] guided-diffusion QKVAttention(Legacy) at the 32x32 / 16x16 UNet levels (T = 1024 / 256), [3P] CLIP
// nn.MultiheadAttention's core for ViT-B/16, L/14 (T = 197, 257) (SURVEY.md K4, K14), and QKVAttentionLegacy of the 128x128
// checkpoint (data/diffusion_model_flags.py: num_heads = 4 and no num_head_channels, so the 32x32 / 16x16 / 8x8 levels attend with
// 512 / 4 = 128, 768 / 4 = 192 and 1024 / 4 = 256 channels per head; the 128^2 model is the default image_size of cgd/cgd.py:20).
// The head dim is cut into NC chunks of 64 columns, each chunk a 64 x 64 shared tile of the layout attn_mma.cuh works on:
//   forward   S = sum_c Q_c K_c^T, online softmax, O_c += P V_c for every chunk (NC accumulator sets per warp); K / V tiles
//             double-buffered with cp.async;
//   backward  delta = rowsum(dO * O); one CTA per (key tile, chunk) accumulates dK_c, dV_c over the query tiles and one CTA per
//             (query tile, chunk) accumulates dQ_c over the key tiles, both halves in one launch.  S and dP need the whole head dim,
//             so for NC > 1 every chunk's CTA recomputes them (NC-fold redundant in two of the five products): that keeps the
//             accumulators at 64 columns instead of 2 * NC * 32 registers per thread.  The streamed tiles are double-buffered for
//             NC = 1 and single-buffered otherwise (af_bwd_bufs).
#include <cuda_fp16.h>

#include "attn_mma.cuh"
#include "common.cuh"
#include "ops.cuh"
#include "pdl.cuh"

namespace cgd {

// 64 rows x (64 * NC) columns of a [T, 64 * NC] matrix, global -> NC shared tiles (chunk c at s + c * AS_TILE); rows >= T zero-filled
template <int NC>
__device__ __forceinline__ void af_load_async(__half* s, const __half* g, int64_t rs, int r0, int T) {
  for (int v = threadIdx.x; v < AS_T * 8 * NC; v += blockDim.x) {
    // row r, 16-byte vector cc of the row; NC = 1 as shifts, which ptxas does not derive from the signed division
    const int r = NC == 1 ? v >> 3 : v / (8 * NC), cc = NC == 1 ? v & 7 : v % (8 * NC);
    const int c = cc >> 3, col = (cc & 7) * 8;
    const int row = r0 + r;
    const __half* src = g + (int64_t)min(row, T - 1) * rs + c * AS_T + col;
    const uint32_t sz = row < T ? 16u : 0u;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(as_smem(s + c * AS_TILE + r * AS_LD + col)), "l"(src), "r"(sz) : "memory");
  }
}
__device__ __forceinline__ void af_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void af_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// acc += X[r0 .. r0+16, 64 cols] * Y^T for one chunk (Y stored [n][k]); as_mm_nk without the zeroing
__device__ __forceinline__ void af_mm_nk_acc(float (&acc)[8][4], const __half* X, const __half* Y, int r0, int lane) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    uint32_t a[4];
    ldsm_x4(as_addr_a(X, r0, ks * 16, lane), a);
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      uint32_t b[4];
      ldsm_x4(as_addr_b_nk(Y, jj * 16, ks * 16, lane), b);
      mma16816(acc[2 * jj], a, b[0], b[1]);
      mma16816(acc[2 * jj + 1], a, b[2], b[3]);
    }
  }
}
// acc = sum over the NC chunks of X_c[r0.., :] * Y_c^T  (S = Q K^T, dP = dO V^T over the whole head dim)
template <int NC>
__device__ __forceinline__ void af_mm_nk(float (&acc)[8][4], const __half* X, const __half* Y, int r0, int lane) {
  as_zero(acc);
#pragma unroll
  for (int c = 0; c < NC; ++c) af_mm_nk_acc(acc, X + c * AS_TILE, Y + c * AS_TILE, r0, lane);
}

// ------------------------------------------------------------------------------------------------ forward
// CAUSAL: query i attends to keys j <= i only (the CLIP text tower).  A CTA's key loop then ends at the diagonal tile (key tile
// blockIdx.x), the only tile that needs masking.  Key tile 0 always holds key 0, so the running max is finite after it.
template <int NC, bool CAUSAL>
__global__ void __launch_bounds__(128) attn_flash_fwd_kernel(const AttnArgs a) {
  // Q | K0 | K1 | V0 | V1, NC tiles each.  NC = 1 (45 KB) fits static shared memory, which compiles to faster code for d = 64;
  // larger NC need the dynamic allocation.
  __half* sm;
  if constexpr (NC == 1) {
    __shared__ __align__(16) __half st[5 * AS_TILE];
    sm = st;
  } else {
    extern __shared__ __align__(16) __half af_dyn[];
    sm = af_dyn;
  }
  __half* Qs = sm;
  __half* Ks = sm + NC * AS_TILE;
  __half* Vs = sm + 3 * NC * AS_TILE;
  pdl_wait();
  pdl_launch_dependents();
  const int q0 = blockIdx.x * AS_T, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t qoff = (int64_t)b * a.qbs + (int64_t)h * a.qhs;
  const int n_kt = CAUSAL ? min((a.T + AS_T - 1) / AS_T, (int)blockIdx.x + 1) : (a.T + AS_T - 1) / AS_T;
  af_load_async<NC>(Qs, a.q + qoff, a.qrs, q0, a.T);
  af_load_async<NC>(Ks, a.k + qoff, a.qrs, 0, a.T);
  af_load_async<NC>(Vs, a.v + qoff, a.qrs, 0, a.T);
  af_commit();
  const int r0 = warp * 16;
  const int cb = (lane & 3) * 2;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float o[NC][8][4];
#pragma unroll
  for (int c = 0; c < NC; ++c) as_zero(o[c]);
  for (int kt = 0; kt < n_kt; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < n_kt) {  // prefetch the next K / V tile into the other buffer (its last readers finished at the barrier below)
      af_load_async<NC>(Ks + (buf ^ 1) * NC * AS_TILE, a.k + qoff, a.qrs, (kt + 1) * AS_T, a.T);
      af_load_async<NC>(Vs + (buf ^ 1) * NC * AS_TILE, a.v + qoff, a.qrs, (kt + 1) * AS_T, a.T);
      af_commit();
      af_wait<1>();
    } else {
      af_wait<0>();
    }
    __syncthreads();
    float s[8][4];
    af_mm_nk<NC>(s, Qs, Ks + buf * NC * AS_TILE, r0, lane);
    const int k0 = kt * AS_T;
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const bool ok = k0 + j * 8 + cb + e < a.T;
        bool ok0 = ok, ok1 = ok;
        if constexpr (CAUSAL) {
          // diagonal tile (q0 == k0): key column c is masked for the tile's query rows < c
          const int col = j * 8 + cb + e, ra = r0 + (lane >> 2);
          const bool diag = kt == (int)blockIdx.x;
          ok0 = ok && !(diag && col > ra);
          ok1 = ok && !(diag && col > ra + 8);
        }
        s[j][e] = ok0 ? s[j][e] * a.scale : -INFINITY;
        s[j][2 + e] = ok1 ? s[j][2 + e] * a.scale : -INFINITY;
        mx0 = fmaxf(mx0, s[j][e]);
        mx1 = fmaxf(mx1, s[j][2 + e]);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);  // finite: every key tile holds at least one valid key per row
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
    uint32_t pa[4][4];
    as_c_to_a(s, pa);
#pragma unroll
    for (int c = 0; c < NC; ++c) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[c][j][0] *= al0;
        o[c][j][1] *= al0;
        o[c][j][2] *= al1;
        o[c][j][3] *= al1;
      }
      as_mm_reg_kn<false>(o[c], pa, Vs + (buf * NC + c) * AS_TILE, lane);
    }
    __syncthreads();  // all warps are done with buffer `buf` before the next iteration's prefetch overwrites it
  }
  const float i0 = 1.f / l0, i1 = 1.f / l1;
  __half* og = a.out + (int64_t)b * a.obs + (int64_t)h * a.ohs + (int64_t)q0 * a.ors;
#pragma unroll
  for (int c = 0; c < NC; ++c) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[c][j][0] *= i0;
      o[c][j][1] *= i0;
      o[c][j][2] *= i1;
      o[c][j][3] *= i1;
    }
    as_store_c(o[c], og + c * AS_T, a.ors, r0, a.T - q0, lane);
  }
  if ((lane & 3) == 0) {
    const int ra = q0 + r0 + (lane >> 2);
    float* lse = a.lse + ((int64_t)b * a.heads + h) * a.T;
    if (ra < a.T) lse[ra] = m0 + __logf(l0);
    if (ra + 8 < a.T) lse[ra + 8] = m1 + __logf(l1);
  }
}

// delta[b,h,q] = sum_d dO[q,d] * O[q,d] over the 64 * NC columns of the head; one warp per row
template <int NC>
__global__ void attn_flash_delta_kernel(const AttnArgs a) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int64_t total = (int64_t)a.B * a.heads * a.T;
  if (row >= total) return;
  const int q = (int)(row % a.T);
  const int h = (int)((row / a.T) % a.heads);
  const int b = (int)(row / ((int64_t)a.T * a.heads));
  const int64_t off = (int64_t)b * a.obs + (int64_t)q * a.ors + (int64_t)h * a.ohs;
  float s = 0.f;
#pragma unroll
  for (int c = lane * 2; c < NC * AS_T; c += 64) {
    const float2 x = __half22float2(*reinterpret_cast<const __half2*>(a.o + off + c));
    const float2 y = __half22float2(*reinterpret_cast<const __half2*>(a.dout + off + c));
    s += x.x * y.x + x.y * y.y;
  }
  s = warp_sum(s);
  if (lane == 0) a.delta[row] = s;
}

// P and dS fragments of the warp's 16 query rows against 64 keys: s <- P = exp(S * scale - lse), dp <- dS = P * (dP - delta) * scale
__device__ __forceinline__ void af_p_ds(float (&s)[8][4], float (&dp)[8][4], float ls0, float ls1, float de0, float de1, bool q0ok, bool q1ok,
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

// Shared-memory buffers per streamed tile of the backward (Q / dO in the dK / dV half, K / V in the dQ half): two for NC = 1, one
// above (a second would halve the CTAs per SM at NC = 2 and not fit 227 KB at NC = 4).  Tile t is loaded in iteration
// t - (kBufs - 1): one iteration ahead when double-buffered, in the iteration that uses it when single-buffered.  Either way the
// barrier that ends an iteration frees the buffer it read.
__host__ __device__ constexpr int af_bwd_bufs(int nc) { return nc == 1 ? 2 : 1; }

// ------------------------------------------------------------------------------------------------ backward: dK_c, dV_c per (key tile, chunk)
template <int NC>
__device__ __forceinline__ void attn_flash_bwd_dkv_body(const AttnArgs& a, __half* dyn, int tile_x, int chunk) {
  constexpr int kBufs = af_bwd_bufs(NC);
  // shared: K | V | Q x kBufs | dO x kBufs (NC tiles each) | P | dS
  __half* Ks = dyn;
  __half* Vs = dyn + NC * AS_TILE;
  __half* Qs = dyn + 2 * NC * AS_TILE;
  __half* dOs = Qs + kBufs * NC * AS_TILE;
  __half* Ps = dOs + kBufs * NC * AS_TILE;
  __half* dSs = Ps + AS_TILE;
  const int k0 = tile_x * AS_T, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t qoff = (int64_t)b * a.qbs + (int64_t)h * a.qhs;
  const int64_t ooff = (int64_t)b * a.obs + (int64_t)h * a.ohs;
  const float* lse = a.lse + ((int64_t)b * a.heads + h) * a.T;
  const float* delta = a.delta + ((int64_t)b * a.heads + h) * a.T;
  const int n_qt = (a.T + AS_T - 1) / AS_T;
  af_load_async<NC>(Ks, a.k + qoff, a.qrs, k0, a.T);
  af_load_async<NC>(Vs, a.v + qoff, a.qrs, k0, a.T);
  if (kBufs == 2) {
    af_load_async<NC>(Qs, a.q + qoff, a.qrs, 0, a.T);
    af_load_async<NC>(dOs, a.dout + ooff, a.ors, 0, a.T);
  }
  af_commit();
  const int r0 = warp * 16;
  float dk[8][4], dv[8][4];
  as_zero(dk);
  as_zero(dv);
  for (int qt = 0; qt < n_qt; ++qt) {
    const int load_t = qt + kBufs - 1;
    if (load_t < n_qt) {
      af_load_async<NC>(Qs + load_t % kBufs * NC * AS_TILE, a.q + qoff, a.qrs, load_t * AS_T, a.T);
      af_load_async<NC>(dOs + load_t % kBufs * NC * AS_TILE, a.dout + ooff, a.ors, load_t * AS_T, a.T);
      af_commit();
      af_wait<kBufs - 1>();  // also covers K / V in the first iteration
    } else {
      af_wait<0>();
    }
    __syncthreads();
    const __half* Qb = Qs + qt % kBufs * NC * AS_TILE;
    const __half* dOb = dOs + qt % kBufs * NC * AS_TILE;
    {
      float s[8][4], dp[8][4];
      af_mm_nk<NC>(s, Qb, Ks, r0, lane);    // S rows = this warp's 16 queries of the tile, whole head dim
      af_mm_nk<NC>(dp, dOb, Vs, r0, lane);  // dP = dO V^T
      const int qa = qt * AS_T + r0 + (lane >> 2), qb = qa + 8;
      const bool okA = qa < a.T, okB = qb < a.T;
      af_p_ds(s, dp, okA ? lse[qa] : 0.f, okB ? lse[qb] : 0.f, okA ? delta[qa] : 0.f, okB ? delta[qb] : 0.f, okA, okB, k0, a.T, a.scale, lane);
      as_store_p_ds(s, dp, Ps, dSs, r0, lane);
    }
    __syncthreads();
    as_mm_t_kn<false>(dv, Ps, dOb + chunk * AS_TILE, r0, lane);  // dV_c[keys r0..] += P^T dO_c
    as_mm_t_kn<false>(dk, dSs, Qb + chunk * AS_TILE, r0, lane);  // dK_c[keys r0..] += dS^T Q_c
    __syncthreads();  // P / dS and buffer qt % kBufs are free again
  }
  as_store_c(dk, a.dk + qoff + (int64_t)k0 * a.qrs + chunk * AS_T, a.qrs, r0, a.T - k0, lane);
  as_store_c(dv, a.dv + qoff + (int64_t)k0 * a.qrs + chunk * AS_T, a.qrs, r0, a.T - k0, lane);
}

// ------------------------------------------------------------------------------------------------ backward: dQ_c per (query tile, chunk)
template <int NC>
__device__ __forceinline__ void attn_flash_bwd_dq_body(const AttnArgs& a, __half* dyn, int tile_x, int chunk) {
  constexpr int kBufs = af_bwd_bufs(NC);
  // shared: Q | dO | K x kBufs | V x kBufs (NC tiles each)
  __half* Qs = dyn;
  __half* dOs = dyn + NC * AS_TILE;
  __half* Ks = dyn + 2 * NC * AS_TILE;
  __half* Vs = Ks + kBufs * NC * AS_TILE;
  const int q0 = tile_x * AS_T, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t qoff = (int64_t)b * a.qbs + (int64_t)h * a.qhs;
  const int64_t ooff = (int64_t)b * a.obs + (int64_t)h * a.ohs;
  const int n_kt = (a.T + AS_T - 1) / AS_T;
  af_load_async<NC>(Qs, a.q + qoff, a.qrs, q0, a.T);
  af_load_async<NC>(dOs, a.dout + ooff, a.ors, q0, a.T);
  if (kBufs == 2) {
    af_load_async<NC>(Ks, a.k + qoff, a.qrs, 0, a.T);
    af_load_async<NC>(Vs, a.v + qoff, a.qrs, 0, a.T);
  }
  af_commit();
  const int r0 = warp * 16;
  const int qa = q0 + r0 + (lane >> 2), qb = qa + 8;
  const bool okA = qa < a.T, okB = qb < a.T;
  const float* lse = a.lse + ((int64_t)b * a.heads + h) * a.T;
  const float* delta = a.delta + ((int64_t)b * a.heads + h) * a.T;
  const float lsA = okA ? lse[qa] : 0.f, lsB = okB ? lse[qb] : 0.f, deA = okA ? delta[qa] : 0.f, deB = okB ? delta[qb] : 0.f;
  float dq[8][4];
  as_zero(dq);
  for (int kt = 0; kt < n_kt; ++kt) {
    const int load_t = kt + kBufs - 1;
    if (load_t < n_kt) {
      af_load_async<NC>(Ks + load_t % kBufs * NC * AS_TILE, a.k + qoff, a.qrs, load_t * AS_T, a.T);
      af_load_async<NC>(Vs + load_t % kBufs * NC * AS_TILE, a.v + qoff, a.qrs, load_t * AS_T, a.T);
      af_commit();
      af_wait<kBufs - 1>();  // also covers Q / dO in the first iteration
    } else {
      af_wait<0>();
    }
    __syncthreads();
    const __half* Kb = Ks + kt % kBufs * NC * AS_TILE;
    float s[8][4], dp[8][4];
    af_mm_nk<NC>(s, Qs, Kb, r0, lane);
    af_mm_nk<NC>(dp, dOs, Vs + kt % kBufs * NC * AS_TILE, r0, lane);
    af_p_ds(s, dp, lsA, lsB, deA, deB, okA, okB, kt * AS_T, a.T, a.scale, lane);
    uint32_t dsa[4][4];
    as_c_to_a(dp, dsa);
    as_mm_reg_kn<false>(dq, dsa, Kb + chunk * AS_TILE, lane);  // dQ_c += dS K_c
    __syncthreads();  // buffer kt % kBufs is free again
  }
  as_store_c(dq, a.dq + qoff + (int64_t)q0 * a.qrs + chunk * AS_T, a.qrs, r0, a.T - q0, lane);
}

// One launch for both: blocks [0, tiles * NC) accumulate dK_c / dV_c of a key tile, blocks [tiles * NC, 2 * tiles * NC) dQ_c of a
// query tile.  The two halves are independent and each runs four warps per CTA, so side by side they fill the SMs twice as well
// as back to back.
template <int NC>
__global__ void __launch_bounds__(128) attn_flash_bwd_kernel(const AttnArgs a, int tiles) {
  extern __shared__ __align__(16) __half af_dyn[];
  pdl_wait();
  pdl_launch_dependents();
  const int bx = (int)blockIdx.x;
  if (bx < tiles * NC) attn_flash_bwd_dkv_body<NC>(a, af_dyn, bx / NC, bx % NC);
  else attn_flash_bwd_dq_body<NC>(a, af_dyn, (bx - tiles * NC) / NC, (bx - tiles * NC) % NC);
}

// ------------------------------------------------------------------------------------------------ host
template <int NC, bool CAUSAL>
static int af_fwd(const AttnArgs& a, cudaStream_t st) {
  constexpr int smem = NC == 1 ? 0 : 5 * NC * AS_TILE * (int)sizeof(__half);  // dynamic shared memory
  static DeviceOnce set;
  if (set.needed()) {
    CGD_CUDA(cudaFuncSetAttribute(attn_flash_fwd_kernel<NC, CAUSAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    set.mark();
  }
  CGD_CUDA(launch_pdl(attn_flash_fwd_kernel<NC, CAUSAL>, dim3((unsigned)ceil_div(a.T, AS_T), a.heads, a.B), dim3(128), smem, st, a));
  return 0;
}

template <int NC>
static int af_bwd(const AttnArgs& a, cudaStream_t st) {
  // the dK / dV half needs (2 + 2 kBufs) NC + 2 tiles, the dQ half 2 fewer
  constexpr int smem = ((2 + 2 * af_bwd_bufs(NC)) * NC + 2) * AS_TILE * (int)sizeof(__half);
  static DeviceOnce set;
  if (set.needed()) {
    CGD_CUDA(cudaFuncSetAttribute(attn_flash_bwd_kernel<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    set.mark();
  }
  const int64_t rows = (int64_t)a.B * a.heads * a.T;
  CGD_CUDA(launch_pdl(attn_flash_delta_kernel<NC>, dim3((unsigned)ceil_div(rows, 8)), dim3(256), 0, st, a));
  const int tiles = (int)ceil_div(a.T, AS_T);
  CGD_CUDA(launch_pdl(attn_flash_bwd_kernel<NC>, dim3((unsigned)(2 * tiles * NC), a.heads, a.B), dim3(128), smem, st, a, tiles));
  return 0;
}

int launch_attn_flash_fwd(const AttnArgs& a, int nc, bool causal, cudaStream_t st) {
  switch (nc) {
    case 1: return causal ? af_fwd<1, true>(a, st) : af_fwd<1, false>(a, st);
    case 2: return causal ? af_fwd<2, true>(a, st) : af_fwd<2, false>(a, st);
    case 3: return causal ? af_fwd<3, true>(a, st) : af_fwd<3, false>(a, st);
    case 4: return causal ? af_fwd<4, true>(a, st) : af_fwd<4, false>(a, st);
    default: break;
  }
  CGD_CHECK_ARG(false, "attention: head dim %d unsupported (64, 128, 192, 256)", nc * AS_T);
  return 0;
}

int launch_attn_flash_bwd(const AttnArgs& a, int nc, cudaStream_t st) {
  switch (nc) {
    case 1: return af_bwd<1>(a, st);
    case 2: return af_bwd<2>(a, st);
    case 3: return af_bwd<3>(a, st);
    case 4: return af_bwd<4>(a, st);
    default: break;
  }
  CGD_CHECK_ARG(false, "attention: head dim %d unsupported (64, 128, 192, 256)", nc * AS_T);
  return 0;
}

}  // namespace cgd
