// linear_small.cu -- small-M fp32 linear layers: y[M,N] (=|+=) act(x[M,K]) @ W[N,K]^T + b.
//
// Replaces the [3P] UNet time_embed MLP and the ~30 per-ResBlock emb_layers Linears (x-independent, forward
// only; SURVEY.md K8) and the [3P] CLIP head ln_post(cls) @ proj with its transpose for the backward (K16).
// M is the batch (1..64 rows) so these are weight-streaming GEMVs: one warp per output column, the weight
// row read once with 128-bit loads, M accumulators per lane, x staged in shared memory.
#include <algorithm>

#include "common.cuh"
#include "pdl.cuh"
#include "ops.cuh"

namespace cgd {

constexpr int LS_MT = 8;  // rows of x per block

// 8 consecutive weights of a row as floats (fp32 or fp16 storage)
__device__ __forceinline__ void ls_load8(const float* w, float* f) {
  const float4 a = *reinterpret_cast<const float4*>(w), b = *reinterpret_cast<const float4*>(w + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
__device__ __forceinline__ void ls_load8(const __half* w, float* f) { unpack8(ld8(w), f); }

// `scatter` (optional, int2 per output column = element offset of row 0, row stride): lets ONE launch produce the outputs of many
// independent Linears that share x -- the ~30 ResBlock emb_layers -- each into its own [M, N_k] block.
template <typename XT, typename WT>
__global__ void linear_small_kernel(const XT* __restrict__ x, const WT* __restrict__ Wt, const float* __restrict__ bias, void* __restrict__ y,
                                    const int2* __restrict__ scatter, int M, int K, int N, int64_t ldx, int64_t ldy, int silu_in,
                                    int accumulate, int y_half) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ float xs[];  // [LS_MT][K]
  const int m0 = blockIdx.y * LS_MT, mt = min(LS_MT, M - m0);
  for (int i = threadIdx.x; i < mt * K; i += blockDim.x) {
    const int r = i / K, c = i % K;
    float v = (float)x[(int64_t)(m0 + r) * ldx + c];
    xs[r * K + c] = silu_in ? silu_f(v) : v;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int n = blockIdx.x * nw + wid; n < N; n += gridDim.x * nw) {
    const WT* wr = Wt + (int64_t)n * K;
    float acc[LS_MT];
#pragma unroll
    for (int r = 0; r < LS_MT; ++r) acc[r] = 0.f;
    for (int c = lane * 8; c < K; c += 256) {
      float w8[8];
      ls_load8(wr + c, w8);
#pragma unroll
      for (int r = 0; r < LS_MT; ++r) {
        if (r < mt) {
          const float4 x0 = *reinterpret_cast<const float4*>(xs + r * K + c), x1 = *reinterpret_cast<const float4*>(xs + r * K + c + 4);
          acc[r] = fmaf(w8[0], x0.x, fmaf(w8[1], x0.y, fmaf(w8[2], x0.z, fmaf(w8[3], x0.w, acc[r]))));
          acc[r] = fmaf(w8[4], x1.x, fmaf(w8[5], x1.y, fmaf(w8[6], x1.z, fmaf(w8[7], x1.w, acc[r]))));
        }
      }
    }
#pragma unroll
    for (int r = 0; r < LS_MT; ++r) acc[r] = warp_sum(acc[r]);
    if (lane == 0) {
      const float bv = bias ? bias[n] : 0.f;
      for (int r = 0; r < mt; ++r) {
        const int64_t o = scatter ? (int64_t)scatter[n].x + (int64_t)(m0 + r) * scatter[n].y : (int64_t)(m0 + r) * ldy + n;
        float v = acc[r] + bv;
        if (y_half) {
          __half* yh = reinterpret_cast<__half*>(y);
          if (accumulate) v += __half2float(yh[o]);
          yh[o] = __float2half_rn(v);
        } else {
          float* yf = reinterpret_cast<float*>(y);
          if (accumulate) v += yf[o];
          yf[o] = v;
        }
      }
    }
  }
}

template <typename XT, typename WT>
static int ls_launch(const CgdOp& op, cudaStream_t st, dim3 grid, int smem, int M, int K, int N, int64_t ldx, int64_t ldy, int silu, int acc, int yh) {
  static DeviceOnce set;
  if (set.needed()) {
    CGD_CUDA(cudaFuncSetAttribute(linear_small_kernel<XT, WT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    set.mark();
  }
  CGD_CUDA(launch_pdl(linear_small_kernel<XT, WT>, grid, dim3(256), smem, st, (const XT*)op.p[0], (const WT*)op.p[1], (const float*)op.p[2], op.p[3],
                      (const int2*)op.p[4], M, K, N, ldx, ldy, silu, acc, yh));
  return 0;
}

int launch_linear_small(const CgdOp& op, cudaStream_t st) {
  const int64_t M = op.i[0], K = op.i[1], N = op.i[2], ldx = op.i[3], ldy = op.i[4];
  CGD_CHECK_ARG(M > 0 && K > 0 && K % 8 == 0 && N > 0 && op.p[0] && op.p[1] && op.p[3], "linear_small: bad args (M=%lld K=%lld N=%lld)",
                (long long)M, (long long)K, (long long)N);
  CGD_CHECK_ARG((size_t)LS_MT * K * sizeof(float) <= 96 * 1024, "linear_small: K=%lld too large", (long long)K);
  const int smem = (int)(LS_MT * K * sizeof(float));
  const int silu = op.flags & 1, acc = (op.flags & 2) ? 1 : 0, xh = (op.flags & 4) ? 1 : 0, yh = (op.flags & 8) ? 1 : 0, wh = (op.flags & 16) ? 1 : 0;
  const dim3 grid((unsigned)std::min<int64_t>(ceil_div(N, 8), 132 * 4), (unsigned)ceil_div(M, LS_MT));
  if (xh && wh) return ls_launch<__half, __half>(op, st, grid, smem, (int)M, (int)K, (int)N, ldx, ldy, silu, acc, yh);
  if (xh) return ls_launch<__half, float>(op, st, grid, smem, (int)M, (int)K, (int)N, ldx, ldy, silu, acc, yh);
  if (wh) return ls_launch<float, __half>(op, st, grid, smem, (int)M, (int)K, (int)N, ldx, ldy, silu, acc, yh);
  return ls_launch<float, float>(op, st, grid, smem, (int)M, (int)K, (int)N, ldx, ldy, silu, acc, yh);
}

}  // namespace cgd
