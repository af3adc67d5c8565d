// resample.cu -- separable resampling of one axis of an fp32 NCHW tensor with host-built tables (CGD_OP_RESIZE_AXIS).
//
// Image prompts (cgd/clip_util.py:90-101) resize a photo of any size so that its short side matches the diffusion size, with
// ResizeRight's antialiased lanczos3 (cgd/ResizeRight/resize_right.py:31-122).  The host builds the tables of one axis
// (clip_guided_diffusion_b200/resize_right.py `tables(S, O, t_max=None)`), this op applies them:
//   out[.., o, ..] = sum_{i < T} w[o, i] * in[.., left[o] + i, ..],   samples outside [0, S) are zero (pad_mode 'constant').
// The tap count T has no fixed cap: reducing a 4000-px side to 64 px takes 375 taps.  Sums run in fp32 in tap order.
// One-shot work (once per image prompt and run), so the aim is sane memory access rather than peak bandwidth.
#include "common.cuh"
#include "ops.cuh"
#include "pdl.cuh"

namespace cgd {

static inline int rs_blocks(int64_t items, int threads = 256) {
  int64_t b = ceil_div(items, threads);
  if (b > 132 * 8) b = 132 * 8;
  if (b < 1) b = 1;
  return (int)b;
}

// H pass: one thread per output element, consecutive threads on consecutive columns, so every tap reads one coalesced row segment
__global__ void resize_axis_h_kernel(const float* __restrict__ in, float* __restrict__ out, const int* __restrict__ left,
                                     const float* __restrict__ wt, int planes, int Hin, int W, int O, int T) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t total = (int64_t)planes * O * W;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(idx % W);
    const int64_t r = idx / W;
    const int o = (int)(r % O), pl = (int)(r / O);
    const int l = left[o];
    const float* w = wt + (int64_t)o * T;
    const float* src = in + (int64_t)pl * Hin * W + x;
    // taps whose row lies inside [0, Hin); the others read zero padding and add nothing
    const int i0 = max(0, -l), i1 = (int)min((int64_t)T, (int64_t)Hin - l);
    float acc = 0.f;
    for (int i = i0; i < i1; ++i) acc = fmaf(w[i], src[(int64_t)(l + i) * W], acc);
    out[idx] = acc;
  }
}

// W pass: one block per input row (grid-stride), one thread per output column in chunks of blockDim.  The span of input columns a
// chunk reads is staged in shared memory, RS_TILE columns at a time; every thread walks its taps in order across the tiles, so the
// sum order does not depend on the tiling.
constexpr int RS_THREADS = 256;
constexpr int RS_TILE = 4096;  // 16 KB of staged input columns

__global__ void __launch_bounds__(RS_THREADS)
resize_axis_w_kernel(const float* __restrict__ in, float* __restrict__ out, const int* __restrict__ left, const float* __restrict__ wt,
                     int64_t rows, int Win, int O, int T) {
  __shared__ float tile[RS_TILE];
  __shared__ int span[2];
  pdl_wait();
  pdl_launch_dependents();
  for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
    const float* src = in + row * Win;
    float* dst = out + row * O;
    for (int o0 = 0; o0 < O; o0 += RS_THREADS) {
      const int o = o0 + (int)threadIdx.x;
      const bool active = o < O;
      const int l = active ? left[o] : 0;
      // taps inside [0, Win): [i0, i1); the chunk's input span is the union over its threads (no ordering of `left` assumed)
      const int i0 = active ? max(0, -l) : 0;
      const int i1 = active ? (int)min((int64_t)T, (int64_t)Win - l) : 0;
      if (threadIdx.x == 0) {
        span[0] = Win;
        span[1] = 0;
      }
      __syncthreads();
      if (i0 < i1) {
        atomicMin(&span[0], l + i0);
        atomicMax(&span[1], l + i1);
      }
      __syncthreads();
      const int lo = span[0], hi = span[1];
      const float* w = wt + (int64_t)(active ? o : 0) * T;
      float acc = 0.f;
      int i = i0;
      for (int base = lo; base < hi; base += RS_TILE) {
        const int n = min(RS_TILE, hi - base);
        __syncthreads();  // the previous tile (or span[]) has been read by every thread
        for (int k = threadIdx.x; k < n; k += RS_THREADS) tile[k] = src[base + k];
        __syncthreads();
        const int iend = min(i1, base + n - l);  // taps whose column lies in this tile
        for (; i < iend; ++i) acc = fmaf(w[i], tile[l + i - base], acc);
      }
      if (active) dst[o] = acc;
      __syncthreads();  // span[] is rewritten by the next chunk
    }
  }
}

int launch_resize_axis(const CgdOp& op, cudaStream_t st) {
  const int64_t planes = op.i[0], Hin = op.i[1], Win = op.i[2], axis = op.i[3], O = op.i[4], T = op.i[5];
  const int64_t lim = (int64_t)1 << 31;
  CGD_CHECK_ARG(op.p[0] && op.p[1] && op.p[2] && op.p[3], "resize_axis: null pointer");
  CGD_CHECK_ARG(planes > 0 && planes < lim && Hin > 0 && Hin < lim && Win > 0 && Win < lim && O > 0 && O < lim && T > 0 && T < lim,
                "resize_axis: dims must lie in [1, 2^31): planes=%lld H=%lld W=%lld O=%lld T=%lld", (long long)planes, (long long)Hin,
                (long long)Win, (long long)O, (long long)T);
  CGD_CHECK_ARG(axis == 0 || axis == 1, "resize_axis: axis %lld is neither 0 (H) nor 1 (W)", (long long)axis);
  // element counts of the table, the input and the output (in double: the products of three 31-bit dims overflow int64)
  const double big = (double)((int64_t)1 << 40);
  CGD_CHECK_ARG((double)O * T < big && (double)planes * Hin * Win < big && (double)planes * (axis == 0 ? (double)O * Win : (double)Hin * O) < big,
                "resize_axis: tensor sizes out of range (2^40 elements)");
  const float* in = (const float*)op.p[0];
  float* out = (float*)op.p[1];
  const int* left = (const int*)op.p[2];
  const float* wt = (const float*)op.p[3];
  if (axis == 0) {
    CGD_CUDA(launch_pdl(resize_axis_h_kernel, dim3(rs_blocks(planes * O * Win)), dim3(256), 0, st, in, out, left, wt, (int)planes, (int)Hin,
                        (int)Win, (int)O, (int)T));
  } else {
    const int64_t rows = planes * Hin;
    CGD_CUDA(launch_pdl(resize_axis_w_kernel, dim3((unsigned)(rows < 132 * 8 ? rows : 132 * 8)), dim3(RS_THREADS), 0, st, in, out, left, wt,
                        rows, (int)Win, (int)O, (int)T));
  }
  return 0;
}

}  // namespace cgd
