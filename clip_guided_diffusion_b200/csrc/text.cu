// text.cu -- the two gathers of the CLIP text tower that the ViT ops do not cover ([3P] clip/model.py CLIP.encode_text):
//   TOKEN_EMBED  x[n, t, :] = fp16(table[ids[n, t], :] + pos[t, :])   (token_embedding(text) + positional_embedding)
//   ROW_GATHER   y[i, :] = x[idx[i], :]                                (the end-of-text token of every sequence)
// One thread per 8 halfs (128-bit loads and stores).  Ids and indices live on the device, so the host cannot bound them before the
// launch: an id or index outside its table yields a row of NaNs instead of a read outside the table (the text tower checks its ids
// on the host before it uploads them).
#include "common.cuh"
#include "ops.cuh"
#include "pdl.cuh"

namespace cgd {

static inline int tx_blocks(int64_t items) {
  int64_t b = ceil_div(items, 256);
  if (b > 132 * 8) b = 132 * 8;
  return (int)(b < 1 ? 1 : b);
}

__device__ __forceinline__ half8 nan8() {
  Half8Bits b;
  b.u = make_uint4(0x7e007e00u, 0x7e007e00u, 0x7e007e00u, 0x7e007e00u);
  return b.h;
}

__global__ void token_embed_kernel(const int* __restrict__ ids, const __half* __restrict__ table, const float* __restrict__ pos,
                                   __half* __restrict__ x, int64_t rows, int T, int w, int V) {
  pdl_wait();
  pdl_launch_dependents();
  const int nv = w / 8;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < rows * nv; idx += (int64_t)gridDim.x * blockDim.x) {
    const int v = (int)(idx % nv);
    const int64_t row = idx / nv;
    const int t = (int)(row % T);
    const int id = ids[row];
    __half* dst = x + row * w + v * 8;
    if (id < 0 || id >= V) {
      st8(dst, nan8());
      continue;
    }
    float a[8];
    unpack8(ld8(table + (int64_t)id * w + v * 8), a);
    const float4 p0 = *reinterpret_cast<const float4*>(pos + (int64_t)t * w + v * 8);
    const float4 p1 = *reinterpret_cast<const float4*>(pos + (int64_t)t * w + v * 8 + 4);
    a[0] += p0.x; a[1] += p0.y; a[2] += p0.z; a[3] += p0.w;
    a[4] += p1.x; a[5] += p1.y; a[6] += p1.z; a[7] += p1.w;
    st8(dst, pack8(a));
  }
}

__global__ void row_gather_kernel(const __half* __restrict__ x, const int* __restrict__ idx, __half* __restrict__ y, int64_t rows, int w,
                                  int64_t ldx, int64_t ldy, int64_t n_src) {
  pdl_wait();
  pdl_launch_dependents();
  const int nv = w / 8;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < rows * nv; k += (int64_t)gridDim.x * blockDim.x) {
    const int v = (int)(k % nv);
    const int64_t r = k / nv;
    const int64_t src = idx[r];
    st8(y + r * ldy + v * 8, (src >= 0 && src < n_src) ? ld8(x + src * ldx + v * 8) : nan8());
  }
}

static bool aligned16(const void* p) { return p && ((uintptr_t)p % 16) == 0; }

int launch_token_embed(const CgdOp& op, cudaStream_t st) {
  const int64_t n = op.i[0], T = op.i[1], w = op.i[2], V = op.i[3];
  const int64_t lim = (int64_t)1 << 31;
  CGD_CHECK_ARG(aligned16(op.p[0]) && aligned16(op.p[1]) && aligned16(op.p[2]) && aligned16(op.p[3]),
                "token_embed: ids / table / pos / x must be non-null and 16-byte aligned");
  CGD_CHECK_ARG(n > 0 && n < lim && T > 0 && T < lim && V > 0 && V < lim && w > 0 && w < lim && w % 8 == 0,
                "token_embed: dims must lie in [1, 2^31) with w %% 8 == 0: n=%lld T=%lld w=%lld V=%lld", (long long)n, (long long)T,
                (long long)w, (long long)V);
  CGD_CHECK_ARG((double)n * T * w < (double)((int64_t)1 << 40) && (double)V * w < (double)((int64_t)1 << 40),
                "token_embed: tensor sizes out of range (2^40 elements)");
  CGD_CUDA(launch_pdl(token_embed_kernel, dim3(tx_blocks(n * T * (w / 8))), dim3(256), 0, st, (const int*)op.p[0], (const __half*)op.p[1],
                      (const float*)op.p[2], (__half*)op.p[3], n * T, (int)T, (int)w, (int)V));
  return 0;
}

int launch_row_gather(const CgdOp& op, cudaStream_t st) {
  const int64_t rows = op.i[0], w = op.i[1], ldx = op.i[2], ldy = op.i[3], n_src = op.i[4];
  const int64_t lim = (int64_t)1 << 31;
  CGD_CHECK_ARG(aligned16(op.p[0]) && op.p[1] && ((uintptr_t)op.p[1] % 4) == 0 && aligned16(op.p[2]),
                "row_gather: x / y must be non-null and 16-byte aligned, idx non-null and 4-byte aligned");
  CGD_CHECK_ARG(rows > 0 && rows < lim && n_src > 0 && n_src < lim && w > 0 && w < lim && w % 8 == 0,
                "row_gather: dims must lie in [1, 2^31) with w %% 8 == 0: rows=%lld w=%lld n_src=%lld", (long long)rows, (long long)w,
                (long long)n_src);
  CGD_CHECK_ARG(ldx >= w && ldx < lim && ldx % 8 == 0 && ldy >= w && ldy < lim && ldy % 8 == 0,
                "row_gather: row strides must be multiples of 8 in [w, 2^31): ldx=%lld ldy=%lld", (long long)ldx, (long long)ldy);
  CGD_CHECK_ARG((double)n_src * ldx < (double)((int64_t)1 << 40) && (double)rows * ldy < (double)((int64_t)1 << 40),
                "row_gather: tensor sizes out of range (2^40 elements)");
  CGD_CUDA(launch_pdl(row_gather_kernel, dim3(tx_blocks(rows * (w / 8))), dim3(256), 0, st, (const __half*)op.p[0], (const int*)op.p[1],
                      (__half*)op.p[2], rows, (int)w, ldx, ldy, n_src));
  return 0;
}

}  // namespace cgd
