// attn_mma.cuh -- warp-level tensor-core building blocks (mma.sync m16n8k16, ldmatrix) shared by the single-tile attention
// (attention_small.cu) and the flash attention kernels (attention_flash.cu): 64 x 64 fp16 tiles in shared memory, row pitch 72.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace cgd {

constexpr int AS_T = 64;        // tile edge: queries, keys, head dim
constexpr int AS_LD = AS_T + 8; // shared-memory row pitch in halfs (144 B: 16-byte aligned, ldmatrix conflict-free)
constexpr int AS_TILE = AS_T * AS_LD;  // halfs per shared tile

// Operands of one ATTN_FWD / ATTN_BWD op (slots in include/cgd_b200.h), unpacked once by attention.cu
struct AttnArgs {
  const __half *q, *k, *v, *o, *dout;
  __half *out, *dq, *dk, *dv;
  float *lse, *delta;
  int B, heads, T;
  int64_t qbs, qrs, qhs;  // qkv batch / row / head strides (elements)
  int64_t obs, ors, ohs;  // out / dout strides
  float scale;
};

__device__ __forceinline__ uint32_t as_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
// D(16x8, fp32) += A(16x16, fp16 row) * B(16x8, fp16 col)
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// 64 x 64 fp16 tile (rows < T valid, zero-filled beyond) global -> shared, 16-byte vectors
__device__ __forceinline__ void as_load_tile(__half* s, const __half* g, int64_t rs, int T) {
  for (int v = threadIdx.x; v < AS_T * 8; v += blockDim.x) {
    const int r = v >> 3, c = (v & 7) * 8;
    half8 val;
    if (r < T) val = ld8(g + (int64_t)r * rs + c);
    else val.a = val.b = val.c = val.d = __floats2half2_rn(0.f, 0.f);
    *reinterpret_cast<half8*>(s + r * AS_LD + c) = val;
  }
}

// Fragment address helpers (lane -> row address for ldmatrix.x4); see the comment block in each product below.
// A operand 16x16 at (r0, c0) of a row-major [m][k] tile
__device__ __forceinline__ uint32_t as_addr_a(const __half* s, int r0, int c0, int lane) {
  const int mi = lane >> 3;
  return as_smem(s + (r0 + (lane & 7) + (mi & 1) * 8) * AS_LD + c0 + (mi >> 1) * 8);
}
// B operand (k16 x n16 = two n-tiles) from a tile stored [n][k] (k contiguous): regs {b0,b1} of n-tile 0, {b0,b1} of n-tile 1
__device__ __forceinline__ uint32_t as_addr_b_nk(const __half* s, int n0, int k0, int lane) {
  const int mi = lane >> 3;
  return as_smem(s + (n0 + (lane & 7) + (mi >> 1) * 8) * AS_LD + k0 + (mi & 1) * 8);
}
// B operand (k16 x n16) from a tile stored [k][n] (n contiguous), with ldmatrix.trans: same register order as above
__device__ __forceinline__ uint32_t as_addr_b_kn(const __half* s, int k0, int n0, int lane) {
  const int mi = lane >> 3;
  return as_smem(s + (k0 + (lane & 7) + (mi & 1) * 8) * AS_LD + n0 + (mi >> 1) * 8);
}
// A operand 16x16 = (X^T)[m0.., k0..] from a tile X stored [k][m] (m contiguous), with ldmatrix.trans
__device__ __forceinline__ uint32_t as_addr_a_t(const __half* s, int m0, int k0, int lane) {
  const int mi = lane >> 3;
  return as_smem(s + (k0 + (lane & 7) + (mi >> 1) * 8) * AS_LD + m0 + (mi & 1) * 8);
}

// acc[j] (8 n-tiles of 8 columns) = X[r0..r0+16, :] * Y^T with Y stored [n][k] (k = head dim contiguous): S = Q K^T, dP = dO V^T
__device__ __forceinline__ void as_zero(float (&acc)[8][4]) {
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;
}
__device__ __forceinline__ void as_mm_nk(float (&acc)[8][4], const __half* X, const __half* Y, int r0, int lane) {
  as_zero(acc);
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
// acc = P[16 rows, 64] (fp16 A fragments held in registers, 4 k-steps) * Y with Y stored [k][n] (n contiguous): O = P V, dQ = dS K
template <bool ZERO = true>
__device__ __forceinline__ void as_mm_reg_kn(float (&acc)[8][4], const uint32_t (&pa)[4][4], const __half* Y, int lane) {
  if (ZERO) as_zero(acc);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      uint32_t b[4];
      ldsm_x4_t(as_addr_b_kn(Y, ks * 16, jj * 16, lane), b);
      mma16816(acc[2 * jj], pa[ks], b[0], b[1]);
      mma16816(acc[2 * jj + 1], pa[ks], b[2], b[3]);
    }
  }
}
// acc = (X^T)[m0..m0+16, :] * Y with X stored [k][m] and Y stored [k][n]: dV = P^T dO, dK = dS^T Q
template <bool ZERO = true>
__device__ __forceinline__ void as_mm_t_kn(float (&acc)[8][4], const __half* X, const __half* Y, int m0, int lane) {
  if (ZERO) as_zero(acc);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    uint32_t a[4];
    ldsm_x4_t(as_addr_a_t(X, m0, ks * 16, lane), a);
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      uint32_t b[4];
      ldsm_x4_t(as_addr_b_kn(Y, ks * 16, jj * 16, lane), b);
      mma16816(acc[2 * jj], a, b[0], b[1]);
      mma16816(acc[2 * jj + 1], a, b[2], b[3]);
    }
  }
}

// Row softmax of the warp's 16 x 64 score fragment (rows r0 + lane/4 and r0 + lane/4 + 8), keys >= T masked, and with CAUSAL
// also keys after the row's query; returns P in `s`.
template <bool CAUSAL = false>
__device__ __forceinline__ void as_softmax(float (&s)[8][4], int T, float scale, int lane, float& lse0, float& lse1, int r0 = 0) {
  const int cbase = (lane & 3) * 2;
  const int ra = r0 + (lane >> 2);
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int col = j * 8 + cbase + e;
      const bool ok = col < T;
      s[j][e] = ok && (!CAUSAL || col <= ra) ? s[j][e] * scale : -INFINITY;  // key 0 is never masked: the row max stays finite
      s[j][2 + e] = ok && (!CAUSAL || col <= ra + 8) ? s[j][2 + e] * scale : -INFINITY;
      mx0 = fmaxf(mx0, s[j][e]);
      mx1 = fmaxf(mx1, s[j][2 + e]);
    }
  }
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
  float l0 = 0.f, l1 = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      s[j][e] = __expf(s[j][e] - mx0);  // exp(-inf) = 0 for masked keys; T >= 1 keeps mx finite
      s[j][2 + e] = __expf(s[j][2 + e] - mx1);
      l0 += s[j][e];
      l1 += s[j][2 + e];
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.f / l0, i1 = 1.f / l1;
  lse0 = mx0 + __logf(l0);
  lse1 = mx1 + __logf(l1);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    s[j][0] *= i0;
    s[j][1] *= i0;
    s[j][2] *= i1;
    s[j][3] *= i1;
  }
}
// fp32 C fragments (16 x 64) -> fp16 A fragments for the next product (4 k-steps of 16)
__device__ __forceinline__ void as_c_to_a(const float (&c)[8][4], uint32_t (&a)[4][4]) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    a[ks][0] = pack_h2(c[2 * ks][0], c[2 * ks][1]);
    a[ks][1] = pack_h2(c[2 * ks][2], c[2 * ks][3]);
    a[ks][2] = pack_h2(c[2 * ks + 1][0], c[2 * ks + 1][1]);
    a[ks][3] = pack_h2(c[2 * ks + 1][2], c[2 * ks + 1][3]);
  }
}
// fp32 C fragments of rows r0 + lane/4 (+8) -> global fp16 rows (row stride rs), rows >= T skipped
__device__ __forceinline__ void as_store_c(const float (&c)[8][4], __half* g, int64_t rs, int r0, int T, int lane) {
  const int ra = r0 + (lane >> 2), rb = ra + 8, cb = (lane & 3) * 2;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (ra < T) *reinterpret_cast<__half2*>(g + (int64_t)ra * rs + j * 8 + cb) = __floats2half2_rn(c[j][0], c[j][1]);
    if (rb < T) *reinterpret_cast<__half2*>(g + (int64_t)rb * rs + j * 8 + cb) = __floats2half2_rn(c[j][2], c[j][3]);
  }
}
// P and dS fragments of rows r0 + lane/4 (+8) -> fp16 shared tiles ([query][key]) for the transposed products dV = P^T dO, dK = dS^T Q
__device__ __forceinline__ void as_store_p_ds(const float (&p)[8][4], const float (&ds)[8][4], __half* Ps, __half* dSs, int r0, int lane) {
  const int ra = r0 + (lane >> 2), cb = (lane & 3) * 2;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    *reinterpret_cast<__half2*>(Ps + ra * AS_LD + j * 8 + cb) = __floats2half2_rn(p[j][0], p[j][1]);
    *reinterpret_cast<__half2*>(Ps + (ra + 8) * AS_LD + j * 8 + cb) = __floats2half2_rn(p[j][2], p[j][3]);
    *reinterpret_cast<__half2*>(dSs + ra * AS_LD + j * 8 + cb) = __floats2half2_rn(ds[j][0], ds[j][1]);
    *reinterpret_cast<__half2*>(dSs + (ra + 8) * AS_LD + j * 8 + cb) = __floats2half2_rn(ds[j][2], ds[j][3]);
  }
}

}  // namespace cgd
