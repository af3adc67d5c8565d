// conv_tc.cu -- implicit-GEMM convolution / GEMM on Hopper wgmma tensor cores.
//
// Replaces (forward and input-gradient directions) the [3P] guided-diffusion UNet Conv2d 3x3 / 1x1 and
// Conv1d k=1 layers and the [3P] CLIP ViT Linear / patch-conv layers that the reference runs through
// cuDNN / cuBLAS (SURVEY.md K1-K3, K12, K13).
//
// Formulation.  Activations are pixel-major fp16 ([n, y, x, c], c contiguous).  One CTA owns a
// 128-pixel x BN-channel output tile; the 128 pixels are a TW x TH x TN box of the image grid.
// For every filter tap and every 64-channel slice of the input, one TMA 4-D tiled load fetches the
// (dx,dy)-shifted box -- out-of-image coordinates are zero-filled by the TMA unit, which *is* the
// conv padding -- into a 128B-swizzled K-major shared-memory tile; one TMA load fetches the matching
// [BN x 64] slice of the pre-packed weights.  Warp 8 is the TMA producer; warps 0-7 are two consumer
// warpgroups, each issuing wgmma.m64nBNk16 x4 per stage for its 64 pixel rows and accumulating in
// registers.  Pipeline: STAGES-deep smem ring with full/empty mbarriers; a stage is released once
// the wgmma group that read it has retired (wait_group 1 keeps one group in flight).
// Epilogue: the accumulators go to an fp32 staging tile that reuses the ring; then each consumer thread
// owns one pixel row and half of the tile's channels and adds bias / residual, stores fp16 / fp32.
// Small-M layers (8x8 .. 32x32 feature maps, long-K Linears) split K over gridDim.z: either into an
// fp32 workspace summed by a reduce kernel, or (CONV i23 = 1) inside a thread-block cluster of
// `splits` CTAs that sum each other's staging tiles through distributed shared memory -- one launch,
// no workspace; CTA s of the cluster finishes columns [s*BN/S, (s+1)*BN/S) of the tile.
#include <cuda.h>
#include <stdlib.h>

#include <algorithm>

#include "common.cuh"
#include "conv_tc.cuh"
#include "pdl.cuh"
#include "tc_ptx.cuh"
#include "wgmma_ptx.cuh"

namespace cgd {

// ---------------------------------------------------------------- kernel
constexpr int BM = 128, BK = 64;
constexpr int kConsumers = 256;            // warps 0..7: two wgmma warpgroups of 64 pixel rows each
constexpr int kThreads = kConsumers + 32;  // warp 8: TMA producer

template <int BN>
struct TcCfg {
  static constexpr int kStages = (BN >= 192) ? 4 : (BN >= 128 ? 6 : 8);
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStageLd = BN + 4;  // fp32 staging row stride (floats): 16-byte aligned rows, rows shifted across banks
  static constexpr int kStagingBytes = BM * kStageLd * 4;
  static constexpr int kAuxBytes = 256 /*barriers*/ + BN * 4 /*epilogue statistics exchange: 4 row quarters x BN/8 octets x 2*/;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + kAuxBytes;
  static_assert(kStagingBytes <= kStages * kStageBytes, "the fp32 staging tile reuses the operand ring");
  static_assert(kSmemBytes <= 227 * 1024, "H100: at most 227 KB of shared memory per block");
};

template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const ConvTcParams p) {
  using Cfg = TcCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + Cfg::kStages * Cfg::kABytes;
  float* staging = reinterpret_cast<float*>(smem);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
  uint64_t* empty_bar = full_bar + Cfg::kStages;
  float* stat_red = reinterpret_cast<float*>(smem + Cfg::kStages * Cfg::kStageBytes + 256);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // ---- tile coordinates
  const int mt = blockIdx.x;
  const int tw_i = mt % p.tiles_w;
  const int th_i = (mt / p.tiles_w) % p.tiles_h;
  const int tn_i = mt / (p.tiles_w * p.tiles_h);
  const int w0 = tw_i * p.TW, h0 = th_i * p.TH, n0 = tn_i * p.TN;
  const int ncol0 = blockIdx.y * BN;
  const int kb0 = blockIdx.z * p.kb_per_split;
  const int kb1 = min(kb0 + p.kb_per_split, p.kblocks);  // non-empty for every split (host)

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kConsumers / 32);  // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();

  if (warp == kConsumers / 32) {
    // ===== TMA producer
    if (lane == 0) {
      const int cblks = p.Cin / BK;
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait_trap(&empty_bar[stage], phase ^ 1);
        mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
        const int tap = kb / cblks, cb = kb - tap * cblks;
        int dy = 0, dx = 0;
        if (p.taps == 9) {
          dy = tap / 3 - 1;
          dx = tap % 3 - 1;
        }
        tma_load_4d(smem_a + stage * Cfg::kABytes, &tmA, &full_bar[stage], cb * BK, w0 + dx, h0 + dy, n0);
        tma_load_4d(smem_b + stage * Cfg::kBBytes, &tmB, &full_bar[stage], kb * BK, ncol0, p.b_batched ? h0 : 0, p.b_batched ? n0 : 0);
        if (++stage == Cfg::kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    } else if (p.pf_bytes > 0) {
      l2_prefetch_slice(p.pf_ptr, p.pf_bytes, (int)(blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z)),
                        (int)(gridDim.x * gridDim.y * gridDim.z), lane - 1, 31);
    }
  } else {
    // ===== consumer warpgroup wg: pixel rows [64 wg, 64 wg + 64) of the tile
    const int wg = warp >> 2;
    float acc[BN / 2];
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait_trap(&full_bar[stage], phase);
      const uint64_t da = make_wgmma_desc_sw128(smem_u32(smem_a + stage * Cfg::kABytes + wg * 64 * 128));
      const uint64_t db = make_wgmma_desc_sw128(smem_u32(smem_b + stage * Cfg::kBBytes));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)  // advance 16 elements (32 B) along K inside the 128 B swizzle row: +2 in the (>>4) address field
        wgmma_f16<BN>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb > kb0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();  // the group of the previous stage has retired: its operands may be overwritten
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      prev = stage;
      if (++stage == Cfg::kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) wgmma_fence_operand(acc[j]);
    named_bar_sync(1, kConsumers);  // both warpgroups are done reading the ring: it becomes the staging tile
    const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), col0 = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      *reinterpret_cast<float2*>(staging + (size_t)row0 * Cfg::kStageLd + 8 * j + col0) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(staging + (size_t)(row0 + 8) * Cfg::kStageLd + 8 * j + col0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  __syncthreads();
  if (p.cluster) cluster_sync_all();  // every CTA of the cluster has staged its partial tile

  if (warp < kConsumers / 32) {
    // ===== epilogue: thread = (pixel row r, half of the columns this CTA finishes)
    const int quad = warp & 3, half = warp >> 2;
    const int r = quad * 32 + lane;
    const int w_off = r % p.TW, h_off = (r / p.TW) % p.TH, n_off = r / (p.TW * p.TH);
    const int n = n0 + n_off, h = h0 + h_off, w = w0 + w_off;
    const bool row_ok = (n < p.NB) && (h < p.H) && (w < p.W);
    const int S = p.cluster ? p.splits : 1;
    const int cw = BN / S;  // columns finished by this CTA (a multiple of 16: host)
    const int c_lo = (p.cluster ? (int)cluster_ctarank() * cw : 0) + half * (cw / 2), c_hi = c_lo + cw / 2;
    const float* srow = staging + (size_t)r * Cfg::kStageLd;
    const int64_t o_off = (int64_t)n * p.out_sn + (int64_t)h * p.out_sh + (int64_t)w * p.out_sw;
    const int64_t r_off = (int64_t)n * p.res_sn + (int64_t)h * p.res_sh + (int64_t)w * p.res_sw;
    const bool vec_ok = !p.out_f32 && p.out_sc == 1;
    const bool to_ws = p.splits > 1 && !p.cluster;
    float* ws = to_ws ? p.ws + ((size_t)blockIdx.z * p.ws_rows + (size_t)mt * BM + r) * p.Npad + ncol0 : nullptr;
#pragma unroll 1
    for (int c = c_lo; c < c_hi; c += 8) {
      float a[8];
      if (p.cluster) {  // fixed order over the cluster's partial tiles: bit-reproducible
#pragma unroll
        for (int e = 0; e < 8; ++e) a[e] = 0.f;
        const uint32_t local = smem_u32(srow + c);
        for (int j = 0; j < S; ++j) {
          const uint32_t remote = mapa_u32(local, (uint32_t)j);
          const float4 u0 = ld_cluster_f4(remote), u1 = ld_cluster_f4(remote + 16);
          a[0] += u0.x; a[1] += u0.y; a[2] += u0.z; a[3] += u0.w;
          a[4] += u1.x; a[5] += u1.y; a[6] += u1.z; a[7] += u1.w;
        }
      } else {
        const float4 u0 = *reinterpret_cast<const float4*>(srow + c), u1 = *reinterpret_cast<const float4*>(srow + c + 4);
        a[0] = u0.x; a[1] = u0.y; a[2] = u0.z; a[3] = u0.w;
        a[4] = u1.x; a[5] = u1.y; a[6] = u1.z; a[7] = u1.w;
      }
      if (to_ws) {  // raw fp32 partials -> workspace [split][tile row][Npad]; rows outside the image are never read back
        if (row_ok) {
          *reinterpret_cast<float4*>(ws + c) = make_float4(a[0], a[1], a[2], a[3]);
          *reinterpret_cast<float4*>(ws + c + 4) = make_float4(a[4], a[5], a[6], a[7]);
        }
        continue;
      }
      const int col = ncol0 + c;
      float st_s = 0.f, st_q = 0.f;  // flags 2: this row's sum / sum of squares of the octet's fp16 outputs
      if (row_ok && col < p.Cout) {
        if (col + 8 <= p.Cout && vec_ok) {
          if (p.bias) {
            const float4 b0 = __ldg(reinterpret_cast<const float4*>(p.bias + col));
            const float4 b1 = __ldg(reinterpret_cast<const float4*>(p.bias + col + 4));
            a[0] += b0.x; a[1] += b0.y; a[2] += b0.z; a[3] += b0.w;
            a[4] += b1.x; a[5] += b1.y; a[6] += b1.z; a[7] += b1.w;
          }
          if (p.res) {
            float rr[8];
            unpack8(ld8(p.res + r_off + col), rr);
            if (p.res_mode == 1) {  // CONV flags 4: out = acc * QuickGELU'(u), u = the tile read through the residual path
#pragma unroll
              for (int e = 0; e < 8; ++e) {
                const float sg = rcp_ftz(1.f + ex2_ftz(-1.702f * 1.4426950408889634f * rr[e]));  // sigmoid(1.702 u), MUFU ex2 + rcp
                a[e] *= sg * fmaf(1.702f * rr[e], 1.f - sg, 1.f);
              }
            } else {
#pragma unroll
              for (int e = 0; e < 8; ++e) a[e] += rr[e];
            }
          }
          const half8 hv = pack8(a);
          st8(reinterpret_cast<__half*>(p.out) + o_off + col, hv);
          if (p.epi_stats) {  // statistics of the ROUNDED values: what the GroupNorm after this conv reads
            float f[8];
            unpack8(hv, f);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              st_s += f[e];
              st_q = fmaf(f[e], f[e], st_q);
            }
          }
        } else {
          for (int e = 0; e < 8 && col + e < p.Cout; ++e) {
            float x = a[e];
            if (p.bias) x += p.bias[col + e];
            if (p.res) x += __half2float(p.res[r_off + col + e]);
            if (p.out_f32) reinterpret_cast<float*>(p.out)[o_off + (col + e) * p.out_sc] = x;
            else reinterpret_cast<__half*>(p.out)[o_off + (col + e) * p.out_sc] = __float2half_rn(x);
          }
        }
      }
      if (p.epi_stats) {  // 32 rows -> one value per octet and row quarter (warp-uniform branch: full tiles, host)
        st_s = warp_sum(st_s);
        st_q = warp_sum(st_q);
        if (lane == 0) {
          stat_red[(quad * (BN / 8) + c / 8) * 2] = st_s;
          stat_red[(quad * (BN / 8) + c / 8) * 2 + 1] = st_q;
        }
      }
    }
    if (p.epi_stats) {
      named_bar_sync(1, kConsumers);
      if ((int)threadIdx.x < BN / 4) {  // thread (octet o = t / 2, kind = t % 2): fixed-order sum over the four row quarters
        const int o = threadIdx.x >> 1, kind = threadIdx.x & 1, stride = (BN / 8) * 2;
        const float* src = stat_red + o * 2 + kind;
        const float v = (src[0] + src[stride]) + (src[2 * stride] + src[3 * stride]);
        p.epi_stats[((size_t)mt * (p.Npad / 8) + (size_t)(ncol0 / 8 + o)) * 2 + kind] = v;
      }
    }
  }
  if (p.cluster) cluster_sync_all();  // the other CTAs' reads of this CTA's staging tile are complete before it exits
}

// split-K second pass: sum partials, add bias / residual, store.  One thread per 4 consecutive columns (float4 partial
// loads, splits unrolled by 4 for memory-level parallelism).
__global__ void conv_splitk_reduce_kernel(const ConvTcParams p, int m_tiles) {
  pdl_wait();
  pdl_launch_dependents();
  const int cq = (p.Cout + 3) / 4;
  const int64_t total = (int64_t)m_tiles * BM * cq;
  const size_t split_stride = (size_t)p.ws_rows * p.Npad;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int col = (int)(idx % cq) * 4;
    const int64_t trow = idx / cq;
    const int r = (int)(trow % BM);
    const int mt = (int)(trow / BM);
    const int tw_i = mt % p.tiles_w, th_i = (mt / p.tiles_w) % p.tiles_h, tn_i = mt / (p.tiles_w * p.tiles_h);
    const int w = tw_i * p.TW + r % p.TW, h = th_i * p.TH + (r / p.TW) % p.TH, n = tn_i * p.TN + r / (p.TW * p.TH);
    if (n >= p.NB || h >= p.H || w >= p.W) continue;
    const float* src = p.ws + (size_t)trow * p.Npad + col;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    int s = 0;
    for (; s + 4 <= p.splits; s += 4) {
      const float4 v0 = __ldcs(reinterpret_cast<const float4*>(src + (size_t)(s + 0) * split_stride));
      const float4 v1 = __ldcs(reinterpret_cast<const float4*>(src + (size_t)(s + 1) * split_stride));
      const float4 v2 = __ldcs(reinterpret_cast<const float4*>(src + (size_t)(s + 2) * split_stride));
      const float4 v3 = __ldcs(reinterpret_cast<const float4*>(src + (size_t)(s + 3) * split_stride));
      a.x += (v0.x + v1.x) + (v2.x + v3.x); a.y += (v0.y + v1.y) + (v2.y + v3.y);
      a.z += (v0.z + v1.z) + (v2.z + v3.z); a.w += (v0.w + v1.w) + (v2.w + v3.w);
    }
    for (; s < p.splits; ++s) {
      const float4 v = __ldcs(reinterpret_cast<const float4*>(src + (size_t)s * split_stride));
      a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
    }
    float acc[4] = {a.x, a.y, a.z, a.w};
    const int64_t o = (int64_t)n * p.out_sn + (int64_t)h * p.out_sh + (int64_t)w * p.out_sw;
    const int64_t ro = (int64_t)n * p.res_sn + (int64_t)h * p.res_sh + (int64_t)w * p.res_sw;
    if (col + 4 <= p.Cout && !p.out_f32 && p.out_sc == 1) {
      if (p.bias) {
        const float4 bv = *reinterpret_cast<const float4*>(p.bias + col);
        acc[0] += bv.x; acc[1] += bv.y; acc[2] += bv.z; acc[3] += bv.w;
      }
      if (p.res) {
        const __half2* rp = reinterpret_cast<const __half2*>(p.res + ro + col);
        const float2 r0 = __half22float2(rp[0]), r1 = __half22float2(rp[1]);
        acc[0] += r0.x; acc[1] += r0.y; acc[2] += r1.x; acc[3] += r1.y;
      }
      __half2* op = reinterpret_cast<__half2*>(reinterpret_cast<__half*>(p.out) + o + col);
      op[0] = __floats2half2_rn(acc[0], acc[1]);
      op[1] = __floats2half2_rn(acc[2], acc[3]);
    } else {
      for (int j = 0; j < 4 && col + j < p.Cout; ++j) {
        float v = acc[j];
        if (p.bias) v += p.bias[col + j];
        if (p.res) v += __half2float(p.res[ro + col + j]);
        if (p.out_f32) reinterpret_cast<float*>(p.out)[o + (col + j) * p.out_sc] = v;
        else reinterpret_cast<__half*>(p.out)[o + (col + j) * p.out_sc] = __float2half_rn(v);
      }
    }
  }
}

// ---------------------------------------------------------------- SIMT verification kernel
// Same contract, CUDA cores only, one thread per output element.  Exists so that GPU tests can
// cross-check the wgmma path layer by layer and so a tensor-core regression cannot block bring-up of the
// rest of the step; never selected by the shipped plans (impl = 0).
__global__ void conv_simt_kernel(const __half* __restrict__ A, const __half* __restrict__ Wp, const ConvTcParams p,
                                 int64_t a_sn, int64_t a_sh, int64_t a_sw, int64_t ldb, int64_t b_sh, int64_t b_sn) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t total = (int64_t)p.NB * p.H * p.W * p.Cout;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int co = (int)(idx % p.Cout);
    int64_t pix = idx / p.Cout;
    const int w = (int)(pix % p.W);
    pix /= p.W;
    const int h = (int)(pix % p.H);
    const int n = (int)(pix / p.H);
    float acc = 0.f;
    for (int tap = 0; tap < p.taps; ++tap) {
      const int dy = p.taps == 9 ? tap / 3 - 1 : 0, dx = p.taps == 9 ? tap % 3 - 1 : 0;
      const int yy = h + dy, xx = w + dx;
      if (yy < 0 || yy >= p.H || xx < 0 || xx >= p.W) continue;
      const __half2* a = reinterpret_cast<const __half2*>(A + n * a_sn + yy * a_sh + xx * a_sw);
      const __half2* wr = reinterpret_cast<const __half2*>(Wp + (int64_t)co * ldb + (int64_t)tap * p.Cin + (int64_t)h * b_sh + (int64_t)n * b_sn);
      for (int c = 0; c < p.Cin / 2; ++c) {
        const float2 av = __half22float2(a[c]), wv = __half22float2(wr[c]);
        acc = fmaf(av.x, wv.x, acc);
        acc = fmaf(av.y, wv.y, acc);
      }
    }
    if (p.bias) acc += p.bias[co];
    if (p.res) acc += __half2float(p.res[(int64_t)n * p.res_sn + (int64_t)h * p.res_sh + (int64_t)w * p.res_sw + co]);
    const int64_t o = (int64_t)n * p.out_sn + (int64_t)h * p.out_sh + (int64_t)w * p.out_sw + co * p.out_sc;
    if (p.out_f32) reinterpret_cast<float*>(p.out)[o] = acc;
    else reinterpret_cast<__half*>(p.out)[o] = __float2half_rn(acc);
  }
}

// ---------------------------------------------------------------- host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  }
  return fn;
}

static int pick_tile(int64_t W, int64_t H, int& TW, int& TH, int& TN) {
  // TW = smallest power of two >= min(W, 128); TH = largest power of two with TW*TH <= 128 not exceeding
  // the power-of-two ceiling of H; TN fills the remaining rows of the 128-pixel tile.
  int tw = 1;
  while (tw < W && tw < 128) tw <<= 1;
  int hceil = 1;
  while (hceil < H) hceil <<= 1;
  int th = 128 / tw;
  if (th > hceil) th = hceil;
  TW = tw;
  TH = th;
  TN = 128 / (tw * th);
  return 0;
}

int conv_tc_prepare(const CgdOp& op, ConvTcLaunch& L) {
  ConvTcParams& p = L.p;
  const int64_t NB = op.i[0], H = op.i[1], W = op.i[2], Cin = op.i[3], Cout = op.i[4], Npad = op.i[5], taps = op.i[6];
  const int64_t BN = op.i[16], splits = op.i[17] > 0 ? op.i[17] : 1;
  CGD_CHECK_ARG(NB > 0 && H > 0 && W > 0, "conv: bad image dims %lld %lld %lld", (long long)NB, (long long)H, (long long)W);
  // tile counts, pixel indices and the TMA box arithmetic below are 32-bit: reject sizes whose pixel count does not fit instead of
  // overflowing (a 2^31-row "image" used to spin in pick_tile's power-of-two search)
  CGD_CHECK_ARG(NB <= (1 << 24) && H <= (1 << 24) && W <= (1 << 24) && NB * H <= (int64_t)0x7fffffff && NB * H * W <= (int64_t)0x7fffffff && Cin <= (1 << 24) &&
                    Cout <= (1 << 24) && Npad <= (1 << 24),
                "conv: dims out of range (N %lld H %lld W %lld Cin %lld Cout %lld Npad %lld; N*H*W must fit 31 bits)", (long long)NB,
                (long long)H, (long long)W, (long long)Cin, (long long)Cout, (long long)Npad);
  CGD_CHECK_ARG(Cin > 0 && Cin % 64 == 0, "conv: Cin=%lld must be a positive multiple of 64", (long long)Cin);
  CGD_CHECK_ARG(taps == 1 || taps == 9, "conv: taps must be 1 or 9");
  CGD_CHECK_ARG(BN == 16 || BN == 32 || BN == 64 || BN == 128 || BN == 192 || BN == 256, "conv: unsupported BN=%lld", (long long)BN);
  CGD_CHECK_ARG(Npad % BN == 0 && Cout <= Npad && Cout > 0, "conv: Npad=%lld must be a multiple of BN=%lld and >= Cout=%lld",
                (long long)Npad, (long long)BN, (long long)Cout);
  CGD_CHECK_ARG(op.p[0] && op.p[1] && op.p[4], "conv: null A / W / out pointer");
  CGD_CHECK_ARG(((uintptr_t)op.p[0] % 16) == 0 && ((uintptr_t)op.p[1] % 16) == 0 && ((uintptr_t)op.p[4] % 16) == 0,
                "conv: A / W / out must be 16-byte aligned");
  for (int k = 7; k <= 9; ++k) CGD_CHECK_ARG(op.i[k] % 8 == 0, "conv: A strides must be multiples of 8 elements (16 B)");
  p.NB = (int)NB; p.H = (int)H; p.W = (int)W; p.Cin = (int)Cin; p.Cout = (int)Cout; p.Npad = (int)Npad; p.taps = (int)taps;
  pick_tile(W, H, p.TW, p.TH, p.TN);
  p.tiles_w = (int)ceil_div(W, p.TW);
  p.tiles_h = (int)ceil_div(H, p.TH);
  p.tiles_n = (int)ceil_div(NB, p.TN);
  p.kblocks = (int)(taps * Cin / 64);
  p.splits = (int)splits;
  CGD_CHECK_ARG(p.splits >= 1 && p.splits <= p.kblocks, "conv: splits=%d out of range (kblocks=%d)", p.splits, p.kblocks);
  p.kb_per_split = (int)ceil_div(p.kblocks, p.splits);
  p.splits = (int)ceil_div(p.kblocks, p.kb_per_split);  // no empty splits
  p.out_sn = op.i[10]; p.out_sh = op.i[11]; p.out_sw = op.i[12];
  p.res_sn = op.i[13]; p.res_sh = op.i[14]; p.res_sw = op.i[15];
  p.bias = reinterpret_cast<const float*>(op.p[2]);
  p.res = reinterpret_cast<const __half*>(op.p[3]);
  p.out = op.p[4];
  p.ws = reinterpret_cast<float*>(op.p[5]);
  p.out_f32 = (op.flags & 1) ? 1 : 0;
  p.out_sc = op.i[19] > 0 ? op.i[19] : 1;
  if (!p.out_f32 && p.out_sc == 1) CGD_CHECK_ARG(op.i[10] % 8 == 0 && op.i[11] % 8 == 0 && op.i[12] % 8 == 0, "conv: fp16 out strides must be multiples of 8");
  if (p.res) CGD_CHECK_ARG(op.i[13] % 8 == 0 && op.i[14] % 8 == 0 && op.i[15] % 8 == 0 && ((uintptr_t)p.res % 16) == 0, "conv: residual must be 16-byte aligned with strides %% 8 == 0");
  const bool want_cluster = op.i[23] == 1 && op.i[18] != 1;  // plan flag; the SIMT twin ignores it
  if (p.splits > 1 && !want_cluster) CGD_CHECK_ARG(p.ws != nullptr, "conv: split-K needs a workspace");
  p.cluster = 0;
  p.epi_stats = nullptr;  // set below when CONV flags 2 asks for epilogue statistics
  L.BN = (int)BN;
  L.impl = (int)op.i[18];
  L.A = reinterpret_cast<const __half*>(op.p[0]);
  L.Wp = reinterpret_cast<const __half*>(op.p[1]);
  L.a_sn = op.i[7]; L.a_sh = op.i[8]; L.a_sw = op.i[9];
  L.ldb = op.i[22] > 0 ? op.i[22] : taps * Cin; L.b_sh = op.i[20]; L.b_sn = op.i[21];
  L.m_tiles = p.tiles_w * p.tiles_h * p.tiles_n;
  p.ws_rows = L.m_tiles * BM;
  L.n_tiles = (int)(Npad / BN);
  if (L.impl == 1) return 0;

  PFN_encodeTiled enc = get_encode_fn();
  CGD_CHECK_ARG(enc != nullptr, "conv: cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)NB};
    cuuint64_t strides[3] = {(cuuint64_t)op.i[9] * 2, (cuuint64_t)op.i[8] * 2, (cuuint64_t)op.i[7] * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)p.TW, (cuuint32_t)p.TH, (cuuint32_t)p.TN};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(&L.tmA, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, op.p[0], dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CGD_CHECK_ARG(r == CUDA_SUCCESS, "conv: cuTensorMapEncodeTiled(A) failed with %d (dims %lld,%lld,%lld,%lld strides %lld,%lld,%lld box %d,%d,%d)",
                  (int)r, (long long)Cin, (long long)W, (long long)H, (long long)NB, (long long)strides[0], (long long)strides[1],
                  (long long)strides[2], p.TW, p.TH, p.TN);
  }
  const int64_t ldb = op.i[22] > 0 ? op.i[22] : taps * Cin;
  p.b_batched = (op.i[20] != 0 || op.i[21] != 0) ? 1 : 0;
  CGD_CHECK_ARG(ldb % 8 == 0 && op.i[20] % 8 == 0 && op.i[21] % 8 == 0, "conv: B strides must be multiples of 8 elements");
  if (p.b_batched) CGD_CHECK_ARG(p.TH == 1 && p.TN == 1, "conv: batched-B GEMMs need W > 64 (one (h, n) per 128-pixel tile)");
  {
    // 4-D map (K, rows, h, n) so batched GEMMs pick their B matrix by the tile's (h, n); plain weights use (0, 0)
    const cuuint64_t K = (cuuint64_t)(taps * Cin);
    const cuuint64_t row_bytes = (cuuint64_t)ldb * 2 * (cuuint64_t)Npad;
    cuuint64_t dims4[4] = {K, (cuuint64_t)Npad, (cuuint64_t)(p.b_batched ? H : 1), (cuuint64_t)(p.b_batched ? NB : 1)};
    cuuint64_t strides4[3] = {(cuuint64_t)ldb * 2, p.b_batched ? (cuuint64_t)op.i[20] * 2 : row_bytes, p.b_batched ? (cuuint64_t)op.i[21] * 2 : row_bytes};
    cuuint32_t box4[4] = {64, (cuuint32_t)BN, 1, 1};
    cuuint32_t estr4[4] = {1, 1, 1, 1};
    CUresult r = enc(&L.tmB, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, op.p[1], dims4, strides4, box4, estr4, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CGD_CHECK_ARG(r == CUDA_SUCCESS, "conv: cuTensorMapEncodeTiled(W) failed with %d", (int)r);
  }
  if (want_cluster) {
    CGD_CHECK_ARG(L.impl != 1 && !p.out_f32 && p.out_sc == 1 && !p.b_batched && p.Cout % 8 == 0 && L.BN >= 64 && p.splits >= 2 && p.splits <= 8 &&
                      L.BN % p.splits == 0 && (L.BN / p.splits) % 16 == 0,
                  "conv: layer flagged for cluster split-K is not eligible (BN=%d splits=%d Cout=%d f32=%d)", L.BN, p.splits, p.Cout, p.out_f32);
    p.cluster = 1;
  }
  // flags 4: the "residual" operand is a QuickGELU pre-activation u and the epilogue computes acc * QuickGELU'(u) instead of acc + res
  p.res_mode = 0;
  if (op.flags & 4) {
    CGD_CHECK_ARG(L.impl != 1 && p.splits == 1 && !p.out_f32 && p.out_sc == 1 && Cout % 8 == 0 && p.res != nullptr && p.bias == nullptr,
                  "conv: flags 4 (QuickGELU' epilogue) needs the tensor-core kernel without split-K, an fp16 contiguous output with Cout %% 8 == 0, a res "
                  "operand and no bias (BN=%d splits=%d Cout=%lld)", (int)BN, p.splits, (long long)Cout);
    p.res_mode = 1;
  }
  // flags 2: the epilogue also reduces its output tile to per-octet sums for the GroupNorm that follows (GN_APPLY_EPI): needs the
  // tensor-core kernel without split-K, fp16 contiguous output, and tiles that are full and are 128 consecutive pixels of one image
  p.epi_stats = nullptr;
  if (op.flags & 2) {
    CGD_CHECK_ARG(L.impl != 1 && p.splits == 1 && !p.out_f32 && p.out_sc == 1 && op.p[7] != nullptr && W % p.TW == 0 && H % p.TH == 0 && p.TN == 1 &&
                      (p.TW == W || p.TH == 1),
                  "conv: epilogue statistics need the tensor-core kernel without split-K, fp16 output and full 128-pixel tiles inside one image (W=%lld H=%lld tile %dx%dx%d)",
                  (long long)W, (long long)H, p.TW, p.TH, p.TN);
    p.epi_stats = reinterpret_cast<float*>(op.p[7]);
  }
  // <= 8 output channels, fp32 output, 3x3 (UNet head, stem dgrad): halo-tile mma.sync kernel (conv_narrow.cu); CGD_CONV_NARROW=0 keeps
  // the wgmma N = 16 tile for A/B runs
  {
    static int narrow_on = -1;
    if (narrow_on < 0) {
      const char* e = getenv("CGD_CONV_NARROW");
      narrow_on = (e && e[0] == '0') ? 0 : 1;
    }
    L.narrow = (narrow_on && conv_narrow_eligible(L)) ? 1 : 0;
  }
  // 8 x 8 images (deepest UNet level): one launch, a CTA per 8 output channels streaming its whole weight slab (conv_narrow.cu,
  // conv_small_kernel) instead of split-K tiles + a reduce launch.  Opt-in (CGD_CONV_SMALL=1): not measured against the wgmma
  // split-K path on the H100.
  {
    static int small_on = -1;
    if (small_on < 0) {
      const char* e = getenv("CGD_CONV_SMALL");
      small_on = (e && e[0] == '1') ? 1 : 0;
    }
    L.small = (small_on && !L.narrow && conv_small_eligible(L)) ? 1 : 0;
    L.tmS = L.tmA;
    if (L.small) {  // one TMA box per 64-channel slice: the 8 x 8 image with its zero border (out-of-image coordinates are zero-filled)
      const cuuint32_t e = taps == 9 ? 10 : 8;
      cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)NB};
      cuuint64_t strides[3] = {(cuuint64_t)op.i[9] * 2, (cuuint64_t)op.i[8] * 2, (cuuint64_t)op.i[7] * 2};
      cuuint32_t box[4] = {64, e, e, 1};
      cuuint32_t estr[4] = {1, 1, 1, 1};
      CUresult r = enc(&L.tmS, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, op.p[0], dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      CGD_CHECK_ARG(r == CUDA_SUCCESS, "conv: cuTensorMapEncodeTiled(8x8 image box) failed with %d", (int)r);
    }
  }
  return 0;
}

template <int BN>
static int set_smem_attr() {
  static DeviceOnce attr_set;
  if (attr_set.needed()) {
    CGD_CUDA(cudaFuncSetAttribute(conv_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<BN>::kSmemBytes));
    attr_set.mark();
  }
  return 0;
}

template <int BN>
static int launch_tc(const ConvTcLaunch& L, cudaStream_t st) {
  using Cfg = TcCfg<BN>;
  if (const int rc = set_smem_attr<BN>()) return rc;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)L.m_tiles, (unsigned)L.n_tiles, (unsigned)L.p.splits);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = Cfg::kSmemBytes;
  cfg.stream = st;
  cudaLaunchAttribute attrs[2];
  int na = 0;
  if (L.p.cluster) {  // the `splits` CTAs of one output tile form a cluster along z
    attrs[na].id = cudaLaunchAttributeClusterDimension;
    attrs[na].val.clusterDim.x = 1;
    attrs[na].val.clusterDim.y = 1;
    attrs[na].val.clusterDim.z = (unsigned)L.p.splits;
    ++na;
  }
  if (pdl_enabled()) {
    attrs[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attrs[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attrs;
  cfg.numAttrs = na;
  CGD_CUDA(cudaLaunchKernelEx(&cfg, conv_tc_kernel<BN>, L.tmA, L.tmB, L.p));
  return 0;
}

template <int BN>
static int max_clusters(int S) {
  if (set_smem_attr<BN>() != 0) {
    cudaGetLastError();
    return -1;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(64, 1, (unsigned)S);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = TcCfg<BN>::kSmemBytes;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = 1;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = (unsigned)S;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, conv_tc_kernel<BN>, &cfg) != cudaSuccess) {
    cudaGetLastError();
    return -1;
  }
  return n;
}
// co-resident clusters of S CTAs the device can hold for tile width BN (cudaOccupancyMaxActiveClusters); -1 without a device
int conv_cluster_capacity(int BN, int S) {
  if (S < 1 || S > 8) return -1;
  switch (BN) {
    case 64: return max_clusters<64>(S);
    case 128: return max_clusters<128>(S);
    case 192: return max_clusters<192>(S);
    case 256: return max_clusters<256>(S);
    default: return -1;
  }
}

// impl: 0 = auto, 1 = SIMT verification twin, 2 / 3 = the wgmma tile kernel for every layer (no narrow / 8 x 8 special kernels;
// the plan uses in-cluster split-K and the fused epilogues with 0 and 3 only)
int conv_tc_launch(const ConvTcLaunch& L, cudaStream_t st) {
  if (L.impl == 1) {
    const int64_t total = (int64_t)L.p.NB * L.p.H * L.p.W * L.p.Cout;
    const int blocks = (int)std::min<int64_t>(ceil_div(total, 256), (int64_t)device_sm_count() * 16);
    ConvTcParams p = L.p;
    p.splits = 1;
    CGD_CUDA(launch_pdl(conv_simt_kernel, dim3(blocks), dim3(256), 0, st, L.A, L.Wp, p, L.a_sn, L.a_sh, L.a_sw, L.ldb, L.b_sh, L.b_sn));
    return 0;
  }
  if (L.narrow) return conv_narrow_launch(L, st);
  if (L.small) return conv_small_launch(L, st);
  int rc = 0;
  switch (L.BN) {
    case 16: rc = launch_tc<16>(L, st); break;
    case 32: rc = launch_tc<32>(L, st); break;
    case 64: rc = launch_tc<64>(L, st); break;
    case 128: rc = launch_tc<128>(L, st); break;
    case 192: rc = launch_tc<192>(L, st); break;
    case 256: rc = launch_tc<256>(L, st); break;
    default: set_error("conv: unsupported BN %d", L.BN); return -1;
  }
  if (rc) return rc;
  if (L.p.splits > 1 && !L.p.cluster) {
    const int64_t total = (int64_t)L.m_tiles * BM * ((L.p.Cout + 3) / 4);
    const int blocks = (int)std::min<int64_t>(ceil_div(total, 256), (int64_t)device_sm_count() * 8);
    CGD_CUDA(launch_pdl(conv_splitk_reduce_kernel, dim3(blocks), dim3(256), 0, st, L.p, L.m_tiles));
  }
  return 0;
}

int conv_tc_num_launches(const ConvTcLaunch& L) {
  return (L.impl != 1 && !L.small && !L.narrow && L.p.splits > 1 && !L.p.cluster) ? 2 : 1;
}

}  // namespace cgd
