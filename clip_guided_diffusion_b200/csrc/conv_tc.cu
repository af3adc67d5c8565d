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
// Launches without split-K that write fp16 channel-contiguous outputs (every wide UNet / ViT layer) run the persistent variant
// `conv_tc_persistent_kernel`: one CTA per SM walks its tiles with the ring carried over; its epilogue goes through an fp16 staging
// tile outside the ring that the TMA unit fills with the residual during the K loop and stores from, so the producer loads the
// next tile while the consumers finish the last one, and the consumers do not wait for their stores.
// conv_tc_kernel's epilogue: the accumulators go to an fp32 staging tile that reuses the ring; then each consumer thread
// owns one pixel row and half of the tile's channels and adds bias / residual, stores fp16 / fp32 (split-K:
// one 8-channel chunk of a row per pass, neighbouring threads on neighbouring chunks).
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
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(kStagingBytes <= kStages * kStageBytes, "the fp32 staging tile reuses the operand ring");
  static_assert(kSmemBytes <= 227 * 1024, "H100: at most 227 KB of shared memory per block");
};

// Phase stamps of conv_tc_persistent_kernel, compiled in only with -DCGD_CONV_PHASES (scripts/conv_tile_phases.py builds that
// variant; the default build has none of it).  Per CTA and tile slot, %globaltimer ns: [0] consumer thread 0 enters the tile's
// K loop, [1] its first full-barrier pass, [2] the end of its K loop (after wgmma wait_group 0), [3] the end of its epilogue,
// [4] the producer's time blocked on empty barriers while loading the tile.  Later launches overwrite earlier ones.
#ifdef CGD_CONV_PHASES
constexpr int kPhaseCtas = 256, kPhaseTiles = 32, kPhaseFields = 5;
__device__ unsigned long long g_conv_phases[kPhaseCtas * kPhaseTiles * kPhaseFields];
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void phase_stamp(int slot, int field, unsigned long long v) {
  if (blockIdx.x < kPhaseCtas && slot < kPhaseTiles) g_conv_phases[(blockIdx.x * kPhaseTiles + slot) * kPhaseFields + field] = v;
}
#define CGD_PHASE(...) __VA_ARGS__
#else
#define CGD_PHASE(...)
#endif

// Origin (w0, h0, n0) in the image grid of pixel tile mt.
__device__ __forceinline__ void tile_origin(const ConvTcParams& p, int mt, int& w0, int& h0, int& n0) {
  const int tw_i = mt % p.tiles_w;
  const int th_i = (mt / p.tiles_w) % p.tiles_h;
  const int tn_i = mt / (p.tiles_w * p.tiles_h);
  w0 = tw_i * p.TW;
  h0 = th_i * p.TH;
  n0 = tn_i * p.TN;
}

// TMA producer, one tile: K-blocks [kb0, kb1) of the pixel tile at (w0, h0, n0) and output columns [ncol0, ncol0 + BN) into the
// ring.  (stage, phase) is the producer's ring position; it advances and carries over to the next tile.  Returns the ns spent
// blocked on empty barriers under CGD_CONV_PHASES, else 0.
template <int BN, int STAGES = TcCfg<BN>::kStages>
__device__ __forceinline__ unsigned long long produce_kblocks(const CUtensorMap* tmA, const CUtensorMap* tmB, uint8_t* smem_a, uint8_t* smem_b,
                                                              uint64_t* full_bar, uint64_t* empty_bar, const ConvTcParams& p, int kb0, int kb1,
                                                              int w0, int h0, int n0, int ncol0, int& stage, uint32_t& phase) {
  using Cfg = TcCfg<BN>;
  const int cblks = p.Cin / BK;
  unsigned long long blocked = 0;
  for (int kb = kb0; kb < kb1; ++kb) {
    CGD_PHASE(const unsigned long long tw = globaltimer_ns();)
    mbar_wait_trap(&empty_bar[stage], phase ^ 1);
    CGD_PHASE(blocked += globaltimer_ns() - tw;)
    mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
    const int tap = kb / cblks, cb = kb - tap * cblks;
    int dy = 0, dx = 0;
    if (p.taps == 9) {
      dy = tap / 3 - 1;
      dx = tap % 3 - 1;
    }
    tma_load_4d(smem_a + stage * Cfg::kABytes, tmA, &full_bar[stage], cb * BK, w0 + dx, h0 + dy, n0);
    tma_load_4d(smem_b + stage * Cfg::kBBytes, tmB, &full_bar[stage], kb * BK, ncol0, 0, 0);
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
  return blocked;
}

// Consumer warpgroup wg, one tile: acc = the sum over K-blocks [kb0, kb1) read from the ring at (stage, phase), which advance.
// A stage is released once the wgmma group that read it has retired; the last stage is returned unreleased, and every wgmma of
// the tile has retired on return.  after_first() runs once the first K-block's wgmma group has been issued.
template <int BN, int STAGES = TcCfg<BN>::kStages, class AfterFirst>
__device__ __forceinline__ int consume_kblocks(float* acc, const uint8_t* smem_a, const uint8_t* smem_b, uint64_t* full_bar,
                                               uint64_t* empty_bar, int wg, int lane, int kb0, int kb1, int& stage, uint32_t& phase,
                                               AfterFirst after_first) {
  using Cfg = TcCfg<BN>;
  int prev = -1;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait_trap(&full_bar[stage], phase);
    const uint64_t da = make_wgmma_desc_sw128(smem_u32(smem_a + stage * Cfg::kABytes + wg * 64 * 128));
    const uint64_t db = make_wgmma_desc_sw128(smem_u32(smem_b + stage * Cfg::kBBytes));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k)  // advance 16 elements (32 B) along K inside the 128 B swizzle row: +2 in the (>>4) address field
      wgmma_f16<BN>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb > kb0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    if (kb == kb0) after_first();
    wgmma_wait<1>();  // the group of the previous stage has retired: its operands may be overwritten
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
    }
    prev = stage;
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
  wgmma_wait<0>();
#pragma unroll
  for (int j = 0; j < BN / 2; ++j) wgmma_fence_operand(acc[j]);
  return prev;
}

// CONV flags 4: acc * QuickGELU'(u), u = the QuickGELU pre-activation read through the residual path
__device__ __forceinline__ float qgelu_grad_mul(float a, float u) {
  const float sg = rcp_ftz(1.f + ex2_ftz(-1.702f * 1.4426950408889634f * u));  // sigmoid(1.702 u), MUFU ex2 + rcp
  return a * (sg * fmaf(1.702f * u, 1.f - sg, 1.f));
}

// CONV flags 8: acc * GELU'(u) = acc * (Phi(u) + u phi(u)), the exact (erf) GELU of the OpenCLIP towers
__device__ __forceinline__ float gelu_grad_mul(float a, float u) {
  const float cdf = 0.5f * erfcf(u * -0.70710678118654752f);  // Phi(u) without the cancellation 1 + erf(.) has for u << 0
  const float pdf = 0.39894228040143268f * __expf(-0.5f * u * u);
  return a * fmaf(u, pdf, cdf);
}

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

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // ---- tile coordinates
  const int mt = blockIdx.x;
  int w0, h0, n0;
  tile_origin(p, mt, w0, h0, n0);
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
      int stage = 0;
      uint32_t phase = 0;
      produce_kblocks<BN>(&tmA, &tmB, smem_a, smem_b, full_bar, empty_bar, p, kb0, kb1, w0, h0, n0, ncol0, stage, phase);
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
    int stage = 0;
    uint32_t phase = 0;
    consume_kblocks<BN>(acc, smem_a, smem_b, full_bar, empty_bar, wg, lane, kb0, kb1, stage, phase, [] {});
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
    // ===== epilogue: 8 consecutive columns c of pixel row r at a time
    const int S = p.cluster ? p.splits : 1;
    const int cw = BN / S;  // columns finished by this CTA (a multiple of 16: host)
    const int c_base = p.cluster ? (int)cluster_ctarank() * cw : 0;
    const bool vec_ok = !p.out_f32 && p.out_sc == 1;
    const bool to_ws = p.splits > 1 && !p.cluster;
    auto finish8 = [&](const int r, const int c) {
      const int w_off = r % p.TW, h_off = (r / p.TW) % p.TH, n_off = r / (p.TW * p.TH);
      const int n = n0 + n_off, h = h0 + h_off, w = w0 + w_off;
      const bool row_ok = (n < p.NB) && (h < p.H) && (w < p.W);
      const float* srow = staging + (size_t)r * Cfg::kStageLd;
      const int64_t o_off = (int64_t)n * p.out_sn + (int64_t)h * p.out_sh + (int64_t)w * p.out_sw;
      const int64_t r_off = (int64_t)n * p.res_sn + (int64_t)h * p.res_sh + (int64_t)w * p.res_sw;
      float a[8];
      // chunks with bit 5 of c set read their upper 4 columns first: with 8-column chunks side by side in a warp, the two float4
      // reads then spread over all 8 16-byte bank groups (4 wavefronts each instead of 8)
      const bool swap = (c & 32) != 0;
      if (p.cluster) {  // fixed order over the cluster's partial tiles: bit-reproducible
#pragma unroll
        for (int e = 0; e < 8; ++e) a[e] = 0.f;
        const uint32_t local = smem_u32(srow + c);
        for (int j = 0; j < S; ++j) {
          const uint32_t remote = mapa_u32(local, (uint32_t)j);
          float4 u0 = ld_cluster_f4(remote + (swap ? 16 : 0)), u1 = ld_cluster_f4(remote + (swap ? 0 : 16));
          if (swap) { const float4 tmp = u0; u0 = u1; u1 = tmp; }
          a[0] += u0.x; a[1] += u0.y; a[2] += u0.z; a[3] += u0.w;
          a[4] += u1.x; a[5] += u1.y; a[6] += u1.z; a[7] += u1.w;
        }
      } else {
        float4 u0 = *reinterpret_cast<const float4*>(srow + c + (swap ? 4 : 0)), u1 = *reinterpret_cast<const float4*>(srow + c + (swap ? 0 : 4));
        if (swap) { const float4 tmp = u0; u0 = u1; u1 = tmp; }
        a[0] = u0.x; a[1] = u0.y; a[2] = u0.z; a[3] = u0.w;
        a[4] = u1.x; a[5] = u1.y; a[6] = u1.z; a[7] = u1.w;
      }
      if (to_ws) {  // raw fp32 partials -> workspace [split][tile row][Npad]; rows outside the image are never read back
        if (row_ok) {
          float* ws = p.ws + ((size_t)blockIdx.z * p.ws_rows + (size_t)mt * BM + r) * p.Npad + ncol0;
          *reinterpret_cast<float4*>(ws + c) = make_float4(a[0], a[1], a[2], a[3]);
          *reinterpret_cast<float4*>(ws + c + 4) = make_float4(a[4], a[5], a[6], a[7]);
        }
        return;
      }
      const int col = ncol0 + c;
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
            if (p.res_mode == 1) {
#pragma unroll
              for (int e = 0; e < 8; ++e) a[e] = qgelu_grad_mul(a[e], rr[e]);
            } else {
#pragma unroll
              for (int e = 0; e < 8; ++e) a[e] += rr[e];
            }
          }
          st8(reinterpret_cast<__half*>(p.out) + o_off + col, pack8(a));
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
    };
    if (p.cluster || to_ws) {
      // split-K: consecutive threads take consecutive 8-column chunks of one row, so a warp's fp32 partial stores to the workspace
      // (or its distributed-shared-memory reads of the cluster's staging rows) cover contiguous runs of a row; with one pixel row
      // per thread every 32-byte partial store of a warp lands on 32 rows (on an H100 the workspace split-K 3x3 convs of the
      // 32 x 32 and 16 x 16 levels took 1.4-1.5x as long)
      const int cpr = cw / 8;              // chunks per row
      const int rows_per_pass = kConsumers / cpr;
      const int t = threadIdx.x;
      if (t < rows_per_pass * cpr) {
        const int c = c_base + (t % cpr) * 8;
#pragma unroll 1
        for (int r = t / cpr; r < BM; r += rows_per_pass) finish8(r, c);
      }
    } else {
      // thread = (pixel row r, half of the columns): measured faster than the chunk mapping above on the one-CTA 256 x 256 layers,
      // and the coalesced order for channel-strided (NCHW fp32) outputs.  Launches that reach it: fp32 or channel-strided outputs
      // and Cout % 8 != 0; every other one-CTA launch runs conv_tc_persistent_kernel
      const int r = (warp & 3) * 32 + lane, half = warp >> 2;
      const int c_lo = c_base + half * (cw / 2), c_hi = c_lo + cw / 2;
#pragma unroll 1
      for (int c = c_lo; c < c_hi; c += 8) finish8(r, c);
    }
  }
  if (p.cluster) cluster_sync_all();  // the other CTAs' reads of this CTA's staging tile are complete before it exits
}

// ---------------------------------------------------------------- persistent one-CTA kernel
// The launches without split-K and with an fp16 channel-contiguous output (Cout % 8 == 0): grid = min(tiles, SMs), CTA b owns the
// tiles b, b + gridDim.x, ... of the (pixel tile, column tile) sequence, pixel tiles fastest.  The producer runs straight on into
// the next tile's K-blocks; ring stage and phase carry over.  The consumers' K loop is conv_tc_kernel's.  Their epilogue goes
// through a staging tile outside the ring, so the producer refills the ring meanwhile:
//   * the staging tile is the 128 x BN fp16 output tile as BN / 64 TMA boxes of 64 channels in the 128-byte-swizzled layout
//     (narrower boxes and swizzles at BN < 64); at BN 256 it holds one 128-column half at a time, the two halves stored in turn,
//     the second half's residual loaded by consumer thread 0 once the first half's store has been read out;
//   * the producer lane TMA-loads a tile's residual into it while the consumers run that tile's K loop, once the previous tile's
//     store has been read out of it (`stg_free`), and signals `stg_full` (with the transaction bytes; a plain arrive without a
//     residual);
//   * the consumers add bias, then residual or QuickGELU' in fp32 registers (the same operations in the same order as
//     conv_tc_kernel), round once to fp16 and write the result in place; after a named barrier consumer thread 0 TMA-stores the
//     tile (the TMA unit clips rows outside the image and columns >= Cout) and the consumers go on into the next K loop;
//   * thread 0 waits for that store to be read out of shared memory after issuing the next tile's first wgmma group, then
//     arrives on `stg_free`; it drains its stores before the CTA exits.
// Results are bitwise those of conv_tc_kernel.
template <int BN>
struct PersistCfg {
  using Ring = TcCfg<BN>;
  static constexpr int kStages = Ring::kStages;
  // at BN 256 four 48 KB stages and a 64 KB staging tile exceed 227 KB: the staging tile holds one 128-column half at a time (measured
  // against a 3-stage ring with the whole tile staged: DESIGN §4)
  static constexpr int kHalves = BN == 256 ? 2 : 1;
  static constexpr int kBoxC = BN < 64 ? BN : 64;                // channels per staging box: one 128-byte swizzle row at BN >= 64
  static constexpr int kRowBytes = kBoxC * 2;
  static constexpr int kSwMask = kRowBytes / 16 - 1;             // swizzle span 128 / 64 / 32 bytes: XOR of 3 / 2 / 1 chunk-index bits
  static constexpr int kBoxBytes = BM * kRowBytes;
  static constexpr int kBoxes = BN / kBoxC;
  static constexpr int kStgOff = kStages * Ring::kStageBytes;    // a multiple of 1024: the swizzle pattern's alignment
  static constexpr int kStgBoxes = kBoxes / kHalves;
  static constexpr int kBiasOff = kStgOff + kStgBoxes * kBoxBytes;
  static constexpr int kBarOff = kBiasOff + BN * 4;
  static constexpr int kSmemBytes = kBarOff + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(kStgOff % 1024 == 0 && kBoxBytes % 1024 == 0, "staging boxes must start on a 1024-byte boundary");
  static_assert(kSmemBytes <= 227 * 1024, "H100: at most 227 KB of shared memory per block");
  // byte offset of (row r, byte b of the row) in a staging box: the TMA unit's swizzle (16-byte chunk index ^= bits 7.. of the offset)
  static __device__ __forceinline__ int swz(int r, int b) {
    const int off = r * kRowBytes + b;
    return off ^ (((off >> 7) & kSwMask) << 4);
  }
};

// EXACT_GELU: the instantiation that runs CONV flags 8 (res_mode 2); the other one keeps its registers free of erff / expf
template <int BN, bool EXACT_GELU = false>
__global__ void __launch_bounds__(kThreads, 1)
conv_tc_persistent_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                          const __grid_constant__ CUtensorMap tmOut, const __grid_constant__ CUtensorMap tmRes, const ConvTcParams p) {
  using Cfg = PersistCfg<BN>;
  constexpr int S = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + S * Cfg::Ring::kABytes;
  uint8_t* stg = smem + Cfg::kStgOff;
  float* bias_s = reinterpret_cast<float*>(smem + Cfg::kBiasOff);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kBarOff);
  uint64_t* empty_bar = full_bar + S;
  uint64_t* stg_free = empty_bar + S;  // the previous tile's store has been read out of the staging tile
  uint64_t* stg_full = stg_free + 1;   // the staging tile holds this tile's residual (or is merely free, without one)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tiles = p.m_tiles, tiles = p.tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmOut);
    if (p.res) tma_prefetch_desc(&tmRes);
    for (int s = 0; s < S; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kConsumers / 32);  // one arrive per consumer warp
    }
    mbar_init(stg_free, 1);
    mbar_init(stg_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();

  if (warp == kConsumers / 32) {
    // ===== TMA producer
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      // the residual goes in from the end of the first ring-full of K-blocks: by then the consumers are in this tile's K loop, so the
      // previous tile's store is issued.  Its boxes are spread over the rest of the K loop, one every `step` K-blocks, so that they
      // do not arrive in one burst on top of the operand loads
      const int kres = min(S, p.kblocks);
      for (int t = blockIdx.x, i = 0; t < tiles; t += gridDim.x, ++i) {
        int w0, h0, n0;
        tile_origin(p, t % m_tiles, w0, h0, n0);
        const int ncol0 = (t / m_tiles) * BN;
        unsigned long long blocked =
            produce_kblocks<BN, S>(&tmA, &tmB, smem_a, smem_b, full_bar, empty_bar, p, 0, kres, w0, h0, n0, ncol0, stage, phase);
        if (i > 0) mbar_wait_trap(stg_free, (i - 1) & 1);
        int kb = kres;
        // boxes wholly beyond Cout are skipped (a column tile may lie wholly beyond it when Npad - Cout >= BN)
        const int nb = max(0, min(Cfg::kStgBoxes, (p.Cout - ncol0 + Cfg::kBoxC - 1) / Cfg::kBoxC));
        if (p.res && nb > 0) {
          const int step = (p.kblocks - kres) / nb;
          mbar_expect_tx(stg_full, nb * Cfg::kBoxBytes);
          for (int b = 0; b < nb; ++b) {
            const int kb_next = kres + b * step;
            blocked += produce_kblocks<BN, S>(&tmA, &tmB, smem_a, smem_b, full_bar, empty_bar, p, kb, kb_next, w0, h0, n0, ncol0, stage, phase);
            kb = kb_next;
            tma_load_4d(stg + b * Cfg::kBoxBytes, &tmRes, stg_full, ncol0 + b * Cfg::kBoxC, w0, h0, n0);
          }
        } else {
          mbar_arrive(stg_full);
        }
        blocked += produce_kblocks<BN, S>(&tmA, &tmB, smem_a, smem_b, full_bar, empty_bar, p, kb, p.kblocks, w0, h0, n0, ncol0, stage, phase);
        CGD_PHASE(phase_stamp(i, 4, blocked);)
        (void)blocked;
      }
    } else if (p.pf_bytes > 0) {
      l2_prefetch_slice(p.pf_ptr, p.pf_bytes, (int)blockIdx.x, (int)gridDim.x, lane - 1, 31);
    }
  } else {
    // ===== consumer warpgroup wg: pixel rows [64 wg, 64 wg + 64) of every tile; this thread's fragment rows r0 and r0 + 8
    const int wg = warp >> 2;
    const int fr = lane >> 2, fc = 2 * (lane & 3);  // accumulator fragment: rows fr, fr + 8, columns fc, fc + 1 of every 8
    const int r0 = warp * 16 + fr;
    float acc[BN / 2];
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
    int stage = 0;
    uint32_t phase = 0, sp = 0;
    for (int t = blockIdx.x, i = 0; t < tiles; t += gridDim.x, ++i) {
      const int mt = t % m_tiles, ncol0 = (t / m_tiles) * BN;
      // this thread's bias column, in flight during the K loop
      const float bias_v = (p.bias && threadIdx.x < BN && ncol0 + (int)threadIdx.x < p.Cout) ? __ldg(p.bias + ncol0 + threadIdx.x) : 0.f;
      CGD_PHASE(if (threadIdx.x == 0) phase_stamp(i, 0, globaltimer_ns());)
      const int last = consume_kblocks<BN, S>(acc, smem_a, smem_b, full_bar, empty_bar, wg, lane, 0, p.kblocks, stage, phase, [&] {
        CGD_PHASE(if (threadIdx.x == 0) phase_stamp(i, 1, globaltimer_ns());)
        // the previous tile's store must be read out of the staging tile before the producer may refill it.  Waiting here, with this
        // tile's first wgmma group in flight, stalls warp 0 (and through its stage releases the producer) only while that read-out
        // is still running; the phase stamps show no longer operand wait at tile start
        if (threadIdx.x == 0 && i > 0) {
          bulk_wait_read<0>();
          mbar_arrive(stg_free);
        }
      });
      CGD_PHASE(if (threadIdx.x == 0) phase_stamp(i, 2, globaltimer_ns());)
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[last]);

      if (p.bias) {  // every consumer has finished the previous tile's epilogue (named barrier 1), so bias_s is free
        if (threadIdx.x < BN) bias_s[threadIdx.x] = bias_v;
        named_bar_sync(2, kConsumers);
      }
      int w0, h0, n0;
      tile_origin(p, mt, w0, h0, n0);
#pragma unroll
      for (int h = 0; h < Cfg::kHalves; ++h) {
        const int bbase = h * Cfg::kStgBoxes;
        const int nbh = max(0, min(Cfg::kStgBoxes, (p.Cout - ncol0 + Cfg::kBoxC - 1) / Cfg::kBoxC - bbase));
        if (h > 0 && threadIdx.x == 0) {  // the first half's store must be read out before the second half's residual lands
          bulk_wait_read<0>();
          if (p.res && nbh > 0) {
            mbar_expect_tx(stg_full, nbh * Cfg::kBoxBytes);
            for (int b = 0; b < nbh; ++b) tma_load_4d(stg + b * Cfg::kBoxBytes, &tmRes, stg_full, ncol0 + (bbase + b) * Cfg::kBoxC, w0, h0, n0);
          } else {
            mbar_arrive(stg_full);
          }
        }
        mbar_wait_trap(stg_full, sp);
        sp ^= 1;
#pragma unroll
        for (int j = h * BN / 8 / Cfg::kHalves; j < (h + 1) * BN / 8 / Cfg::kHalves; ++j) {
          if (ncol0 + 8 * j < p.Cout) {
            float v0 = acc[4 * j], v1 = acc[4 * j + 1], v2 = acc[4 * j + 2], v3 = acc[4 * j + 3];
            if (p.bias) {
              const float2 b = *reinterpret_cast<const float2*>(bias_s + 8 * j + fc);
              v0 += b.x; v1 += b.y; v2 += b.x; v3 += b.y;
            }
            uint8_t* box = stg + (8 * j / Cfg::kBoxC - bbase) * Cfg::kBoxBytes;
            const int cb = 2 * (8 * j % Cfg::kBoxC + fc);
            __half2* lo = reinterpret_cast<__half2*>(box + Cfg::swz(r0, cb));
            __half2* hi = reinterpret_cast<__half2*>(box + Cfg::swz(r0 + 8, cb));
            if (p.res) {
              const float2 u0 = __half22float2(*lo), u1 = __half22float2(*hi);
              if constexpr (EXACT_GELU) {
                v0 = gelu_grad_mul(v0, u0.x); v1 = gelu_grad_mul(v1, u0.y);
                v2 = gelu_grad_mul(v2, u1.x); v3 = gelu_grad_mul(v3, u1.y);
              } else if (p.res_mode == 1) {
                v0 = qgelu_grad_mul(v0, u0.x); v1 = qgelu_grad_mul(v1, u0.y);
                v2 = qgelu_grad_mul(v2, u1.x); v3 = qgelu_grad_mul(v3, u1.y);
              } else {
                v0 += u0.x; v1 += u0.y; v2 += u1.x; v3 += u1.y;
              }
            }
            *lo = __floats2half2_rn(v0, v1);
            *hi = __floats2half2_rn(v2, v3);
          }
        }
        fence_proxy_async_smem();  // this half's generic-proxy writes, before the TMA unit reads them
        named_bar_sync(1, kConsumers);
        if (threadIdx.x == 0) {
          for (int b = 0; b < nbh; ++b) tma_store_4d(&tmOut, stg + b * Cfg::kBoxBytes, ncol0 + (bbase + b) * Cfg::kBoxC, w0, h0, n0);
          bulk_commit();
        }
      }
      CGD_PHASE(if (threadIdx.x == 0) phase_stamp(i, 3, globaltimer_ns());)
    }
    if (threadIdx.x == 0) bulk_wait<0>();  // the CTA's stores are complete before its shared memory is released
  }
  // every store of this CTA has completed: a dependent launch may take the SM
  pdl_launch_dependents();
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
                                 int64_t a_sn, int64_t a_sh, int64_t a_sw, int64_t ldb) {
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
      const __half2* wr = reinterpret_cast<const __half2*>(Wp + (int64_t)co * ldb + (int64_t)tap * p.Cin);
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
  CGD_CHECK_ARG(op.i[20] == 0 && op.i[21] == 0 && op.i[22] == 0 && (op.flags & 2) == 0, "conv: i20..i22 and flags 2 are reserved and must be 0");
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
  L.BN = (int)BN;
  L.impl = (int)op.i[18];
  L.narrow = 0;
  L.persistent = 0;
  L.A = reinterpret_cast<const __half*>(op.p[0]);
  L.Wp = reinterpret_cast<const __half*>(op.p[1]);
  L.a_sn = op.i[7]; L.a_sh = op.i[8]; L.a_sw = op.i[9];
  L.ldb = taps * Cin;
  L.m_tiles = p.tiles_w * p.tiles_h * p.tiles_n;
  p.ws_rows = L.m_tiles * BM;
  L.n_tiles = (int)(Npad / BN);
  p.m_tiles = L.m_tiles;
  p.tiles = L.m_tiles * L.n_tiles;
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
  {
    // [Npad, K] weights as a 4-D map with unit outer dimensions (the kernel's loads are 4-D)
    const cuuint64_t K = (cuuint64_t)L.ldb;
    const cuuint64_t row_bytes = K * 2 * (cuuint64_t)Npad;
    cuuint64_t dims4[4] = {K, (cuuint64_t)Npad, 1, 1};
    cuuint64_t strides4[3] = {K * 2, row_bytes, row_bytes};
    cuuint32_t box4[4] = {64, (cuuint32_t)BN, 1, 1};
    cuuint32_t estr4[4] = {1, 1, 1, 1};
    CUresult r = enc(&L.tmB, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, op.p[1], dims4, strides4, box4, estr4, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CGD_CHECK_ARG(r == CUDA_SUCCESS, "conv: cuTensorMapEncodeTiled(W) failed with %d", (int)r);
  }
  if (want_cluster) {
    CGD_CHECK_ARG(L.impl != 1 && !p.out_f32 && p.out_sc == 1 && p.Cout % 8 == 0 && L.BN >= 64 && p.splits >= 2 && p.splits <= 8 &&
                      L.BN % p.splits == 0 && (L.BN / p.splits) % 16 == 0,
                  "conv: layer flagged for cluster split-K is not eligible (BN=%d splits=%d Cout=%d f32=%d)", L.BN, p.splits, p.Cout, p.out_f32);
    p.cluster = 1;
  }
  // flags 4: the "residual" operand is a QuickGELU pre-activation u and the epilogue computes acc * QuickGELU'(u) instead of acc + res;
  // flags 8: the same with the exact GELU'(u) = Phi(u) + u phi(u)
  p.res_mode = 0;
  CGD_CHECK_ARG((op.flags & 12) != 12, "conv: flags 4 (QuickGELU') and 8 (GELU') exclude each other");
  if (op.flags & 12) {
    CGD_CHECK_ARG(L.impl != 1 && p.splits == 1 && !p.out_f32 && p.out_sc == 1 && Cout % 8 == 0 && p.res != nullptr && p.bias == nullptr,
                  "conv: flags %d (GELU' epilogue) needs the tensor-core kernel without split-K, an fp16 contiguous output with Cout %% 8 == 0, a res "
                  "operand and no bias (BN=%d splits=%d Cout=%lld)", op.flags & 12, (int)BN, p.splits, (long long)Cout);
    p.res_mode = (op.flags & 4) ? 1 : 2;
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
  L.persistent = (!L.narrow && p.splits == 1 && !p.cluster && !p.out_f32 && p.out_sc == 1 && p.Cout % 8 == 0) ? 1 : 0;
  CGD_CHECK_ARG(p.res_mode != 2 || (L.persistent && BN >= 64), "conv: flags 8 (GELU' epilogue) runs on the persistent kernel with BN >= 64 (BN=%d)", (int)BN);
  if (L.persistent) {
    // output / residual boxes of the persistent epilogue: 128 pixels x min(BN, 64) channels, swizzled like the staging tile.  The C
    // extent is Cout, so the TMA unit clips padded columns and pixels outside the image; channel slices are a base pointer plus
    // the row strides checked above
    const cuuint32_t boxc = (cuuint32_t)std::min<int64_t>(BN, 64);
    const CUtensorMapSwizzle sw = boxc == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : boxc == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
    auto encode_io = [&](CUtensorMap* tm, const void* ptr, int64_t sn, int64_t sh, int64_t sw_, const char* what) {
      cuuint64_t dims[4] = {(cuuint64_t)Cout, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)NB};
      cuuint64_t strides[3] = {(cuuint64_t)sw_ * 2, (cuuint64_t)sh * 2, (cuuint64_t)sn * 2};
      cuuint32_t box[4] = {boxc, (cuuint32_t)p.TW, (cuuint32_t)p.TH, (cuuint32_t)p.TN};
      cuuint32_t estr[4] = {1, 1, 1, 1};
      CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       sw, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      CGD_CHECK_ARG(r == CUDA_SUCCESS, "conv: cuTensorMapEncodeTiled(%s) failed with %d (strides %lld,%lld,%lld)", what, (int)r,
                    (long long)sw_, (long long)sh, (long long)sn);
      return 0;
    };
    if (const int rc = encode_io(&L.tmOut, p.out, p.out_sn, p.out_sh, p.out_sw, "out")) return rc;
    if (p.res) {
      if (const int rc = encode_io(&L.tmRes, p.res, p.res_sn, p.res_sh, p.res_sw, "res")) return rc;
    }
  }
  return 0;
}

template <int BN>
static int set_smem_attr() {
  static DeviceOnce attr_set;
  if (attr_set.needed()) {
    CGD_CUDA(cudaFuncSetAttribute(conv_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<BN>::kSmemBytes));
    CGD_CUDA(cudaFuncSetAttribute(conv_tc_persistent_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, PersistCfg<BN>::kSmemBytes));
    if constexpr (BN >= 64)
      CGD_CUDA(cudaFuncSetAttribute(conv_tc_persistent_kernel<BN, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, PersistCfg<BN>::kSmemBytes));
    attr_set.mark();
  }
  return 0;
}

template <int BN>
static int launch_tc(const ConvTcLaunch& L, cudaStream_t st) {
  if (const int rc = set_smem_attr<BN>()) return rc;
  cudaLaunchConfig_t cfg = {};
  if (L.persistent) {
    cfg.gridDim = dim3((unsigned)std::min(L.m_tiles * L.n_tiles, device_sm_count()));
    cfg.dynamicSmemBytes = PersistCfg<BN>::kSmemBytes;
  } else {
    cfg.gridDim = dim3((unsigned)L.m_tiles, (unsigned)L.n_tiles, (unsigned)L.p.splits);
    cfg.dynamicSmemBytes = TcCfg<BN>::kSmemBytes;
  }
  cfg.blockDim = dim3(kThreads);
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
  if (L.persistent && L.p.res_mode == 2) {
    if constexpr (BN >= 64) CGD_CUDA(cudaLaunchKernelEx(&cfg, conv_tc_persistent_kernel<BN, true>, L.tmA, L.tmB, L.tmOut, L.tmRes, L.p));
    else CGD_CHECK_ARG(false, "conv: flags 8 (GELU' epilogue) needs BN >= 64, got %d", BN);
  } else if (L.persistent) {
    CGD_CUDA(cudaLaunchKernelEx(&cfg, conv_tc_persistent_kernel<BN>, L.tmA, L.tmB, L.tmOut, L.tmRes, L.p));
  } else {
    CGD_CUDA(cudaLaunchKernelEx(&cfg, conv_tc_kernel<BN>, L.tmA, L.tmB, L.p));
  }
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

// impl: 0 = auto, 1 = SIMT verification twin, 2 / 3 = the wgmma tile kernel for every layer (no narrow special kernel;
// the plan uses in-cluster split-K and the fused epilogues with 0 and 3 only)
int conv_tc_launch(const ConvTcLaunch& L, cudaStream_t st) {
  if (L.impl == 1) {
    const int64_t total = (int64_t)L.p.NB * L.p.H * L.p.W * L.p.Cout;
    const int blocks = (int)std::min<int64_t>(ceil_div(total, 256), (int64_t)device_sm_count() * 16);
    ConvTcParams p = L.p;
    p.splits = 1;
    CGD_CUDA(launch_pdl(conv_simt_kernel, dim3(blocks), dim3(256), 0, st, L.A, L.Wp, p, L.a_sn, L.a_sh, L.a_sw, L.ldb));
    return 0;
  }
  if (L.narrow) return conv_narrow_launch(L, st);
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
  return (L.impl != 1 && !L.narrow && L.p.splits > 1 && !L.p.cluster) ? 2 : 1;
}

}  // namespace cgd

#ifdef CGD_CONV_PHASES
// The instrumented build only: copies the [kPhaseCtas][kPhaseTiles][kPhaseFields] stamps to `host` (n elements), then zeroes them.
extern "C" int cgd_conv_phases(unsigned long long* host, int n) {
  if (n != cgd::kPhaseCtas * cgd::kPhaseTiles * cgd::kPhaseFields) return -1;
  if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(host, cgd::g_conv_phases, sizeof(cgd::g_conv_phases)) != cudaSuccess)
    return -1;
  static unsigned long long zeros[cgd::kPhaseCtas * cgd::kPhaseTiles * cgd::kPhaseFields];
  return cudaMemcpyToSymbol(cgd::g_conv_phases, zeros, sizeof(zeros)) == cudaSuccess ? 0 : -1;
}
#endif
