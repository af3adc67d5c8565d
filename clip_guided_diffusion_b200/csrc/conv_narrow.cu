// conv_narrow.cu -- 3x3 convolution with at most 8 output channels and an fp32 (NCHW) output: the UNet head (256 -> 6, [3P] `out[2]`)
// and the stem's input gradient (256 -> 3, the last op of the backward that cgd/cgd.py:228 triggers).
//
// Why a separate kernel: on the wgmma tile kernel the N = 16 tile of these two layers uses 1/16 of the tensor width while the A operand
// (33.5 MB at 256x256) is still streamed nine times, once per tap, from L2 (302 MB per launch).  Here a CTA owns a 4 x 32 pixel tile: per 64-channel slice its (4+2) x (32+2) halo is loaded ONCE into shared
// memory (cp.async, zero-filled outside the image = the conv padding), the nine taps are shifted ldmatrix reads of that tile, and the
// product runs on mma.sync.m16n8k16 whose N = 8 is exactly this layer's width.  A traffic: 1.6x the tensor (halo), 53 MB instead of
// 302 MB.  fp16 operands, fp32 accumulate, like the other conv paths.
#include <algorithm>

#include "attn_mma.cuh"
#include "common.cuh"
#include "conv_tc.cuh"
#include "pdl.cuh"
#include "tc_ptx.cuh"

namespace cgd {

constexpr int NR_TH = 4, NR_TW = 32;                   // output tile: 4 rows x 32 pixels = one row per warp
constexpr int NR_HW = NR_TW + 2, NR_HH = NR_TH + 2;    // halo tile
constexpr int NR_PIX = NR_HW * NR_HH;                  // 204 pixels per slice
constexpr int NR_STAGE = NR_PIX * 128;                 // 64 channels x 2 B per pixel
constexpr int NR_STAGES = 2;
constexpr int NR_THREADS = 128;

__device__ __forceinline__ void nr_cp16(uint32_t dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;  // src-size 0: the 16 bytes are zero-filled (conv padding / image border)
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}

__global__ void __launch_bounds__(NR_THREADS)
conv_narrow_kernel(const __half* __restrict__ A, const __half* __restrict__ Wp, const float* __restrict__ bias, float* __restrict__ out, int NB,
                   int H, int W, int Cin, int Cout, int64_t a_sn, int64_t a_sh, int64_t a_sw, int64_t ldb, int64_t o_sn, int64_t o_sh,
                   int64_t o_sw, int64_t o_sc, int tiles_x, int tiles_y) {
  extern __shared__ __align__(128) uint8_t nr_smem[];
  const int K = 9 * Cin, wld = K + 8;  // weight rows padded by 16 B: the 8 rows land on different banks
  uint8_t* stage_base = nr_smem;
  __half* ws = reinterpret_cast<__half*>(nr_smem + NR_STAGES * NR_STAGE);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tx = blockIdx.x % tiles_x, ty = (blockIdx.x / tiles_x) % tiles_y, n = blockIdx.x / (tiles_x * tiles_y);
  const int x0 = tx * NR_TW, y0 = ty * NR_TH;
  // weights do not depend on the previous kernel: stage them before the grid dependency resolves
  for (int v = tid; v < 8 * (K / 8); v += NR_THREADS) {
    const int r = v / (K / 8), c = (v - r * (K / 8)) * 8;
    *reinterpret_cast<half8*>(ws + r * wld + c) = ld8(Wp + (int64_t)r * ldb + c);
  }
  pdl_wait();
  pdl_launch_dependents();
  const __half* An = A + (int64_t)n * a_sn;
  const int nslices = Cin / 64;
  auto load_slice = [&](int s, int st) {
    const uint32_t base = as_smem(stage_base + st * NR_STAGE);
    for (int v = tid; v < NR_PIX * 8; v += NR_THREADS) {
      const int pix = v >> 3, ch = v & 7;
      const int hy = pix / NR_HW, hx = pix - hy * NR_HW;
      const int y = y0 - 1 + hy, x = x0 - 1 + hx;
      const bool ok = y >= 0 && y < H && x >= 0 && x < W;
      const __half* src = ok ? An + (int64_t)y * a_sh + (int64_t)x * a_sw + s * 64 + ch * 8 : A;
      nr_cp16(base + pix * 128 + ((ch ^ (pix & 7)) << 4), src, ok);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  load_slice(0, 0);
  if (nslices > 1) load_slice(1, 1);
  float acc[2][4];
#pragma unroll
  for (int t = 0; t < 2; ++t)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[t][e] = 0.f;
  const int mi = lane >> 3;
  const int wrow = lane >> 2, wcol = (lane & 3) * 2;
  for (int s = 0; s < nslices; ++s) {
    if (s + 1 < nslices) asm volatile("cp.async.wait_group 1;" ::: "memory");
    else asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    const uint32_t base = as_smem(stage_base + (s & 1) * NR_STAGE);
#pragma unroll 1
    for (int tap = 0; tap < 9; ++tap) {
      const int dy = tap / 3 - 1, dx = tap - (tap / 3) * 3 - 1;
      const int prow = (warp + 1 + dy) * NR_HW + 1 + dx;  // halo index of this warp's pixel x = 0 under this tap
      const __half* wk = ws + wrow * wld + tap * Cin + s * 64 + wcol;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(wk + ks * 16);
        const uint32_t b1 = *reinterpret_cast<const uint32_t*>(wk + ks * 16 + 8);
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          const int pix = prow + t * 16 + (lane & 7) + (mi & 1) * 8;
          const int ch = ks * 2 + (mi >> 1);
          uint32_t a[4];
          ldsm_x4(base + pix * 128 + ((ch ^ (pix & 7)) << 4), a);
          mma16816(acc[t], a, b0, b1);
        }
      }
    }
    __syncthreads();  // every warp is done with this stage before it is refilled
    if (s + 2 < nslices) load_slice(s + 2, s & 1);
  }
  const int y = y0 + warp;
  if (y < H) {
#pragma unroll
    for (int t = 0; t < 2; ++t)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int x = x0 + t * 16 + wrow + (e >> 1) * 8, c = wcol + (e & 1);
        if (x < W && c < Cout) out[(int64_t)n * o_sn + (int64_t)y * o_sh + (int64_t)x * o_sw + (int64_t)c * o_sc] = acc[t][e] + (bias ? bias[c] : 0.f);
      }
  }
}

bool conv_narrow_eligible(const ConvTcLaunch& L) {
  const ConvTcParams& p = L.p;
  return p.taps == 9 && p.Cout <= 8 && p.Cin % 64 == 0 && p.Cin <= 1024 && p.out_f32 && p.res == nullptr && p.splits == 1 && !p.b_batched &&
         L.impl == 0 && L.ldb % 8 == 0;
}

int conv_narrow_launch(const ConvTcLaunch& L, cudaStream_t st) {
  const ConvTcParams& p = L.p;
  const int smem = NR_STAGES * NR_STAGE + 8 * (9 * p.Cin + 8) * 2;
  static DeviceOnce attr_set;
  if (attr_set.needed()) {
    CGD_CUDA(cudaFuncSetAttribute(conv_narrow_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, NR_STAGES * NR_STAGE + 8 * (9 * 1024 + 8) * 2));
    attr_set.mark();
  }
  const int tiles_x = (int)ceil_div(p.W, NR_TW), tiles_y = (int)ceil_div(p.H, NR_TH);
  CGD_CUDA(launch_pdl(conv_narrow_kernel, dim3((unsigned)(tiles_x * tiles_y * p.NB)), dim3(NR_THREADS), (size_t)smem, st, L.A, L.Wp, p.bias, (float*)p.out,
                      p.NB, p.H, p.W, p.Cin, p.Cout, L.a_sn, L.a_sh, L.a_sw, L.ldb, p.out_sn, p.out_sh, p.out_sw, p.out_sc, tiles_x, tiles_y));
  return 0;
}


// ================================================================================================ 8 x 8 images: weight-streaming kernel
// conv_small_kernel -- 3x3 / 1x1 convolution of an 8 x 8 image (M = 64 pixels): the UNet's deepest level and its attention 1x1s.
//
// Why: on the wgmma tiles these layers are 64 pixels in a 128-row tile, split many ways along K with an fp32 workspace and a reduce
// launch (or a cluster), so their time is launch and reduction latency rather than the weight stream (18.9 MB for the 1024 -> 1024 3x3).  Here the problem is turned around: a CTA
// owns EIGHT OUTPUT CHANNELS of one image and the whole K extent -- no split-K, no reduction, one launch.  Its 8 x K weight slab
// (at most 8 x 9216 halfs) is fetched with cp.async BEFORE the grid dependency resolves (weights are step-invariant: under programmatic dependent
// launch the HBM stream overlaps the previous kernel's tail), the activations stream through a 4-stage ring of 64-channel slices (halo
// tile for 3x3), and the product runs on mma.sync.m16n8k16 whose N = 8 is exactly the CTA's channel slab: 8 warps = 4 pixel tiles x 2
// halves of every slice's K, two independent accumulator chains per warp, one shared-memory add at the end.
constexpr int SM_THREADS = 256, SM_STAGES = 4;

// Data movement: per 64-channel slice ONE TMA tensor load of the box [64 ch x 10 x 10 x 1] anchored at (-1, -1) -- the 8 x 8 image with
// its zero border, out-of-image coordinates zero-filled by the TMA unit, 128-byte swizzle (slot = pixel, 16-byte chunk ^= slot & 7) --
// and eight cp.async.bulk copies for the weight slab (one row of K halfs per output channel): a few large requests rather than one
// cp.async per 16-byte piece or one small bulk copy per pixel, which would make the kernel request-bound.
template <int TAPS>
__global__ void __launch_bounds__(SM_THREADS)
conv_small_kernel(const __grid_constant__ CUtensorMap tmA, const __half* __restrict__ Wp, const float* __restrict__ bias,
                  const __half* __restrict__ res, __half* __restrict__ out, int Cin, int64_t ldb, int64_t o_sn, int64_t o_sh, int64_t o_sw, int64_t r_sn,
                  int64_t r_sh, int64_t r_sw) {
  constexpr int HALO = TAPS == 9 ? 10 : 8;           // stage tile edge in pixel slots (3x3: a zero border around the 8 x 8 image)
  constexpr int PIXS = HALO * HALO;
  constexpr int STAGE = ((PIXS * 128 + 1023) / 1024) * 1024;  // 1024-byte aligned stages: the swizzle pattern is address-based
  extern __shared__ uint8_t sm_smem_raw[];
  uint8_t* sm_smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(sm_smem_raw) + 1023) & ~uintptr_t(1023));
  const int K = TAPS * Cin, wld = K + 8;
  uint8_t* stage_base = sm_smem;
  __half* ws = reinterpret_cast<__half*>(sm_smem + SM_STAGES * STAGE);
  __shared__ float red[4][32][4];
  __shared__ __align__(8) uint64_t wbar, full_bar[SM_STAGES];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n0 = blockIdx.x * 8, img = blockIdx.y;
  if (tid == 0) {
    tma_prefetch_desc(&tmA);
    mbar_init(&wbar, 1);
    for (int s = 0; s < SM_STAGES; ++s) mbar_init(&full_bar[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // weight slab of this CTA's 8 output channels: independent of the previous kernel -> issued before the grid dependency resolves
  if (warp == 0) {
    if (lane == 0) mbar_expect_tx(&wbar, (uint32_t)(8 * K * 2));
    __syncwarp();
    if (lane < 8) bulk_load_1d(ws + lane * wld, Wp + (int64_t)(n0 + lane) * ldb, (uint32_t)(K * 2), &wbar);
  }
  pdl_wait();
  pdl_launch_dependents();
  const int nslices = Cin / 64;
  auto load_slice = [&](int s) {  // one thread: the whole (bordered) image slice as one tensor box
    const int st = s % SM_STAGES;
    mbar_expect_tx(&full_bar[st], PIXS * 128);
    tma_load_4d(stage_base + st * STAGE, &tmA, &full_bar[st], s * 64, TAPS == 9 ? -1 : 0, TAPS == 9 ? -1 : 0, img);
  };
  if (tid == 0)
    for (int s = 0; s < SM_STAGES && s < nslices; ++s) load_slice(s);
  float acc[2][4];
#pragma unroll
  for (int t = 0; t < 2; ++t)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[t][e] = 0.f;
  const int mt = warp & 3, kh = warp >> 2;  // pixel tile (image rows 2 mt, 2 mt + 1), half of each slice's k16 steps
  const int mi = lane >> 3;
  const int wrow = lane >> 2, wcol = (lane & 3) * 2;
  const int p = (lane & 7) + (mi & 1) * 8;        // pixel of this lane's ldmatrix row inside the 16-pixel tile
  const int py = 2 * mt + (p >> 3), px = p & 7;   // its image coordinates
  mbar_wait(&wbar, 0);
  for (int s = 0; s < nslices; ++s) {
    const int st = s % SM_STAGES;
    mbar_wait(&full_bar[st], (uint32_t)((s / SM_STAGES) & 1));
    const uint32_t base = as_smem(stage_base + st * STAGE);
#pragma unroll
    for (int tap = 0; tap < TAPS; ++tap) {
      const int dy = TAPS == 9 ? tap / 3 - 1 : 0, dx = TAPS == 9 ? tap % 3 - 1 : 0;
      const int pix = TAPS == 9 ? (py + 1 + dy) * HALO + px + 1 + dx : py * HALO + px;
      const __half* wk = ws + wrow * wld + tap * Cin + s * 64 + wcol;
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int ks = kh * 2 + j;
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(wk + ks * 16);
        const uint32_t b1 = *reinterpret_cast<const uint32_t*>(wk + ks * 16 + 8);
        const int ch = ks * 2 + (mi >> 1);
        uint32_t a[4];
        ldsm_x4(base + pix * 128 + ((ch ^ (pix & 7)) << 4), a);
        mma16816(acc[j], a, b0, b1);
      }
    }
    __syncthreads();  // every warp is done with this stage before it is refilled
    if (tid == 0 && s + SM_STAGES < nslices) load_slice(s + SM_STAGES);
  }
  float c[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) c[e] = acc[0][e] + acc[1][e];
  if (kh == 1) {
#pragma unroll
    for (int e = 0; e < 4; ++e) red[mt][lane][e] = c[e];
  }
  __syncthreads();
  if (kh == 0) {
#pragma unroll
    for (int e = 0; e < 4; ++e) c[e] += red[mt][lane][e];
    const int ch = n0 + wcol;
    const float b0 = bias ? bias[ch] : 0.f, b1 = bias ? bias[ch + 1] : 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {  // accumulator rows lane / 4 and lane / 4 + 8 of the 16-pixel tile
      const int q = wrow + h * 8, y = 2 * mt + (q >> 3), x = q & 7;
      float v0 = c[2 * h] + b0, v1 = c[2 * h + 1] + b1;
      if (res) {
        const float2 r = __half22float2(*reinterpret_cast<const __half2*>(res + (int64_t)img * r_sn + (int64_t)y * r_sh + (int64_t)x * r_sw + ch));
        v0 += r.x;
        v1 += r.y;
      }
      *reinterpret_cast<__half2*>(out + (int64_t)img * o_sn + (int64_t)y * o_sh + (int64_t)x * o_sw + ch) = __floats2half2_rn(v0, v1);
    }
  }
}

static inline int conv_small_smem(int taps, int Cin) {  // 1024-byte aligned stages (+ alignment slack) + the weight slab
  return 1024 + SM_STAGES * (((taps == 9 ? 100 : 64) * 128 + 1023) / 1024) * 1024 + 8 * (taps * Cin + 8) * 2;
}

bool conv_small_eligible(const ConvTcLaunch& L) {
  const ConvTcParams& p = L.p;
  return (p.taps == 9 || p.taps == 1) && p.H == 8 && p.W == 8 && p.Cin % 64 == 0 && p.Cout % 8 == 0 && !p.out_f32 && p.out_sc == 1 && !p.b_batched &&
         p.res_mode == 0 && p.epi_stats == nullptr && L.impl == 0 && L.ldb % 8 == 0 && p.out_sw % 2 == 0 &&
         (p.res == nullptr || p.res_sw % 2 == 0) && L.a_sn % 8 == 0 && L.a_sh % 8 == 0 && L.a_sw % 8 == 0 &&
         (reinterpret_cast<uintptr_t>(L.A) % 16) == 0 && (reinterpret_cast<uintptr_t>(L.Wp) % 16) == 0 && conv_small_smem(p.taps, p.Cin) <= 212 * 1024;
}

int conv_small_launch(const ConvTcLaunch& L, cudaStream_t st) {
  const ConvTcParams& p = L.p;
  const int smem = conv_small_smem(p.taps, p.Cin);
  static DeviceOnce attr_set;
  if (attr_set.needed()) {
    CGD_CUDA(cudaFuncSetAttribute(conv_small_kernel<9>, cudaFuncAttributeMaxDynamicSharedMemorySize, 212 * 1024));
    CGD_CUDA(cudaFuncSetAttribute(conv_small_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 212 * 1024));
    attr_set.mark();
  }
  const dim3 grid((unsigned)(p.Cout / 8), (unsigned)p.NB);
  if (p.taps == 9)
    CGD_CUDA(launch_pdl(conv_small_kernel<9>, grid, dim3(SM_THREADS), (size_t)smem, st, L.tmS, L.Wp, p.bias, p.res, (__half*)p.out, p.Cin, L.ldb, p.out_sn,
                        p.out_sh, p.out_sw, p.res_sn, p.res_sh, p.res_sw));
  else
    CGD_CUDA(launch_pdl(conv_small_kernel<1>, grid, dim3(SM_THREADS), (size_t)smem, st, L.tmS, L.Wp, p.bias, p.res, (__half*)p.out, p.Cin, L.ldb, p.out_sn,
                        p.out_sh, p.out_sw, p.res_sn, p.res_sh, p.res_sw));
  return 0;
}

}  // namespace cgd
