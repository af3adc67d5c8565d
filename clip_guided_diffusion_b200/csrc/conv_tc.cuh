// conv_tc.cuh -- parameter blocks of the wgmma implicit-GEMM conv (see conv_tc.cu).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "../../include/cgd_b200.h"

namespace cgd {

struct ConvTcParams {
  int NB, H, W, Cin, Cout, Npad, taps;
  int TW, TH, TN;                    // 128-pixel tile = TW x TH x TN box of the (W, H, N) grid
  int tiles_w, tiles_h, tiles_n;
  int m_tiles, tiles;                // pixel tiles (tiles_w * tiles_h * tiles_n); output tiles (m_tiles * Npad / BN)
  int kblocks, splits, kb_per_split; // K loop = taps * Cin/64 blocks, optionally split over gridDim.z
  int out_f32;
  int ws_rows;                       // rows per split in the split-K workspace (= m_tiles * 128)
  int cluster;                       // split-K inside a cluster of `splits` CTAs along z, reduced through distributed shared memory
  const void* pf_ptr;                // next conv's packed weights: prefetched into L2 by the idle lanes of the TMA warp (0 = none)
  int64_t pf_bytes;
  int64_t out_sn, out_sh, out_sw;    // output / residual strides in elements (channel contiguous)
  int64_t res_sn, res_sh, res_sw;
  int64_t out_sc;                    // output channel stride (1 except for NCHW fp32 outputs; scalar-store paths only)
  const float* bias;
  const __half* res;
  void* out;
  float* ws;                         // split-K partials [splits][m_tiles*128][Npad]
  int res_mode;                      // 0 = out = acc (+bias) + res ; 1 = out = acc * QuickGELU'(res) (CONV flags 4: the dgrad of the ViT's
                                     // c_proj writes d(c_fc output) directly, `res` = the saved pre-activation) ; 2 = out = acc * GELU'(res)
                                     // (CONV flags 8: the same for the exact-GELU MLPs of the OpenCLIP towers)
};

struct ConvTcLaunch {
  CUtensorMap tmA, tmB;              // A: 4-D pixel box; B: [Npad, K] weights (4-D map, unit outer dims), [BN x 64] weight slice per load
  CUtensorMap tmOut, tmRes;          // persistent kernel: output / residual (C = Cout, W, H, N), one 128-pixel x 64-channel box per load / store
  ConvTcParams p;
  int BN, impl, m_tiles, n_tiles;
  int narrow;                        // <= 8 output channels, fp32 out, 3x3: the halo-tile mma.sync kernel of conv_narrow.cu instead of a wgmma tile
  int persistent;                    // no split-K, fp16 channel-contiguous out, Cout % 8 == 0: conv_tc_persistent_kernel (min(tiles, SMs) CTAs)
  const __half* A;
  const __half* Wp;
  int64_t a_sn, a_sh, a_sw;
  int64_t ldb;
};

int conv_tc_prepare(const CgdOp& op, ConvTcLaunch& L);
int conv_tc_launch(const ConvTcLaunch& L, cudaStream_t st);
int conv_tc_num_launches(const ConvTcLaunch& L);
bool conv_narrow_eligible(const ConvTcLaunch& L);              // conv_narrow.cu
int conv_narrow_launch(const ConvTcLaunch& L, cudaStream_t st);
int conv_cluster_capacity(int BN, int S);

}  // namespace cgd
