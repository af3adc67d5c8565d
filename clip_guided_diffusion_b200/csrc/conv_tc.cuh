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
  int kblocks, splits, kb_per_split; // K loop = taps * Cin/64 blocks, optionally split over gridDim.z
  int out_f32;
  int b_batched;                     // B operand indexed by the tile's (h, n) (batched GEMM: attention)
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
                                     // c_proj writes d(c_fc output) directly, `res` = the saved pre-activation)
  float* epi_stats;                  // flags 2: per (128-pixel tile, 8-channel octet) sum / sum of squares of the fp16 OUTPUT, [m_tiles][Npad/8][2]
};

struct ConvTcLaunch {
  CUtensorMap tmA, tmB;              // A: 4-D pixel box; B: 4-D (K, rows, h, n) map, [BN x 64] weight slice per load
  CUtensorMap tmS;                   // 8 x 8 images (conv_small_kernel): the whole image + zero border as one [64 ch x 10 x 10 x 1] box (3x3) / [64 x 8 x 8 x 1] (1x1)
  ConvTcParams p;
  int BN, impl, m_tiles, n_tiles;
  int small;                         // 8 x 8 images: the weight-streaming mma.sync kernel of conv_narrow.cu (8 output channels per CTA, no split-K)
  int narrow;                        // <= 8 output channels, fp32 out, 3x3: the halo-tile mma.sync kernel of conv_narrow.cu instead of a wgmma tile
  const __half* A;
  const __half* Wp;
  int64_t a_sn, a_sh, a_sw;
  int64_t ldb, b_sh, b_sn;
};

int conv_tc_prepare(const CgdOp& op, ConvTcLaunch& L);
int conv_tc_launch(const ConvTcLaunch& L, cudaStream_t st);
int conv_tc_num_launches(const ConvTcLaunch& L);
bool conv_narrow_eligible(const ConvTcLaunch& L);              // conv_narrow.cu
int conv_narrow_launch(const ConvTcLaunch& L, cudaStream_t st);
bool conv_small_eligible(const ConvTcLaunch& L);
int conv_small_launch(const ConvTcLaunch& L, cudaStream_t st);
int conv_cluster_capacity(int BN, int S);

}  // namespace cgd
