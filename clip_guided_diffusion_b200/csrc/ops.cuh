// ops.cuh -- launcher prototypes, one per CGD_OP_* code (slot tables in include/cgd_b200.h).
#pragma once
#include <cuda_runtime.h>

#include "../../include/cgd_b200.h"

namespace cgd {
int launch_gn_stats(const CgdOp& op, cudaStream_t st);
int launch_gn_apply(const CgdOp& op, cudaStream_t st);
int launch_gn_bwd_stats(const CgdOp& op, cudaStream_t st);
int launch_gn_bwd_apply(const CgdOp& op, cudaStream_t st);
int launch_gn_fwd_fused(const CgdOp& op, cudaStream_t st);
int launch_gn_bwd_fused(const CgdOp& op, cudaStream_t st);
int launch_gn_fwd_grid(const CgdOp& op, cudaStream_t st);
int launch_gn_bwd_grid(const CgdOp& op, cudaStream_t st);
int launch_relu_fwd(const CgdOp& op, cudaStream_t st);
int launch_relu_bwd(const CgdOp& op, cudaStream_t st);
int launch_maxpool2_fwd(const CgdOp& op, cudaStream_t st);
int launch_maxpool2_bwd(const CgdOp& op, cudaStream_t st);
int launch_lpips_tap(const CgdOp& op, cudaStream_t st);
int launch_fill(const CgdOp& op, cudaStream_t st);
int launch_ln_fwd(const CgdOp& op, cudaStream_t st);
int launch_ln_bwd(const CgdOp& op, cudaStream_t st);
int launch_pool2(const CgdOp& op, cudaStream_t st);
int launch_up2(const CgdOp& op, cudaStream_t st);
int launch_add(const CgdOp& op, cudaStream_t st);
int launch_copy(const CgdOp& op, cudaStream_t st);
int launch_attn_fwd(const CgdOp& op, cudaStream_t st);
int launch_attn_bwd(const CgdOp& op, cudaStream_t st);
int attn_bwd_num_launches(const CgdOp& op);
int launch_linear_small(const CgdOp& op, cudaStream_t st);
int launch_timestep_emb(const CgdOp& op, cudaStream_t st);
int launch_label_add(const CgdOp& op, cudaStream_t st);
int launch_nchw_to_pm(const CgdOp& op, cudaStream_t st);
int launch_pm_to_nchw(const CgdOp& op, cudaStream_t st);
int launch_qgelu_fwd(const CgdOp& op, cudaStream_t st);
int launch_qgelu_bwd(const CgdOp& op, cudaStream_t st);
int launch_vit_embed(const CgdOp& op, cudaStream_t st);
int launch_cutouts_fwd(const CgdOp& op, cudaStream_t st);
int launch_cutouts_bwd(const CgdOp& op, cudaStream_t st);
int launch_cutouts_rr_fwd(const CgdOp& op, cudaStream_t st);
int launch_cutouts_rr_bwd(const CgdOp& op, cudaStream_t st);
int launch_cutouts_aug_fwd(const CgdOp& op, cudaStream_t st);
int launch_cutouts_aug_bwd(const CgdOp& op, cudaStream_t st);
int launch_resize_axis(const CgdOp& op, cudaStream_t st);
int launch_token_embed(const CgdOp& op, cudaStream_t st);
int launch_row_gather(const CgdOp& op, cudaStream_t st);
int launch_seed_quant(const CgdOp& op, cudaStream_t st);
int launch_mag_clamp(const CgdOp& op, cudaStream_t st);
int launch_attnpool_embed_fwd(const CgdOp& op, cudaStream_t st);
int launch_attnpool_embed_bwd(const CgdOp& op, cudaStream_t st);
int launch_spherical(const CgdOp& op, cudaStream_t st);
int launch_pmv_blend(const CgdOp& op, cudaStream_t st);
int launch_guide_grad(const CgdOp& op, cudaStream_t st);
int launch_final_grad(const CgdOp& op, cudaStream_t st);
int launch_sample_ancestral(const CgdOp& op, cudaStream_t st);
int launch_sample_ddim(const CgdOp& op, cudaStream_t st);
int launch_grad_seed(const CgdOp& op, cudaStream_t st);
int launch_grad_unscale(const CgdOp& op, cudaStream_t st);
int launch_pmv_bwd(const CgdOp& op, cudaStream_t st);
int launch_clip_patchify(const CgdOp& op, cudaStream_t st);
int launch_clip_seed(const CgdOp& op, cudaStream_t st);
int launch_clip_unpatchify(const CgdOp& op, cudaStream_t st);
int launch_lpips_pair_fwd(const CgdOp& op, cudaStream_t st);
int launch_lpips_loss(const CgdOp& op, cudaStream_t st);
int launch_lpips_seed(const CgdOp& op, cudaStream_t st);
int launch_lpips_pair_bwd(const CgdOp& op, cudaStream_t st);
int launch_img_loss_fwd(const CgdOp& op, cudaStream_t st);
int launch_img_loss_bwd(const CgdOp& op, cudaStream_t st);
int launch_sph_dist_fwd(const CgdOp& op, cudaStream_t st);
int launch_sph_dist_bwd(const CgdOp& op, cudaStream_t st);
}  // namespace cgd
