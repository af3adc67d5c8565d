// api.cu -- the extern "C" surface of libcgd_b200.so (include/cgd_b200.h): plans (op lists with pre-encoded
// TMA descriptors), per-op dispatch, network / step aliases and stand-alone operator entry points.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <new>
#include <vector>

#include "common.cuh"
#include "conv_tc.cuh"
#include "ops.cuh"
#include "pdl.cuh"

namespace cgd {

bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("CGD_PDL");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v != 0;
}

static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

struct Plan {
  std::vector<CgdOp> ops;
  std::vector<int> conv_index;        // op -> index into convs (or -1)
  std::vector<ConvTcLaunch> convs;
  int n_fwd = 0;                      // for the network aliases
};

static int dispatch(const CgdOp& op, const ConvTcLaunch* conv, cudaStream_t st) {
  switch (op.code) {
    case CGD_OP_CONV: return conv_tc_launch(*conv, st);
    case CGD_OP_GN_STATS: return launch_gn_stats(op, st);
    case CGD_OP_GN_APPLY: return launch_gn_apply(op, st);
    case CGD_OP_GN_BWD_STATS: return launch_gn_bwd_stats(op, st);
    case CGD_OP_GN_BWD_APPLY: return launch_gn_bwd_apply(op, st);
    case CGD_OP_POOL2: return launch_pool2(op, st);
    case CGD_OP_UP2: return launch_up2(op, st);
    case CGD_OP_ADD: return launch_add(op, st);
    case CGD_OP_COPY: return launch_copy(op, st);
    case CGD_OP_ATTN_FWD: return launch_attn_fwd(op, st);
    case CGD_OP_ATTN_BWD: return launch_attn_bwd(op, st);
    case CGD_OP_GN_FWD_FUSED: return launch_gn_fwd_fused(op, st);
    case CGD_OP_GN_BWD_FUSED: return launch_gn_bwd_fused(op, st);
    case CGD_OP_GN_FWD_GRID: return launch_gn_fwd_grid(op, st);
    case CGD_OP_GN_BWD_GRID: return launch_gn_bwd_grid(op, st);
    case CGD_OP_RELU_FWD: return launch_relu_fwd(op, st);
    case CGD_OP_RELU_BWD: return launch_relu_bwd(op, st);
    case CGD_OP_MAXPOOL2_FWD: return launch_maxpool2_fwd(op, st);
    case CGD_OP_MAXPOOL2_BWD: return launch_maxpool2_bwd(op, st);
    case CGD_OP_LPIPS_TAP: return launch_lpips_tap(op, st);
    case CGD_OP_FILL: return launch_fill(op, st);
    case CGD_OP_CUTOUTS_RR_FWD: return launch_cutouts_rr_fwd(op, st);
    case CGD_OP_CUTOUTS_RR_BWD: return launch_cutouts_rr_bwd(op, st);
    case CGD_OP_CUTOUTS_AUG_FWD: return launch_cutouts_aug_fwd(op, st);
    case CGD_OP_CUTOUTS_AUG_BWD: return launch_cutouts_aug_bwd(op, st);
    case CGD_OP_RESIZE_AXIS: return launch_resize_axis(op, st);
    case CGD_OP_TOKEN_EMBED: return launch_token_embed(op, st);
    case CGD_OP_ROW_GATHER: return launch_row_gather(op, st);
    case CGD_OP_SEED_QUANT: return launch_seed_quant(op, st);
    case CGD_OP_MAG_CLAMP: return launch_mag_clamp(op, st);
    case CGD_OP_ATTNPOOL_EMBED_FWD: return launch_attnpool_embed_fwd(op, st);
    case CGD_OP_ATTNPOOL_EMBED_BWD: return launch_attnpool_embed_bwd(op, st);
    case CGD_OP_LINEAR_SMALL: return launch_linear_small(op, st);
    case CGD_OP_TIMESTEP_EMB: return launch_timestep_emb(op, st);
    case CGD_OP_LABEL_ADD: return launch_label_add(op, st);
    case CGD_OP_NCHW_TO_PM: return launch_nchw_to_pm(op, st);
    case CGD_OP_PM_TO_NCHW: return launch_pm_to_nchw(op, st);
    case CGD_OP_LN_FWD: return launch_ln_fwd(op, st);
    case CGD_OP_LN_BWD: return launch_ln_bwd(op, st);
    case CGD_OP_QGELU_FWD: return launch_qgelu_fwd(op, st);
    case CGD_OP_QGELU_BWD: return launch_qgelu_bwd(op, st);
    case CGD_OP_VIT_EMBED: return launch_vit_embed(op, st);
    case CGD_OP_CUTOUTS_FWD: return launch_cutouts_fwd(op, st);
    case CGD_OP_CUTOUTS_BWD: return launch_cutouts_bwd(op, st);
    case CGD_OP_SPHERICAL: return launch_spherical(op, st);
    case CGD_OP_PMV_BLEND: return launch_pmv_blend(op, st);
    case CGD_OP_GUIDE_GRAD: return launch_guide_grad(op, st);
    case CGD_OP_FINAL_GRAD: return launch_final_grad(op, st);
    case CGD_OP_SAMPLE_ANCESTRAL: return launch_sample_ancestral(op, st);
    case CGD_OP_SAMPLE_DDIM: return launch_sample_ddim(op, st);
    case CGD_OP_GRAD_SEED: return launch_grad_seed(op, st);
    case CGD_OP_GRAD_UNSCALE: return launch_grad_unscale(op, st);
    case CGD_OP_PMV_BWD: return launch_pmv_bwd(op, st);
    case CGD_OP_CLIP_PATCHIFY: return launch_clip_patchify(op, st);
    case CGD_OP_CLIP_SEED: return launch_clip_seed(op, st);
    case CGD_OP_CLIP_UNPATCHIFY: return launch_clip_unpatchify(op, st);
    case CGD_OP_LPIPS_PAIR_FWD: return launch_lpips_pair_fwd(op, st);
    case CGD_OP_LPIPS_LOSS: return launch_lpips_loss(op, st);
    case CGD_OP_LPIPS_SEED: return launch_lpips_seed(op, st);
    case CGD_OP_LPIPS_PAIR_BWD: return launch_lpips_pair_bwd(op, st);
    case CGD_OP_IMG_LOSS_FWD: return launch_img_loss_fwd(op, st);
    case CGD_OP_IMG_LOSS_BWD: return launch_img_loss_bwd(op, st);
    case CGD_OP_SPH_DIST_FWD: return launch_sph_dist_fwd(op, st);
    case CGD_OP_SPH_DIST_BWD: return launch_sph_dist_bwd(op, st);
    default: set_error("unknown op code %d", op.code); return -1;
  }
}

static int op_launches(const CgdOp& op, const ConvTcLaunch* conv) {
  switch (op.code) {
    case CGD_OP_CONV: return conv_tc_num_launches(*conv);
    case CGD_OP_ATTN_BWD: return attn_bwd_num_launches(op);
    case CGD_OP_FINAL_GRAD: return ((op.flags & 1) && !(op.flags & 4)) ? 2 : 1;
    case CGD_OP_GRAD_SEED: return 2;
    case CGD_OP_IMG_LOSS_FWD: return 2;
    default: return 1;
  }
}

// codes of removed ops (include/cgd_b200.h): rejected when the plan is built rather than when it runs
static bool op_retired(int32_t code) { return code == 30 || code == 31 || code == 32 || code == 49; }

static int plan_create(const CgdOp* ops, int32_t n_ops, Plan** out) {
  CGD_CHECK_ARG(ops != nullptr && n_ops > 0 && out != nullptr, "plan_create: bad arguments");
  Plan* pl = new (std::nothrow) Plan();
  CGD_CHECK_ARG(pl != nullptr, "plan_create: out of host memory");
  pl->ops.assign(ops, ops + n_ops);
  pl->conv_index.assign(n_ops, -1);
  for (int i = 0; i < n_ops; ++i) {
    if (ops[i].code <= 0 || ops[i].code >= CGD_OP__COUNT || op_retired(ops[i].code)) {
      set_error("plan_create: op %d has unknown code %d", i, ops[i].code);
      delete pl;
      return -1;
    }
    if (ops[i].code == CGD_OP_CONV) {
      ConvTcLaunch L;
      memset(&L, 0, sizeof(L));
      const int rc = conv_tc_prepare(ops[i], L);
      if (rc) {
        char tmp[900];
        snprintf(tmp, sizeof(tmp), "%s", g_err);
        set_error("plan_create: op %d: %s", i, tmp);
        delete pl;
        return rc;
      }
      pl->conv_index[i] = (int)pl->convs.size();
      pl->convs.push_back(L);
    }
  }
  // L2 prefetch chain: every conv prefetches the packed weights of the next conv of the list while its own epilogue warps
  // wait for the accumulator (the 8x8 .. 32x32 layers and the ViT GEMMs are bound by the HBM latency of their weight stream)
  if (!(getenv("CGD_CONV_PREFETCH") && getenv("CGD_CONV_PREFETCH")[0] == '0')) {
    for (size_t k = 0; k + 1 < pl->convs.size(); ++k) {
      const ConvTcLaunch& nx = pl->convs[k + 1];
      if (nx.impl == 1) continue;
      pl->convs[k].p.pf_ptr = nx.Wp;
      pl->convs[k].p.pf_bytes = (int64_t)nx.p.Npad * nx.ldb * 2;
    }
  }
  *out = pl;
  return 0;
}

static int plan_run(Plan* pl, int32_t first, int32_t count, cudaStream_t st) {
  CGD_CHECK_ARG(pl != nullptr, "plan_run: null plan");
  CGD_CHECK_ARG(first >= 0 && count >= 0 && (size_t)first + (size_t)count <= pl->ops.size(), "plan_run: range [%d,%d) outside plan of %zu ops",
                first, first + count, pl->ops.size());
  for (int i = first; i < first + count; ++i) {
    const ConvTcLaunch* conv = pl->conv_index[i] >= 0 ? &pl->convs[pl->conv_index[i]] : nullptr;
    const int rc = dispatch(pl->ops[i], conv, st);
    if (rc) {
      char tmp[900];
      snprintf(tmp, sizeof(tmp), "%s", g_err);
      set_error("op %d (code %d): %s", i, pl->ops[i].code, tmp);
      return rc;
    }
  }
  return 0;
}

}  // namespace cgd

using cgd::Plan;

extern "C" {

int cgd_abi_version(void) { return CGD_ABI_VERSION; }
const char* cgd_last_error(void) { return cgd::g_err; }
int cgd_conv_cluster_capacity(int32_t bn, int32_t splits) { return cgd::conv_cluster_capacity(bn, splits); }

int cgd_plan_create(const CgdOp* ops, int32_t n_ops, void** plan_out) {
  Plan* pl = nullptr;
  const int rc = cgd::plan_create(ops, n_ops, &pl);
  if (rc == 0) *plan_out = pl;
  return rc;
}
int cgd_plan_run(void* plan, int32_t first, int32_t count, void* stream) {
  return cgd::plan_run(static_cast<Plan*>(plan), first, count, static_cast<cudaStream_t>(stream));
}
int cgd_plan_num_launches(void* plan, int32_t first, int32_t count) {
  Plan* pl = static_cast<Plan*>(plan);
  if (!pl || first < 0 || count < 0 || (size_t)first + (size_t)count > pl->ops.size()) return -1;
  int n = 0;
  for (int i = first; i < first + count; ++i)
    n += cgd::op_launches(pl->ops[i], pl->conv_index[i] >= 0 ? &pl->convs[pl->conv_index[i]] : nullptr);
  return n;
}
int cgd_plan_destroy(void* plan) {
  delete static_cast<Plan*>(plan);
  return 0;
}
int cgd_run_op(const CgdOp* op, void* stream) {
  if (!op) { cgd::set_error("cgd_run_op: null op"); return -1; }
  if (op->code == CGD_OP_CONV) {
    cgd::ConvTcLaunch L;
    memset(&L, 0, sizeof(L));
    if (int rc = cgd::conv_tc_prepare(*op, L)) return rc;
    return cgd::dispatch(*op, &L, static_cast<cudaStream_t>(stream));
  }
  return cgd::dispatch(*op, nullptr, static_cast<cudaStream_t>(stream));
}

// ---- network aliases: forward segment [0, n_fwd), backward segment [n_fwd, n_fwd + n_bwd)
static int net_create(const CgdOp* ops, int32_t n_fwd, int32_t n_bwd, void** out) {
  if (n_fwd < 0 || n_bwd < 0) { cgd::set_error("create: negative segment length"); return -1; }
  Plan* pl = nullptr;
  const int rc = cgd::plan_create(ops, n_fwd + n_bwd, &pl);
  if (rc) return rc;
  pl->n_fwd = n_fwd;
  *out = pl;
  return 0;
}
static int net_fwd(void* h, void* stream) {
  Plan* pl = static_cast<Plan*>(h);
  if (!pl) { cgd::set_error("null handle"); return -1; }
  return cgd::plan_run(pl, 0, pl->n_fwd, static_cast<cudaStream_t>(stream));
}
static int net_bwd(void* h, void* stream) {
  Plan* pl = static_cast<Plan*>(h);
  if (!pl) { cgd::set_error("null handle"); return -1; }
  return cgd::plan_run(pl, pl->n_fwd, (int)pl->ops.size() - pl->n_fwd, static_cast<cudaStream_t>(stream));
}
int cgd_unet_create(const CgdOp* ops, int32_t n_fwd, int32_t n_bwd, void** handle_out) { return net_create(ops, n_fwd, n_bwd, handle_out); }
int cgd_unet_fwd(void* handle, void* stream) { return net_fwd(handle, stream); }
int cgd_unet_bwd_input(void* handle, void* stream) { return net_bwd(handle, stream); }
int cgd_unet_destroy(void* handle) { return cgd_plan_destroy(handle); }
int cgd_vit_create(const CgdOp* ops, int32_t n_fwd, int32_t n_bwd, void** handle_out) { return net_create(ops, n_fwd, n_bwd, handle_out); }
int cgd_vit_fwd(void* handle, void* stream) { return net_fwd(handle, stream); }
int cgd_vit_bwd_input(void* handle, void* stream) { return net_bwd(handle, stream); }
int cgd_vit_destroy(void* handle) { return cgd_plan_destroy(handle); }
int cgd_step_create(const CgdOp* ops, int32_t n_ops, void** handle_out) { return net_create(ops, n_ops, 0, handle_out); }
int cgd_step(void* handle, void* stream) { return net_fwd(handle, stream); }
int cgd_step_destroy(void* handle) { return cgd_plan_destroy(handle); }

// ---- stand-alone operators
int cgd_cutouts_fwd(const float* x_in, const int32_t* coords, void* patches_h, int64_t B, int64_t H, int64_t W, int64_t cutn,
                    int64_t cut_size, int64_t patch, int64_t kpad, const float* mean3, const float* std3, void* stream) {
  if (!mean3 || !std3) { cgd::set_error("cutouts_fwd: null mean/std"); return -1; }
  CgdOp op;
  memset(&op, 0, sizeof(op));
  op.code = CGD_OP_CUTOUTS_FWD;
  op.p[0] = (void*)x_in; op.p[1] = (void*)coords; op.p[2] = patches_h;
  op.i[0] = B; op.i[1] = H; op.i[2] = W; op.i[3] = cutn; op.i[4] = cut_size; op.i[5] = patch; op.i[6] = kpad;
  for (int k = 0; k < 3; ++k) { op.f[k] = mean3[k]; op.f[3 + k] = std3[k]; }
  return cgd_run_op(&op, stream);
}
int cgd_cutouts_bwd(const void* dpatches_h, const int32_t* coords, float* dx_in, int64_t B, int64_t H, int64_t W, int64_t cutn,
                    int64_t cut_size, int64_t patch, int64_t kpad, const float* std3, float scale, void* stream) {
  if (!std3) { cgd::set_error("cutouts_bwd: null std"); return -1; }
  CgdOp op;
  memset(&op, 0, sizeof(op));
  op.code = CGD_OP_CUTOUTS_BWD;
  op.p[0] = (void*)dpatches_h; op.p[1] = (void*)coords; op.p[2] = dx_in;
  op.i[0] = B; op.i[1] = H; op.i[2] = W; op.i[3] = cutn; op.i[4] = cut_size; op.i[5] = patch; op.i[6] = kpad;
  for (int k = 0; k < 3; ++k) op.f[3 + k] = std3[k];
  op.f[6] = scale;
  return cgd_run_op(&op, stream);
}
int cgd_spherical_fwd_bwd(const float* emb, const float* targets, const float* weights, float* d_emb, float* loss, int64_t cutn, int64_t B,
                          int64_t P, int64_t D, float clip_guidance_scale, float grad_scale, void* stream) {
  CgdOp op;
  memset(&op, 0, sizeof(op));
  op.code = CGD_OP_SPHERICAL;
  op.p[0] = (void*)emb; op.p[1] = (void*)targets; op.p[2] = (void*)weights; op.p[3] = d_emb; op.p[4] = loss;
  op.i[0] = cutn; op.i[1] = B; op.i[2] = P; op.i[3] = D;
  op.f[0] = clip_guidance_scale; op.f[1] = grad_scale;
  return cgd_run_op(&op, stream);
}
int cgd_guidance_losses_fwd_bwd(const float* x_in, const float* pred_xstart, const float* g_clip, const float* sc, void* seed_h,
                                float* dx_direct, float* loss, int64_t B, int64_t H, int64_t W, int64_t ld, float tv_scale,
                                float range_scale, float sat_scale, float seed_scale, void* stream) {
  CgdOp op;
  memset(&op, 0, sizeof(op));
  op.code = CGD_OP_GUIDE_GRAD;
  op.p[0] = (void*)x_in; op.p[1] = (void*)pred_xstart; op.p[2] = (void*)g_clip; op.p[3] = (void*)sc; op.p[4] = seed_h; op.p[5] = dx_direct;
  op.p[6] = loss;
  op.i[0] = B; op.i[1] = H; op.i[2] = W; op.i[3] = ld;
  op.f[0] = tv_scale; op.f[1] = range_scale; op.f[2] = sat_scale; op.f[3] = seed_scale;
  return cgd_run_op(&op, stream);
}
int cgd_sample_update_ancestral(const float* mean, const float* variance, const float* log_variance, const float* g, const float* noise,
                                const float* sc, float* sample, int64_t n, void* stream) {
  CgdOp op;
  memset(&op, 0, sizeof(op));
  op.code = CGD_OP_SAMPLE_ANCESTRAL;
  op.p[0] = (void*)mean; op.p[1] = (void*)variance; op.p[2] = (void*)log_variance; op.p[3] = (void*)g; op.p[4] = (void*)noise;
  op.p[5] = (void*)sc; op.p[6] = sample;
  op.i[0] = n;
  return cgd_run_op(&op, stream);
}
int cgd_sample_update_ddim(const float* x, const float* pred_xstart, const float* g, const float* noise, const float* sc, float* sample,
                           int64_t n, void* stream) {
  CgdOp op;
  memset(&op, 0, sizeof(op));
  op.code = CGD_OP_SAMPLE_DDIM;
  op.p[0] = (void*)x; op.p[1] = (void*)pred_xstart; op.p[2] = (void*)g; op.p[3] = (void*)noise; op.p[4] = (void*)sc; op.p[5] = sample;
  op.i[0] = n;
  return cgd_run_op(&op, stream);
}

}  // extern "C"
