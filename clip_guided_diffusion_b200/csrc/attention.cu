// attention.cu -- multi-head softmax attention ops (ATTN_FWD / ATTN_BWD): argument checks and the choice of kernel.
//
// Replaces [3P] guided-diffusion QKVAttention / QKVAttentionLegacy and [3P] CLIP nn.MultiheadAttention's core (SURVEY.md K4, K14).
// The q/k/v operands are addressed by (batch, row, head) strides so both the legacy per-head [q|k|v] interleave and the
// [q..|k..|v..] order read straight out of the fused qkv GEMM output.  Head dims 128 / 192 / 256 go to attention_wide.cu; head
// dim 64 goes to attention_small.cu when all keys fit one 64-row tile and to the flash kernels of attention_mma.cu otherwise.
#include "common.cuh"
#include "ops.cuh"

namespace cgd {

int attn_wide_supported(int64_t d);                          // attention_wide.cu: head dims 128 / 192 / 256 (the 128x128 checkpoint's 4 heads)
int launch_attn_wide_fwd(const CgdOp& op, cudaStream_t st);
int launch_attn_wide_bwd(const CgdOp& op, cudaStream_t st);
int attn_small_supported(int64_t T);                         // attention_small.cu: one 64-key tile per head on warp MMAs
int launch_attn_small_fwd(const CgdOp& op, cudaStream_t st);
int launch_attn_small_bwd(const CgdOp& op, cudaStream_t st);
int launch_attn_mma_fwd(const CgdOp& op, cudaStream_t st);   // attention_mma.cu: flash attention on warp MMAs (any T)
int launch_attn_mma_bwd(const CgdOp& op, cudaStream_t st);

static int attn_args(const CgdOp& op, bool bwd) {
  CGD_CHECK_ARG(op.i[3] == 64 || attn_wide_supported(op.i[3]), "attention: head dim %lld unsupported (64, 128, 192, 256)", (long long)op.i[3]);
  CGD_CHECK_ARG((int)op.i[0] > 0 && (int)op.i[1] > 0 && (int)op.i[2] > 0, "attention: bad dims");
  for (int k = 4; k <= 9; ++k) CGD_CHECK_ARG(op.i[k] % 8 == 0, "attention: strides must be multiples of 8 elements");
  for (int k = 0; k < 3; ++k) CGD_CHECK_ARG(op.p[k] && ((uintptr_t)op.p[k] % 16) == 0, "attention: q/k/v must be non-null and 16-byte aligned");
  if (!bwd) CGD_CHECK_ARG(op.p[3] && op.p[4], "attention: null out / lse");
  else CGD_CHECK_ARG(op.p[3] && op.p[4] && op.p[5] && op.p[6] && op.p[7] && op.p[8] && op.p[9], "attention bwd: null pointer");
  return 0;
}

int attn_bwd_num_launches(const CgdOp& op) { return (op.i[3] == 64 && attn_small_supported(op.i[2])) ? 1 : 2; }

int launch_attn_fwd(const CgdOp& op, cudaStream_t st) {
  if (int rc = attn_args(op, false)) return rc;
  if (op.i[3] != 64) return launch_attn_wide_fwd(op, st);
  if (attn_small_supported(op.i[2])) return launch_attn_small_fwd(op, st);
  return launch_attn_mma_fwd(op, st);
}

int launch_attn_bwd(const CgdOp& op, cudaStream_t st) {
  if (int rc = attn_args(op, true)) return rc;
  if (op.i[3] != 64) return launch_attn_wide_bwd(op, st);
  if (attn_small_supported(op.i[2])) return launch_attn_small_bwd(op, st);
  return launch_attn_mma_bwd(op, st);
}

}  // namespace cgd
