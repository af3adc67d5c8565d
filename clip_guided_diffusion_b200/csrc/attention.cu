// attention.cu -- multi-head softmax attention ops (ATTN_FWD / ATTN_BWD): argument checks and the choice of kernel.
//
// Replaces [3P] guided-diffusion QKVAttention / QKVAttentionLegacy and [3P] CLIP nn.MultiheadAttention's core (SURVEY.md K4, K14).
// The q/k/v operands are addressed by (batch, row, head) strides so both the legacy per-head [q|k|v] interleave and the
// [q..|k..|v..] order read straight out of the fused qkv GEMM output.  Head dim 64 goes to attention_small.cu when all keys fit
// one 64-row tile; everything else goes to the flash kernels of attention_flash.cu, which cut the head dim into d / 64 chunks.
#include "attn_mma.cuh"
#include "common.cuh"
#include "ops.cuh"

namespace cgd {

int attn_small_supported(int64_t T);                         // attention_small.cu: one 64-key tile per head on warp MMAs
int launch_attn_small_fwd(const AttnArgs& a, bool causal, cudaStream_t st);
int launch_attn_small_bwd(const AttnArgs& a, cudaStream_t st);
int launch_attn_flash_fwd(const AttnArgs& a, int nc, bool causal, cudaStream_t st);  // attention_flash.cu: flash attention, head dim 64 * nc (any T)
int launch_attn_flash_bwd(const AttnArgs& a, int nc, cudaStream_t st);

static int attn_args(const CgdOp& op, bool bwd, AttnArgs& a) {
  const int64_t d = op.i[3];
  // flags 1 (forward only) = causal; nothing differentiates a causal attention, so the backward takes no flags
  if (!bwd) CGD_CHECK_ARG((op.flags & ~1) == 0, "attention: flags %d unsupported (1 = causal)", (int)op.flags);
  else CGD_CHECK_ARG(op.flags == 0, "attention bwd: flags %d unsupported (no causal backward)", (int)op.flags);
  CGD_CHECK_ARG(d == 64 || d == 128 || d == 192 || d == 256, "attention: head dim %lld unsupported (64, 128, 192, 256)", (long long)d);
  CGD_CHECK_ARG((int)op.i[0] > 0 && (int)op.i[1] > 0 && (int)op.i[2] > 0, "attention: bad dims");
  for (int k = 4; k <= 9; ++k) CGD_CHECK_ARG(op.i[k] % 8 == 0, "attention: strides must be multiples of 8 elements");
  for (int k = 0; k < 3; ++k) CGD_CHECK_ARG(op.p[k] && ((uintptr_t)op.p[k] % 16) == 0, "attention: q/k/v must be non-null and 16-byte aligned");
  if (!bwd) CGD_CHECK_ARG(op.p[3] && op.p[4], "attention: null out / lse");
  else CGD_CHECK_ARG(op.p[3] && op.p[4] && op.p[5] && op.p[6] && op.p[7] && op.p[8] && op.p[9], "attention bwd: null pointer");
  a = AttnArgs{};
  a.B = (int)op.i[0]; a.heads = (int)op.i[1]; a.T = (int)op.i[2];
  a.qbs = op.i[4]; a.qrs = op.i[5]; a.qhs = op.i[6]; a.obs = op.i[7]; a.ors = op.i[8]; a.ohs = op.i[9];
  a.scale = op.f[0];
  a.q = (const __half*)op.p[0]; a.k = (const __half*)op.p[1]; a.v = (const __half*)op.p[2];
  if (!bwd) {
    a.out = (__half*)op.p[3]; a.lse = (float*)op.p[4];
  } else {
    a.o = (const __half*)op.p[3]; a.dout = (const __half*)op.p[4]; a.lse = (float*)op.p[5];
    a.dq = (__half*)op.p[6]; a.dk = (__half*)op.p[7]; a.dv = (__half*)op.p[8]; a.delta = (float*)op.p[9];
  }
  return 0;
}

static bool attn_small(const CgdOp& op) { return op.i[3] == 64 && attn_small_supported(op.i[2]); }

int attn_bwd_num_launches(const CgdOp& op) { return attn_small(op) ? 1 : 2; }

int launch_attn_fwd(const CgdOp& op, cudaStream_t st) {
  AttnArgs a;
  if (int rc = attn_args(op, false, a)) return rc;
  const bool causal = op.flags & 1;
  return attn_small(op) ? launch_attn_small_fwd(a, causal, st) : launch_attn_flash_fwd(a, (int)(op.i[3] / AS_T), causal, st);
}

int launch_attn_bwd(const CgdOp& op, cudaStream_t st) {
  AttnArgs a;
  if (int rc = attn_args(op, true, a)) return rc;
  return attn_small(op) ? launch_attn_small_bwd(a, st) : launch_attn_flash_bwd(a, (int)(op.i[3] / AS_T), st);
}

}  // namespace cgd
