/*
 * cgd_b200.h -- C ABI of libcgd_b200.so: the H100 (sm_90a) kernels behind the reference's
 * per-timestep CLIP-guided sampling step.
 *
 * The reference (afiaka87/clip-guided-diffusion) has no FFI of its own: its hot path is Python
 * calling PyTorch (SURVEY.md section 8b).  This header is therefore the design contract a
 * maintainer binds with ctypes (INTEGRATION.md shows the stub).  Each entry point names the
 * reference code it replaces (file:line relative to the reference tree; "[3P]" = third-party
 * package the reference imports, restated in oracle/).
 *
 * Conventions
 *   - Plain C: raw device pointers (tensor.data_ptr()), int64 dims, float scalars, a cudaStream_t
 *     passed as void*.  No torch types.
 *   - The caller owns every buffer (inputs, outputs, saved activations, workspaces); the library
 *     allocates no device memory and keeps no mutable global state besides plan handles.
 *   - Every call is asynchronous on the given stream and never synchronises the device.
 *   - Return value: 0 = ok; negative = invalid argument / unsupported shape; positive = cudaError_t.
 *     cgd_last_error() returns a thread-local message for the last non-zero return.
 *   - Activations inside the networks are "pixel-major" fp16: [rows, C] with C contiguous and an
 *     explicit row stride (ld, in elements) so channel-concatenation is a pointer offset.
 *     Images at the sampler boundary are fp32 NCHW exactly like the reference's tensors.
 *
 * The unit of work is an *op* (one kernel launch, two for split-K GEMMs / attention backward);
 * a network is a flat op list ("plan") built once by the host and replayed every timestep
 * (normally from inside a captured CUDA graph).
 */
#ifndef CGD_B200_H
#define CGD_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CGD_ABI_VERSION 3  /* 3: op codes 30, 31, 32, 49 retired; CONV i20..i22 and flags 2 reserved (must be 0); GN_*_GRID without the
                              partials-capacity operand (GN_FWD_GRID i6, GN_BWD_GRID i7)
                              2: CONV i23 clusters of `splits` CTAs (were 2 * splits), p6 unused, i18 = 3 no longer the narrow kernels */
#define CGD_OP_NI 24
#define CGD_OP_NF 8
#define CGD_OP_NP 12

typedef struct CgdOp {
  int32_t code;           /* CGD_OP_* */
  int32_t flags;          /* op-specific bits, see below */
  int64_t i[CGD_OP_NI];   /* integer operands (dims, strides in ELEMENTS) */
  float f[CGD_OP_NF];     /* float operands */
  void* p[CGD_OP_NP];     /* device pointers */
} CgdOp;

/* ------------------------------------------------------------------ op codes ------------------
 * Slot tables: iN / fN / pN are CgdOp.i[N] / .f[N] / .p[N].  "h" = fp16, "f" = fp32.
 */
enum {
  /* Implicit-GEMM convolution / GEMM on Hopper tensor cores (TMA-fed, wgmma, register accumulators).
   * Replaces [3P] UNet Conv2d 3x3 / 1x1, Conv1d k=1, and [3P] CLIP Linear / patch conv
   * (SURVEY K1-K3, K12, K13) in both directions (dgrad = same kernel, host-transformed weights).
   *   out[n,y,x,co] = sum_{tap,ci} A[n, y+dy(tap), x+dx(tap), ci] * Wp[co, tap*Cin+ci] (+bias[co]) (+res[n,y,x,co])
   *   p0 A(h)  p1 Wp(h, [Npad, taps*Cin] K-major)  p2 bias(f)|0  p3 res(h)|0  p4 out(h|f)  p5 splitK ws(f)|0
   *   i0 NB i1 H i2 W i3 Cin(%64==0) i4 Cout i5 Npad(%BN==0) i6 taps(1|9)
   *   i7..9 A strides (n,h,w)  i10..12 out strides  i13..15 res strides  i16 BN  i17 splits
   *   i18 impl (0 = wgmma, with the mma.sync kernel for narrow layers; 1 = SIMT verification kernel; 2 = the wgmma tile kernel for
   *   every layer, workspace split-K only; 3 = the wgmma tile kernel for every layer, with in-cluster split-K and the fused epilogues)  i19 out channel stride (0/1 = contiguous; >1 only
   *   with scalar stores, e.g. fp32 NCHW outputs of the UNet head / stem dgrad)
   *   i20, i21, i22 reserved (0)
   *   p6 unused (0)
   *   i23 = 1: split-K inside a thread-block cluster of `splits` CTAs, reduced through distributed shared memory (one launch, no
   *   workspace; splits in 2..8, BN >= 64, BN / splits a multiple of 16, fp16 contiguous output, Cout % 8 == 0)
   *   flags: 1 = out is fp32 ; 2 reserved (0) ; 4 = p3 is a QuickGELU pre-activation u and out = acc * QuickGELU'(u) instead of acc + res
   *   (dgrad of the CLIP MLP's c_proj writing d c_fc directly; wgmma kernel, no split-K, Cout % 8 == 0, no bias) ; 8 = the same with the
   *   exact GELU: out = acc * (Phi(u) + u phi(u)) (the OpenCLIP towers' MLPs; same preconditions; 4 | 8 is rejected) */
  CGD_OP_CONV = 1,
  /* GroupNorm(32) statistics: per (image, chunk, group) partial sum / sum of squares; the last block per image
   * folds the chunks (fixed order, fp64) into (mean, rstd).  [3P] GroupNorm32 (SURVEY K5).
   * p0 x(h) p1 partials(f [N,nchunk,32,2]) p2 stats(f [N,32,2] = mean, rstd) p3 counters(u32 [N], zero-initialised,
   * self-resetting) ; i0 N i1 HW i2 C i3 ld i4 nchunk ; f0 eps */
  CGD_OP_GN_STATS = 2,
  /* y = silu?( GN(x)*(1+scale)+shift ) ; p0 x p1 stats p2 gamma(f) p3 beta(f) p4 emb(f [N,2C] = scale|shift)|0 p5 y(h)
   * i0 N i1 HW i2 C i3 ldx i5 ldy ; flags 1 = SiLU.  (SURVEY K5, K6) */
  CGD_OP_GN_APPLY = 3,
  /* backward of GN_APPLY, pass 1: per-group sums of dxhat and dxhat*xhat.
   * p0 dy p1 x p2 stats p3 gamma p4 beta p5 emb|0 p6 partials(f [N,nchunk,32,2]) p7 sums(f [N,32,2] = means of
   * dxhat, dxhat*xhat) p8 counters(u32 [N]) ; i0 N i1 HW i2 C i3 ld_dy i4 ldx i5 nchunk ; flags 1 = SiLU */
  CGD_OP_GN_BWD_STATS = 4,
  /* pass 2: dx (=|+=) rstd*(dxhat - mean(dxhat) - xhat*mean(dxhat*xhat)).
   * p0 dy p1 x p2 stats p3 gamma p4 beta p5 emb|0 p6 sums p7 dx(h) ; i0 N i1 HW i2 C i3 ld_dy i4 ldx i6 ld_dx
   * flags 1 = SiLU, 2 = accumulate into dx */
  CGD_OP_GN_BWD_APPLY = 5,
  /* 2x2 mean pool (x scale): p0 x p1 y ; i0 N i1 H i2 W (input) i3 C i4 ldx i5 ldy ; f0 scale(0.25 = avg_pool2d).
   * [3P] ResBlock down h_upd/x_upd and the backward of nearest-up (scale 1.0). (SURVEY K7) */
  CGD_OP_POOL2 = 6,
  /* nearest x2 up-sample (x scale): p0 x p1 y ; i0 N i1 H i2 W (input) i3 C i4 ldx i5 ldy ; f0 scale.
   * Also the backward of avg-pool (scale 0.25). */
  CGD_OP_UP2 = 7,
  /* c = a + b on [rows, C] fp16: p0 a p1 b p2 c ; i0 rows i1 C i2 lda i3 ldb i4 ldc */
  CGD_OP_ADD = 8,
  /* Multi-head softmax attention forward, head dim 64 / 128 / 192 / 256 (SURVEY K4, K14).
   * p0 q p1 k p2 v p3 out p4 lse(f [B,heads,T]) ; i0 B i1 heads i2 T i3 d
   * i4 qkv batch stride i5 qkv row stride i6 qkv head stride i7 out batch stride i8 out row stride i9 out head stride
   * f0 softmax scale (applied to q.k) ; flags 1 = causal: key j > i is masked for query i (the CLIP text tower) */
  CGD_OP_ATTN_FWD = 9,
  /* backward: p0 q p1 k p2 v p3 out p4 dout p5 lse p6 dq p7 dk p8 dv p9 delta ws(f [B,heads,T])
   * i/f as forward (dq/dk/dv use the qkv strides, dout the out strides) ; flags 0 (there is no causal backward) */
  CGD_OP_ATTN_BWD = 10,
  /* Small-M fp32 linear: y[M,N] (=|+=) act(x[M,K]) @ W[N,K]^T + b.  time_embed / emb_layers / CLIP head (SURVEY K8, K16).
   * p0 x(f|h) p1 W(f|h) p2 b(f)|0 p3 y(f|h) p4 scatter(i32 [N,2] = element offset of row 0, row stride)|0 ; i0 M i1 K (% 8 == 0)
   * i2 N i3 ldx i4 ldy ; flags 1 = SiLU on x, 2 = accumulate, 4 = x is fp16, 8 = y is fp16, 16 = W is fp16.
   * With the scatter table one launch evaluates all ResBlock emb_layers (same x, concatenated W) into per-block [M, N_k] outputs. */
  CGD_OP_LINEAR_SMALL = 11,
  /* sinusoidal timestep embedding: p0 t(f [B]) p1 out(f [B,dim]) ; i0 B i1 dim ; f0 t scale */
  CGD_OP_TIMESTEP_EMB = 12,
  /* emb[b,:] += table[y[b],:] : p0 emb(f) p1 table(f) p2 y(int64) ; i0 B i1 D */
  CGD_OP_LABEL_ADD = 13,
  /* fp32 NCHW -> fp16 pixel-major zero-padded to ld channels: p0 src p1 dst ; i0 N i1 C i2 HW i3 ld ; f0 scale
   * flags 4 (C <= 3): per-channel affine (x - f[1+c]) * f[4+c] * f0 (the LPIPS ScalingLayer) */
  CGD_OP_NCHW_TO_PM = 14,
  /* pixel-major (h, or f with flag 1) -> fp32 NCHW (first C channels): p0 src p1 dst ; i0 N i1 C i2 HW i3 ld ; f0 scale
   * flags 1 = src fp32, 2 = accumulate, 4 (C <= 3) = per-channel multiplier f[1+c], 8 = image n divided by p2[n] (fp32 [N]: the
   * per-image power-of-two scale of LPIPS_SEED, so the division is exact) */
  CGD_OP_PM_TO_NCHW = 15,
  /* LayerNorm rows: p0 x(h) p1 gamma(f) p2 beta(f) p3 y(h) p4 stats(f [rows,2]) ; i0 rows i1 w i2 ldx i3 ldy ; f0 eps (SURVEY K15) */
  CGD_OP_LN_FWD = 16,
  /* p0 dy p1 x p2 gamma p3 stats p4 dx ; i0 rows i1 w i2 ld_dy i3 ldx i4 ld_dx ; flags 2 = accumulate */
  CGD_OP_LN_BWD = 17,
  /* QuickGELU a = u*sigmoid(1.702u): p0 u p1 a ; i0 n (contiguous) ; flags 1 = exact GELU a = 0.5 u (1 + erf(u / sqrt 2)) instead (fp32
   * from the fp16 u, one rounding to fp16; the OpenCLIP towers), any other flag bit is rejected */
  CGD_OP_QGELU_FWD = 18,
  /* p0 da p1 u p2 du ; i0 n */
  CGD_OP_QGELU_BWD = 19,
  /* ViT token assembly in place: tok[n,0,:] = cls ; tok[n,t,:] += pos[t,:]  : p0 tok(h [n,T,w]) p1 cls(f) p2 pos(f) ; i0 n i1 T i2 w */
  CGD_OP_VIT_EMBED = 20,
  /* MakeCutouts + CLIP_NORMALIZE, all cutouts in one launch (cgd/modules.py:60-66, cgd/clip_util.py:45,
   * cgd/cgd.py:189-193; SURVEY K11).  Input is x_in in [-1,1]; the (x+1)/2 of cgd/cgd.py:190 is folded in.
   * Output is written directly in ViT patch order: [cutn*B (row k*B+b), g*g, Kpad] with k = (c, ky, kx).
   * p0 x_in(f NCHW [B,3,H,W]) p1 coords(int32 [cutn,3] = offsetx, offsety, size) p2 patches(h)
   * i0 B i1 H i2 W i3 cutn i4 cut_size i5 patch i6 Kpad ; f0..2 mean f3..5 std */
  /* (CUTOUTS_FWD flags 1: p2 is fp32 instead of fp16 -- the stand-alone MakeCutouts surface returns fp32 like the reference) */
  CGD_OP_CUTOUTS_FWD = 21,
  /* gather-style backward (no atomics): p0 dpatches(h) p1 coords p2 dx_in(f NCHW) ; i as fwd ; f3..5 std ; f6 scale
   * flags 0 = store into dx_in ; 2 = add to it (several CLIP towers: the first stores, the others add in launch order, so the sum is
   * deterministic and bitwise old + the flags-0 result) ; any other flags are rejected
   * flags 4 (alone or with 2): p0 is fp32 d cutouts [cutn*B, 3, cs, cs] (what CUTOUTS_FWD flags 1 writes: patch i5 == cut_size,
   * Kpad i6 == 3 cut_size^2), the stand-alone MakeCutouts backward; still a gather, so the sum is deterministic */
  CGD_OP_CUTOUTS_BWD = 22,
  /* spherical_dist_loss + prompt weights + cutout mean, with analytic d/d(embed) (cgd/losses.py:10-14,
   * cgd/cgd.py:196-200,204; SURVEY K17).  p0 emb(f [cutn*B, D]) p1 targets(f [P,D]) p2 weights(f [P])
   * p3 d_emb(f) p4 loss(f [B], += clip term) ; i0 cutn i1 B i2 P i3 D ; f0 clip_guidance_scale f1 grad scale */
  CGD_OP_SPHERICAL = 23,
  /* p_mean_variance algebra + blend ([3P] GaussianDiffusion.p_mean_variance, cgd/cgd.py:177-179; SURVEY K9, K10).
   * p0 x(f NCHW [B,3,HW]) p1 model_out(f NCHW [B,6,HW]) p2 sc(f, per-step scalars) p3 pred_xstart p4 mean p5 variance
   * p6 log_variance p7 x_in p8 loss buffer to zero|0 ; i0 B i1 HW i2 number of floats to zero (<= 256).
   * p4..p7 may be null.  sc[] indices: CGD_SC_* */
  CGD_OP_PMV_BLEND = 24,
  /* tv_loss + range_loss (+ sat) forward and analytic backward, merged with the CLIP-path gradient
   * (cgd/losses.py:5-7,17-22, cgd/cgd.py:201-218; SURVEY K18, K19).
   * p0 x_in(f) p1 pred_xstart(f) p2 g_clip(f, dL/dx_in from the CLIP path)|0 p3 sc p4 seed(h pixel-major [B*HW, ld], UNet dgrad seed)
   * p5 dx_direct(f NCHW) p6 loss(f [3B] = tv[B], range[B], sat[B]) ; i0 B i1 H i2 W i3 ld i4 batch of the whole job (sat is
   * mean over ALL ranks' images, cgd/cgd.py:215; 0 = B) ; f0 tv_scale f1 range_scale f2 sat_scale f3 seed scale
   * flags 1 = dynamic seed scaling: p7 seed_f32(f [B,HW,3]) p8 dyn(f [2B]) are written instead of p4 (see CGD_OP_SEED_QUANT), f3 unused */
  CGD_OP_GUIDE_GRAD = 25,
  /* g = -(dx_direct + dx_unet / seed scale), optional RMS clamp (cgd/cgd.py:228-232; SURVEY K20).
   * p0 dx_direct(f NCHW) p1 dx_unet(f NCHW, still multiplied by the seed scale)|0 p2 g(f NCHW) p3 ws(f [128])|0
   * i0 B i1 HW ; f0 1/seed scale f1 max rms ; flags 1 = use_magnitude (whole-batch RMS clamp, two launches),
   * flags 2 = dynamic seed scaling: p4 dyn(f [2B]), per-image 1/scale instead of f0
   * flags 4 (with 1) = only the partial sums of squares are written to ws; the clamp is a separate CGD_OP_MAG_CLAMP (batch sharded
   * over ranks: the caller all-reduces ws in between) */
  CGD_OP_FINAL_GRAD = 26,
  /* ancestral update ([3P] p_sample_with_grad / condition_mean_with_grad): sample = mean + var*g + nz*exp(.5 logvar)*noise
   * p0 mean p1 variance p2 log_variance p3 g|0 p4 noise p5 sc p6 sample ; i0 n elements */
  CGD_OP_SAMPLE_ANCESTRAL = 27,
  /* DDIM update ([3P] ddim_sample_with_grad / condition_score_with_grad), eta from sc
   * p0 x p1 pred_xstart p2 g|0 p3 noise p4 sc p5 sample ; i0 n elements */
  CGD_OP_SAMPLE_DDIM = 28,
  /* fp16 copy of a [rows, C] block: p0 src p1 dst ; i0 rows i1 C i2 lds i3 ldd */
  CGD_OP_COPY = 29,
  /* 30, 31, 32 retired (batched-GEMM attention: TRANSPOSE, SOFTMAX_FWD, SOFTMAX_BWD); not to be reused */
  /* single-launch GroupNorm(32) forward for activations whose (image, group) slab fits one thread-block cluster's
   * registers (C % 256 == 0, ceil(HW / CS) <= 16 * 512 / vectors-per-pixel): exact two-pass statistics exchanged through
   * distributed shared memory, y = silu?( GN(x)*(1+scale)+shift ), stats written for the backward.
   * p0 x(h) p1 gamma(f) p2 beta(f) p3 emb(f [N,2C])|0 p4 y(h) p5 stats(f [N,32,2] = mean, rstd)
   * i0 N i1 HW i2 C i3 ldx i4 ldy i5 CS (cluster size 1|2|4|8 along the pixels) ; f0 eps ; flags 1 = SiLU */
  CGD_OP_GN_FWD_FUSED = 33,
  /* single-launch backward of the above (same math as GN_BWD_STATS + GN_BWD_APPLY; slab limit 8 * 512 / vectors-per-pixel)
   * p0 dy p1 x p2 stats p3 gamma p4 beta p5 emb|0 p6 dx(h) ; i0 N i1 HW i2 C i3 ld_dy i4 ldx i5 ld_dx i6 CS
   * flags 1 = SiLU, 2 = accumulate into dx */
  CGD_OP_GN_BWD_FUSED = 34,
  /* single persistent launch for LARGE activations: statistics pass, grid-wide barrier (generation counted, no reset needed),
   * apply pass over the same pixel range (L2 hit).  One 512-thread CTA per SM: N * Gn must not exceed the SM count.
   * p0 x(h) p1 gamma p2 beta p3 emb|0 p4 y(h) p5 stats(f [N,32,2]) p6 partials(f [N,Gn,32,2]) p7 barrier(u32 [2], zero-initialised)
   * i0 N i1 HW i2 C i3 ldx i4 ldy i5 Gn (CTAs per image) ; f0 eps ; flags 1 = SiLU.  C % 64 == 0 */
  CGD_OP_GN_FWD_GRID = 35,
  /* backward of the above: p0 dy p1 x p2 stats p3 gamma p4 beta p5 emb|0 p6 dx(h) p7 partials(f [N,Gn,32,2]) p8 barrier
   * p9 scratch(h, dense [N,HW,C])|0: d xhat is stored once and streamed back instead of recomputing SiLU' in the apply pass
   * i0 N i1 HW i2 C i3 ld_dy i4 ldx i5 ld_dx i6 Gn ; flags 1 = SiLU, 2 = accumulate into dx */
  CGD_OP_GN_BWD_GRID = 36,
  /* y = max(x, 0) on n fp16 elements (n % 8 == 0; in place allowed): p0 x p1 y ; i0 n.  [3P] VGG16 ReLU of lpips.LPIPS (K21) */
  CGD_OP_RELU_FWD = 37,
  /* dx (=|+=) dy where y > 0: p0 dy p1 y (ReLU output) p2 dx ; i0 n ; flags 2 = accumulate */
  CGD_OP_RELU_BWD = 38,
  /* 2x2 stride-2 max pool on pixel-major [N,H,W,C] (H, W even, C % 8 == 0): p0 x p1 y ; i0 N i1 H i2 W i3 C */
  CGD_OP_MAXPOOL2_FWD = 39,
  /* its input gradient (dy to the first window position holding the maximum, like ATen): p0 dy p1 x p2 dx ; i0 N i1 H i2 W i3 C */
  CGD_OP_MAXPOOL2_BWD = 40,
  /* one LPIPS tap: xh = f / (||f||_C + 1e-10); loss[b] += mean_p sum_c w_c (xh - tn)^2 ; df = f0 * d loss / d f.
   * p0 f(h [B,HW,C]) p1 tn(h [Bt,HW,C], normalised init-image features) p2 w(f [C]) p3 df(h) p4 loss(f [B], accumulated)
   * i0 B i1 HW i2 C (<= 512) i3 Bt (1 = broadcast) ; f0 gradient scale.  cgd/cgd.py:220-224, SURVEY A.4 */
  CGD_OP_LPIPS_TAP = 41,
  /* dst[0..n) = f0 (fp32): p0 dst ; i0 n */
  CGD_OP_FILL = 42,
  /* MakeCutouts in ResizeRight mode (lanczos3, antialiased; cgd/ResizeRight/resize_right.py:31-122): like CUTOUTS_FWD / _BWD with
   * host-built separable tables per cutout: p3 left(i32 [cutn,cs]) p4 weights(f [cutn,cs,16]) p5 taps(i32 [cutn]) (fwd)
   * / inverse ranges(i32 [cutn,Smax,2]) (bwd) ; i7 Smax >= min(H, W) (bwd; fwd with flags 2).  The crop of window (ox, oy, S) is
   * Sy x Sx = min(S, H - oy) x min(S, W - ox), as the reference's slicing clips it.  Unknown flags are rejected.
   * flags 1: p6 left p7 weights p8 taps (fwd) / inverse ranges (bwd) of the x axis, built for Sx (p3..p5 then hold the y axis's, for
   *   Sy); without it one table set serves both axes (square crops)
   * flags 2 (use_augs): fwd reads p0 = the augmented crops CUTOUTS_AUG_FWD flags 1 wrote (f [cutn,B,3,Smax,Smax], values in [0, 1],
   *   origin 0) and normalises (acc - mean) / std ; bwd stores d crop (f [cutn,B,3,Smax,Smax], Sy x Sx of each plane) into p2 instead of
   *   gathering into dx_in, for CUTOUTS_AUG_BWD flags 1 */
  CGD_OP_CUTOUTS_RR_FWD = 43,
  CGD_OP_CUTOUTS_RR_BWD = 44,
  /* dynamic scaling of the UNet-backward seed (GUIDE_GRAD flags 1 writes the fp32 seed p7 and the per-image max |.| into p8[0..B)):
   * scale_b = 2^floor(log2(4096 / max_b)); seed(h, [B,HW,ld], channels 0..2) = seed_f32 * scale_b; p8[B + b] = scale_b.
   * p0 seed_f32(f [B,HW,3]) p1 dyn(f [2B]) p2 seed(h) ; i0 B i1 HW i2 ld.  FINAL_GRAD flags 2 (p4 = dyn) divides dx_unet by
   * scale_b and resets the maxima. */
  CGD_OP_SEED_QUANT = 45,
  /* whole-batch RMS clamp of cgd/cgd.py:229-232 from (all-reduced) partial sums: g *= min(rms, f0) / rms, rms = sqrt(sum(ws) / i1).
   * p0 g(f, i0 local elements) p1 ws(f [128]) ; i0 n local i1 n of the whole batch ; f0 max rms */
  CGD_OP_MAG_CLAMP = 46,
  /* CLIP ModifiedResNet AttentionPool2d token assembly ([3P] clip/model.py): y[n,0,:] = mean_t x[n,t,:] + pos[0,:] ;
   * y[n,1+t,:] = x[n,t,:] + pos[1+t,:].  p0 x(h [n,HW,C], row stride i3) p1 pos(f [HW+1,C]) p2 y(h [n,HW+1,C]) ; i0 n i1 HW i2 C i3 ldx */
  CGD_OP_ATTNPOOL_EMBED_FWD = 47,
  /* dx[n,t,:] (=|+=) dy[n,1+t,:] + dy[n,0,:] / HW : p0 dy(h [n,HW+1,C]) p1 dx(h, row stride i3) ; i0 n i1 HW i2 C i3 ld_dx ; flags 2 = accumulate */
  CGD_OP_ATTNPOOL_EMBED_BWD = 48,
  /* 49 retired (GroupNorm from conv-epilogue statistics: GN_APPLY_EPI); not to be reused */
  /* MakeCutouts with use_augs=True (cgd/modules.py:12-24, 60-64): crop -> RandomHorizontalFlip -> +noise -> RandomAffine (nearest,
   * fill 0) -> +noise -> RandomPerspective (bilinear, fill 0) -> +noise -> RandomGrayscale -> +noise -> adaptive_avg_pool2d ->
   * CLIP_NORMALIZE, one gather launch; like CUTOUTS_FWD plus p3 params(f [cutn,20]: flip | inverse affine matrix[6] | perspective on |
   * coefficients[8] | grayscale | 3 reserved -- drawn on the host in torchvision's order, clip_guided_diffusion_b200/augs.py)
   * p4 noise(f [cutn,4,B,3,Smax,Smax], the four N(0, .01^2) fields of every cutout)|0 ; i7 Smax (row stride of the noise planes).
   * _BWD: the transposed gather scattered with fp32 atomics INTO p2 dx (zero it first: CGD_OP_FILL); p3 params; f6 gradient scale;
   * flags 4: p0 is fp32 d cutouts [cutn*B, 3, cs, cs] (patch i5 == cut_size, Kpad i6 == 3 cut_size^2) instead of fp16 patch rows
   * flags 1 (ResizeRight after use_augs): _FWD writes the augmented crops themselves, f [cutn,B,3,Smax,Smax] in [0, 1] (Sy x Sx of each
   * plane), into p2 instead of pooled patches, for CUTOUTS_RR_FWD flags 2; _BWD reads p0 = d crop in that layout (CUTOUTS_RR_BWD flags 2)
   * and scatters it through the augmentations into p2 (f6 scale; i7 Smax) */
  CGD_OP_CUTOUTS_AUG_FWD = 50,
  CGD_OP_CUTOUTS_AUG_BWD = 51,
  /* one axis of a separable resampling (image prompts: ResizeRight lanczos3 with antialiasing, cgd/clip_util.py:95-97), with host-built
   * tables of any tap count: out[.., o, ..] = sum_{i<T} w[o,i] * in[.., left[o] + i, ..], samples outside [0, S) are zero; fp32, summed
   * in tap order.  p0 in(f [planes, H, W]) p1 out(f [planes, O, W] for axis 0, [planes, H, O] for axis 1) p2 left(i32 [O])
   * p3 weights(f [O, T]) ; i0 planes i1 H i2 W i3 axis (0 = H, 1 = W) i4 O i5 T */
  CGD_OP_RESIZE_AXIS = 52,
  /* CLIP text tower input ([3P] clip/model.py encode_text): x[n,t,:] = fp16(table[ids[n,t],:] + pos[t,:]), the sum in fp32.
   * p0 ids(i32 [n,T]) p1 table(h [V,w]) p2 pos(f [T,w]) p3 x(h [n,T,w]) ; i0 n i1 T i2 w (% 8 == 0) i3 V.
   * An id outside [0, V) gives a row of NaNs (never a read outside the table); callers check ids on the host. */
  CGD_OP_TOKEN_EMBED = 53,
  /* y[i,:] = x[idx[i],:] on fp16 rows (the end-of-text token of every sequence: idx[i] = i * T + eot_i).
   * p0 x(h [n_src rows, row stride i2]) p1 idx(i32 [rows], 4-byte aligned) p2 y(h [rows, row stride i3]) ; i0 rows i1 w (% 8 == 0) i2 ldx i3 ldy
   * i4 n_src.  An index outside [0, n_src) gives a row of NaNs. */
  CGD_OP_ROW_GATHER = 54,
  /* The UNet under torch.autograd (clip_guided_diffusion_b200/guidance.py, EngineModel): a cond_fn's d loss / d model_out seeds the
   * input-gradient plan.  d_out(f NCHW [B,6,HW]) -> seed(h pixel-major [B,HW,ld], channels 0..5) * scale_b, with SEED_QUANT's per-image
   * power of two: pass 1 puts max_b |d_out| into dyn[b] (atomicMax on the float bits; a NaN is dropped, an inf counts as 3e38; dyn[0..B)
   * must be 0 on entry), pass 2 scale_b = 2^clamp(floor(log2(4096 / max_b)), -60, 60) (1 for an all-zero image), values saturated at
   * +-60000, dyn[B + b] = scale_b.  Two launches.  p0 d_out p1 dyn(f [2B]) p2 seed ; i0 B i1 HW i2 ld (even, >= 6) */
  CGD_OP_GRAD_SEED = 55,
  /* dx = dx_unet / scale_b (+ dx_direct), then dyn[0..B) = 0 and seed channels 0..5 = 0 (the fused step's GUIDE_GRAD / SEED_QUANT write
   * channels 0..2 only).  p0 dx_unet(f NCHW [B,3,HW]) p1 dx_direct(f NCHW)|0 p2 dyn(f [2B]) p3 seed(h [B,HW,ld]) p4 dx(f NCHW)
   * i0 B i1 HW i2 ld */
  CGD_OP_GRAD_UNSCALE = 56,
  /* transpose of CGD_OP_PMV_BLEND's p_mean_variance algebra (without the x_in blend): G = g_x0 + c1 g_mean ; d_out[:, 0:3] = -bb G ;
   * d_out[:, 3:6] = (maxl - minl) / 2 * (g_logvar + variance * g_variance) ; dx_direct = a G + c2 g_mean.
   * p0 sc p1 variance(f NCHW [B,3,HW], needed with p4) p2 g_pred_xstart|0 p3 g_mean|0 p4 g_variance|0 p5 g_log_variance|0
   * p6 d_out(f NCHW [B,6,HW]) p7 dx_direct(f NCHW [B,3,HW]) ; i0 B i1 HW */
  CGD_OP_PMV_BWD = 57,
  /* A CLIP visual tower under torch.autograd (clip_guided_diffusion_b200/clip_model.py, load_clip): a user's NCHW image batch becomes the
   * tower's patch rows, k = (c, ky, kx) within a P x P patch, G = R / P patches per side (the ViTs' patch size, P = 2 for the ModifiedResNet
   * towers' space-to-depth stem).  patches[b, gy*G + gx, c*P*P + ky*P + kx] = fp16_rn(x[b, c, gy*P + ky, gx*P + kx]) for b < n; columns
   * 3*P*P..kpad and rows n..n_built are zero.  One rounding per element, 128-bit stores.
   * p0 x(f NCHW [n,3,R,R]) p1 patches(h [n_built, G*G, kpad], 16-byte aligned) ; i0 n i1 n_built i2 R i3 P i4 kpad (% 8 == 0, >= 3*P*P) */
  CGD_OP_CLIP_PATCHIFY = 58,
  /* the dynamic loss scale of the tower backward, one CTA per image: m_b = max |d[b, :]| (a NaN is dropped, an inf counts as 3e38),
   * scale_b = 2^clamp(floor(log2(f0 / m_b)), -60, 60) (1 for an all-zero row), d_embeds[b, :] = d[b, :] * scale_b, dyn[b] = scale_b;
   * rows n..n_built get zeros and scale 1.  f0 = BAND, the target of the largest seed value: 2^9 (clip_model.py CLIP_SEED_BAND), the
   * largest power of two that left 2^4 or more of headroom below 65504 in every fp16 gradient buffer of the seeded ViT-B/32, ViT-B/16,
   * ViT-L/14 and RN50 towers at 16 images: 2^4.46 (ViT-B/16) to 2^6.88 (RN50) on an H100 (scripts/clip_seed_band.py, DESIGN.md section 2;
   * seeded weights, not the published checkpoints).
   * p0 d(f [n_built, D]) p1 d_embeds(f [n_built, D]) p2 dyn(f [n_built]) ; i0 n i1 n_built i2 D (<= 1024) ; f0 BAND (a power of two) */
  CGD_OP_CLIP_SEED = 59,
  /* transpose of CGD_OP_CLIP_PATCHIFY with the seed's scale undone: dx[b, c, gy*P + ky, gx*P + kx] = float(d_patches[b, gy*G + gx,
   * c*P*P + ky*P + kx]) * (1 / dyn[b]) for b < n (exact: the scale is a power of two); pad columns and rows n.. are not read.
   * p0 d_patches(h [n_built, G*G, kpad]) p1 dyn(f [n_built]) p2 dx(f NCHW [n,3,R,R]) ; i0 n i1 n_built i2 R i3 P i4 kpad */
  CGD_OP_CLIP_UNPATCHIFY = 60,
  /* LPIPS(in0, in1) under torch.autograd (clip_guided_diffusion_b200/lpips.py, LPIPS): one VGG16 trunk per side over the same weights,
   * tap features f0 (h [N0, HW, C]) and f1 (h [N1, HW, C]) post-ReLU, N0 and N1 each B or 1 (row 0 broadcast over the B images).
   * Per tap, per pixel: sum_c w_c (f0_c / (||f0|| + 1e-10) - f1_c / (||f1|| + 1e-10))^2.  Nothing normalised is stored, no atomics.
   * LPIPS_PAIR_FWD: grid (nblk, B) of 8-warp CTAs, each CTA's pixel sum (fixed order) into partial[b * nblk + cta].
   * p0 f0 p1 f1 p2 w(f [C]) p3 partial(f [B, nblk]) ; i0 B i1 HW i2 C (% 8 == 0, <= 512) i3 N0 i4 N1 i5 nblk (1..4096) */
  CGD_OP_LPIPS_PAIR_FWD = 61,
  /* loss[b] = sum over taps k = 0..4 in order of (sum of tap k's nblk_k partials of image b, fixed order) * f_k (= 1 / HW_k): two runs give
   * the same bits.  p0..p4 partials of taps 0..4 p5 loss(f [B]) ; i0 B i1..i5 nblk of taps 0..4 ; f0..f4 1 / HW of taps 0..4 */
  CGD_OP_LPIPS_LOSS = 62,
  /* the dynamic loss scale of the two trunk backwards from the upstream d_loss alone (the backward is linear in it): for trunk row j of
   * [trunk 0's N0 rows | trunk 1's N1 rows], m = |d_loss[b]| for a row of its own image b, the maximum over all B images for a broadcast
   * row (a NaN is dropped, an inf counts as 3e38); dyn[j] = 2^clamp(floor(log2(f0 / m)), -60, 60), 1 where m == 0.  f0 = BAND, the
   * target of |d_loss| * scale: 2^23 (lpips.py LPIPS_SEED_BAND), the largest power of two that left 2^4 or more of headroom below 65504
   * in every fp16 gradient buffer at 64^2, 256^2 and 512^2 on seeded weights (scripts/lpips_seed_band.py, DESIGN.md section 2).
   * p0 d_loss(f [B]) p1 dyn(f [N0 + N1]) ; i0 B i1 N0 i2 N1 ; f0 BAND (a power of two in [1, 2^30]) */
  CGD_OP_LPIPS_SEED = 63,
  /* the per-tap seeds of the trunk backwards: d f_side[row] = sum over the images b the row serves (in order, fp32) of
   * (d_loss[b] * dyn[row]) / HW * d LPIPS_tap_b / d f_side[row], rounded once to fp16.  Finite values saturate at +-60000 (like GRAD_SEED);
   * inf and NaN pass, so a non-finite d_loss[b] gives a non-finite seed and never a finite wrong one.  Deviation from the fp32 math: at a
   * pixel where every channel of the tap is zero after ReLU the factor 1 / (||f|| + 1e-10) makes the true gradient ~1e10 times its usual
   * size; the seed holds +-60000 there instead of overflowing to inf (the fused LPIPS_TAP would store inf).
   * p0 f0 p1 f1 p2 w(f [C]) p3 d_loss(f [B]) p4 dyn(f [N0 + N1]) p5 d f0(h [N0, HW, C])|0 p6 d f1(h [N1, HW, C])|0 ;
   * i0 B i1 HW i2 C i3 N0 i4 N1 ; flags 1 = write d f0, 2 = write d f1 (p5 / p6 set exactly for the selected sides) */
  CGD_OP_LPIPS_PAIR_BWD = 64,
  /* The reference's tv_loss / range_loss (cgd/losses.py:5-7, 17-22) per image of x (f NCHW [B, C, H, W]) for a PyTorch cond_fn
   * (clip_guided_diffusion_b200/losses.py): flags 1 = tv_loss (replicate pad: sum of squared right and down differences), 2 = range_loss
   * (sum of (x - clamp(x, -1, 1))^2), each divided by C*H*W.  Two launches: a grid (nblk, B) writes each CTA's sum (fixed order) to
   * partial[b * nblk + j], then loss[b] = the nblk partials of image b summed in order / (C*H*W).  No atomics: two runs give the same bits.
   * p0 x p1 partial(f [B, nblk]) p2 loss(f [B]) ; i0 B i1 C i2 H i3 W i4 nblk (1..4096) */
  CGD_OP_IMG_LOSS_FWD = 65,
  /* dx = d_loss[b] * d loss_b / d x, one elementwise pass (flags as IMG_LOSS_FWD).  p0 x p1 d_loss(f [B]) p2 dx(f NCHW) ; i0 B i1 C i2 H i3 W */
  CGD_OP_IMG_LOSS_BWD = 66,
  /* spherical_dist_loss (cgd/losses.py:10-14) over a list of row pairs: out[m] = 2 asin(min(|x^ - y^| / 2, 1))^2 with
   * x^ = x[pairs[m][0]] / max(||.||, 1e-12) and y^ = y[pairs[m][1]] likewise (F.normalize).  The host maps any broadcast of x [..., D]
   * against y [..., D] to the pair list.  A row index out of range gives NaN.
   * p0 x(f [Nx, D]) p1 y(f [Ny, D]) p2 pairs(i32 [M, 2]) p3 out(f [M]) ; i0 M i1 D i2 Nx i3 Ny */
  CGD_OP_SPH_DIST_FWD = 67,
  /* its input gradients from d_out (f [M]): every row of x (flags 1) and / or y (flags 2) sums d_out[m] * d out[m] / d row over the
   * pairs that use it, in the order of a host-built CSR (ptr i32 [N + 1], idx i32 [M] = pair ids), then goes back through the
   * normalisation.  A gather, no atomics.  An index out of range makes the row NaN.
   * p0 x p1 y p2 pairs p3 d_out p4 dx(f [Nx, D])|0 p5 dy(f [Ny, D])|0 p6 x ptr|0 p7 x idx|0 p8 y ptr|0 p9 y idx|0 (set exactly for the
   * selected sides) ; i0 M i1 D i2 Nx i3 Ny */
  CGD_OP_SPH_DIST_BWD = 68,
  CGD_OP__COUNT
};

/* per-step scalar table (device fp32 array, refreshed by one H2D copy per step) */
enum {
  CGD_SC_SQRT_RECIP_AC = 0,   /* sqrt(1/abar_t)                 */
  CGD_SC_SQRT_RECIPM1_AC = 1, /* sqrt(1/abar_t - 1)             */
  CGD_SC_POST_COEF1 = 2,      /* posterior_mean_coef1[t]        */
  CGD_SC_POST_COEF2 = 3,      /* posterior_mean_coef2[t]        */
  CGD_SC_MIN_LOG = 4,         /* posterior_log_variance_clipped */
  CGD_SC_MAX_LOG = 5,         /* log(beta_t)                    */
  CGD_SC_FAC = 6,             /* sqrt(1-abar)[current_timestep] (cgd/cgd.py:177) */
  CGD_SC_NONZERO = 7,         /* 1 if t != 0 else 0             */
  CGD_SC_SQRT_1M_AC = 8,      /* sqrt(1-abar_t)                 */
  CGD_SC_AC_PREV = 9,         /* abar_{t-1}                     */
  CGD_SC_AC = 10,             /* abar_t                         */
  CGD_SC_ETA = 11,            /* DDIM eta                       */
  CGD_SC_ONE_MINUS_FAC = 12,  /* 1 - fac, rounded from fp64 like the reference's `sigmas` (cgd/cgd.py:178) */
  CGD_SC__COUNT = 16
};

/* ------------------------------------------------------------------ entry points --------------- */
int cgd_abi_version(void);
const char* cgd_last_error(void);
/* How many thread-block clusters of `splits` CTAs of the in-cluster split-K conv kernel (CONV i23 = 1, tile width bn in
 * {64, 128, 192, 256}) the current device holds at once (cudaOccupancyMaxActiveClusters); -1 without a device.  Plans use it to
 * keep such a layer within one wave of clusters. */
int cgd_conv_cluster_capacity(int32_t bn, int32_t splits);

/* Validate an op list, pre-encode TMA descriptors, return a handle.  The op array is copied. */
int cgd_plan_create(const CgdOp* ops, int32_t n_ops, void** plan_out);
/* Launch ops [first, first+count) on `stream` (cudaStream_t). */
int cgd_plan_run(void* plan, int32_t first, int32_t count, void* stream);
/* Number of kernel launches ops [first, first+count) perform. */
int cgd_plan_num_launches(void* plan, int32_t first, int32_t count);
int cgd_plan_destroy(void* plan);
/* One-off execution of a single op (no plan; TMA descriptors encoded on the fly). */
int cgd_run_op(const CgdOp* op, void* stream);

/* Network-level aliases named in SURVEY.md 8b: a UNet / ViT handle is a plan whose op list holds the
 * forward segment [0, n_fwd) and the input-gradient backward segment [n_fwd, n_ops).
 *   cgd_unet_fwd        replaces [3P] UNetModel.forward               (called inside p_mean_variance)
 *   cgd_unet_bwd_input  replaces autograd of it w.r.t. x              (cgd/cgd.py:228)
 *   cgd_vit_fwd / _bwd_input  replace [3P] CLIP.encode_image fwd/bwd  (cgd/cgd.py:194,228) */
int cgd_unet_create(const CgdOp* ops, int32_t n_fwd, int32_t n_bwd, void** handle_out);
int cgd_unet_fwd(void* handle, void* stream);
int cgd_unet_bwd_input(void* handle, void* stream);
int cgd_unet_destroy(void* handle);
int cgd_vit_create(const CgdOp* ops, int32_t n_fwd, int32_t n_bwd, void** handle_out);
int cgd_vit_fwd(void* handle, void* stream);
int cgd_vit_bwd_input(void* handle, void* stream);
int cgd_vit_destroy(void* handle);
/* The whole guided step (UNet fwd -> cond_fn -> UNet dgrad -> update) as one op list. */
int cgd_step_create(const CgdOp* ops, int32_t n_ops, void** handle_out);
int cgd_step(void* handle, void* stream);
int cgd_step_destroy(void* handle);

/* Stand-alone operator entry points (each = one op; arguments as in the op tables above). */
int cgd_cutouts_fwd(const float* x_in, const int32_t* coords, void* patches_h, int64_t B, int64_t H, int64_t W,
                    int64_t cutn, int64_t cut_size, int64_t patch, int64_t kpad, const float* mean3,
                    const float* std3, void* stream);
int cgd_cutouts_bwd(const void* dpatches_h, const int32_t* coords, float* dx_in, int64_t B, int64_t H, int64_t W,
                    int64_t cutn, int64_t cut_size, int64_t patch, int64_t kpad, const float* std3, float scale,
                    void* stream);
int cgd_spherical_fwd_bwd(const float* emb, const float* targets, const float* weights, float* d_emb, float* loss,
                          int64_t cutn, int64_t B, int64_t P, int64_t D, float clip_guidance_scale,
                          float grad_scale, void* stream);
int cgd_guidance_losses_fwd_bwd(const float* x_in, const float* pred_xstart, const float* g_clip, const float* sc,
                                void* seed_h, float* dx_direct, float* loss, int64_t B, int64_t H, int64_t W,
                                int64_t ld, float tv_scale, float range_scale, float sat_scale, float seed_scale,
                                void* stream);
int cgd_sample_update_ancestral(const float* mean, const float* variance, const float* log_variance, const float* g,
                                const float* noise, const float* sc, float* sample, int64_t n, void* stream);
int cgd_sample_update_ddim(const float* x, const float* pred_xstart, const float* g, const float* noise,
                           const float* sc, float* sample, int64_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CGD_B200_H */
