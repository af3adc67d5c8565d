// elementwise.cu -- resampling, residual adds, layout conversion, embeddings, QuickGELU.
//
// The HBM-bound glue of the [3P] UNet / ViT graphs that the reference issues as many small ATen launches
// (SURVEY.md K6, K7, K8, K15): 128-bit vectorised, coalesced along channels, grid-stride loops sized to a
// multiple of the 132 SMs.
#include "common.cuh"
#include "pdl.cuh"
#include "ops.cuh"

namespace cgd {

static inline int ew_blocks(int64_t work_items, int threads = 256) {
  int64_t b = ceil_div(work_items, threads);
  const int64_t cap = 132 * 8;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

// Index arithmetic: these kernels decode a flat index into (n, y, x, vector).  With int64 operands every / and % is a ~100-instruction
// software routine and the decode, not the memory system, would bound them.  IdxT = uint32_t whenever the element count allows (always, here).
// ---- 2x2 pooling (sum * scale) on pixel-major [N,H,W,C]
template <typename IdxT>
__global__ void pool2_kernel(const __half* __restrict__ x, __half* __restrict__ y, int N, int H, int W, int C, int64_t ldx,
                             int64_t ldy, float scale) {
  pdl_wait();
  pdl_launch_dependents();
  const IdxT V = (IdxT)(C / 8), Ho = (IdxT)(H / 2), Wo = (IdxT)(W / 2);
  const IdxT total = (IdxT)N * Ho * Wo * V;
  for (IdxT idx = (IdxT)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (IdxT)gridDim.x * blockDim.x) {
    const IdxT pixv = idx / V;
    const int v = (int)(idx - pixv * V);
    const IdxT row = pixv / Wo;
    const int xo = (int)(pixv - row * Wo);
    const IdxT n_ = row / Ho;
    const int yo = (int)(row - n_ * Ho), n = (int)n_;
    const __half* s = x + (((int64_t)n * H + 2 * yo) * W + 2 * xo) * ldx + v * 8;
    float a[8], b[8], c[8], d[8], o[8];
    unpack8(ld8(s), a);
    unpack8(ld8(s + ldx), b);
    unpack8(ld8(s + (int64_t)W * ldx), c);
    unpack8(ld8(s + (int64_t)W * ldx + ldx), d);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = (a[j] + b[j] + c[j] + d[j]) * scale;
    st8(y + (((int64_t)n * Ho + yo) * Wo + xo) * ldy + v * 8, pack8(o));
  }
}
// ---- nearest x2 up-sampling (* scale): one thread per INPUT vector, written to its four output pixels
template <typename IdxT>
__global__ void up2_kernel(const __half* __restrict__ x, __half* __restrict__ y, int N, int H, int W, int C, int64_t ldx,
                           int64_t ldy, float scale) {
  pdl_wait();
  pdl_launch_dependents();
  const IdxT V = (IdxT)(C / 8), Hi = (IdxT)H, Wi = (IdxT)W;
  const int64_t Wo = 2 * (int64_t)W;
  const IdxT total = (IdxT)N * Hi * Wi * V;
  for (IdxT idx = (IdxT)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (IdxT)gridDim.x * blockDim.x) {
    const IdxT pixv = idx / V;
    const int v = (int)(idx - pixv * V);
    const IdxT row = pixv / Wi;
    const int xi = (int)(pixv - row * Wi);
    const IdxT n_ = row / Hi;
    const int yi = (int)(row - n_ * Hi), n = (int)n_;
    half8 h = ld8(x + (((int64_t)n * H + yi) * W + xi) * ldx + v * 8);
    if (scale != 1.f) {
      float a[8];
      unpack8(h, a);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] *= scale;
      h = pack8(a);
    }
    __half* o = y + (((int64_t)n * 2 * H + 2 * yi) * Wo + 2 * xi) * ldy + v * 8;
    st8(o, h);
    st8(o + ldy, h);
    st8(o + Wo * ldy, h);
    st8(o + Wo * ldy + ldy, h);
  }
}
__global__ void add_kernel(const __half* __restrict__ a, const __half* __restrict__ b, __half* __restrict__ c, int64_t rows, int C,
                           int64_t lda, int64_t ldb, int64_t ldc) {
  pdl_wait();
  pdl_launch_dependents();
  const int V = C / 8;
  const int64_t total = rows * V;
  const bool small = total + (int64_t)gridDim.x * blockDim.x < (int64_t(1) << 32);  // 32-bit decode (a 64-bit / and % cost ~200 instructions)
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = small ? (int64_t)((uint32_t)idx / (uint32_t)V) : idx / V;
    const int v = (int)(idx - r * V);
    float x[8], y[8];
    unpack8(ld8(a + r * lda + v * 8), x);
    unpack8(ld8(b + r * ldb + v * 8), y);
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] += y[j];
    st8(c + r * ldc + v * 8, pack8(x));
  }
}
__global__ void copy_kernel(const __half* __restrict__ a, __half* __restrict__ c, int64_t rows, int C, int64_t lda, int64_t ldc) {
  pdl_wait();
  pdl_launch_dependents();
  const int V = C / 8;
  const int64_t total = rows * V;
  const bool small = total + (int64_t)gridDim.x * blockDim.x < (int64_t(1) << 32);
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = small ? (int64_t)((uint32_t)idx / (uint32_t)V) : idx / V;
    const int v = (int)(idx - r * V);
    st8(c + r * ldc + v * 8, ld8(a + r * lda + v * 8));
  }
}

int launch_pool2(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], H = op.i[1], W = op.i[2], C = op.i[3], ldx = op.i[4], ldy = op.i[5];
  CGD_CHECK_ARG(N > 0 && H % 2 == 0 && W % 2 == 0 && C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0 && op.p[0] && op.p[1], "pool2: bad args");
  const int64_t items = N * (H / 2) * (W / 2) * (C / 8);
  if (items + (int64_t)132 * 8 * 256 < (int64_t(1) << 32))
    CGD_CUDA(launch_pdl(pool2_kernel<uint32_t>, dim3(ew_blocks(items)), dim3(256), 0, st, (const __half*)op.p[0], (__half*)op.p[1], (int)N, (int)H, (int)W,
                        (int)C, ldx, ldy, op.f[0]));
  else
    CGD_CUDA(launch_pdl(pool2_kernel<int64_t>, dim3(ew_blocks(items)), dim3(256), 0, st, (const __half*)op.p[0], (__half*)op.p[1], (int)N, (int)H, (int)W,
                        (int)C, ldx, ldy, op.f[0]));
  CGD_LAUNCH_CHECK();
  return 0;
}
int launch_up2(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], H = op.i[1], W = op.i[2], C = op.i[3], ldx = op.i[4], ldy = op.i[5];
  CGD_CHECK_ARG(N > 0 && H > 0 && W > 0 && C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0 && op.p[0] && op.p[1], "up2: bad args");
  const int64_t items = N * H * W * (C / 8);  // one thread per input vector
  if (items + (int64_t)132 * 8 * 256 < (int64_t(1) << 32))
    CGD_CUDA(launch_pdl(up2_kernel<uint32_t>, dim3(ew_blocks(items)), dim3(256), 0, st, (const __half*)op.p[0], (__half*)op.p[1], (int)N, (int)H, (int)W, (int)C,
                        ldx, ldy, op.f[0]));
  else
    CGD_CUDA(launch_pdl(up2_kernel<int64_t>, dim3(ew_blocks(items)), dim3(256), 0, st, (const __half*)op.p[0], (__half*)op.p[1], (int)N, (int)H, (int)W, (int)C,
                        ldx, ldy, op.f[0]));
  CGD_LAUNCH_CHECK();
  return 0;
}
int launch_add(const CgdOp& op, cudaStream_t st) {
  const int64_t rows = op.i[0], C = op.i[1];
  CGD_CHECK_ARG(rows > 0 && C % 8 == 0 && op.i[2] % 8 == 0 && op.i[3] % 8 == 0 && op.i[4] % 8 == 0 && op.p[0] && op.p[1] && op.p[2], "add: bad args");
  CGD_CUDA(launch_pdl(add_kernel, dim3(ew_blocks(rows * (C / 8))), dim3(256), 0, st, (const __half*)op.p[0], (const __half*)op.p[1], (__half*)op.p[2], rows, (int)C,
                                                       op.i[2], op.i[3], op.i[4]));
  CGD_LAUNCH_CHECK();
  return 0;
}
int launch_copy(const CgdOp& op, cudaStream_t st) {
  const int64_t rows = op.i[0], C = op.i[1];
  CGD_CHECK_ARG(rows > 0 && C % 8 == 0 && op.i[2] % 8 == 0 && op.i[3] % 8 == 0 && op.p[0] && op.p[1], "copy: bad args");
  CGD_CUDA(launch_pdl(copy_kernel, dim3(ew_blocks(rows * (C / 8))), dim3(256), 0, st, (const __half*)op.p[0], (__half*)op.p[1], rows, (int)C, op.i[2], op.i[3]));
  CGD_LAUNCH_CHECK();
  return 0;
}

// ---- layout conversion at the sampler boundary
// fp32 NCHW [N,C,HW] -> fp16 pixel-major [N*HW, ld], channels >= C zero-filled
// optional per-channel affine (C <= 3: the LPIPS ScalingLayer): value = (x - shift_c) * mul_c * scale
__global__ void nchw_to_pm_kernel(const float* __restrict__ src, __half* __restrict__ dst, int N, int C, int64_t HW, int64_t ld, float scale,
                                  float3 shift, float3 mul) {
  pdl_wait();
  pdl_launch_dependents();
  const int V = (int)(ld / 8);
  const int64_t total = (int64_t)N * HW * V;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int v = (int)(idx % V);
    const int64_t pix = idx / V;
    const int64_t n = pix / HW, p = pix % HW;
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = v * 8 + j;
      const float sh = c == 0 ? shift.x : (c == 1 ? shift.y : shift.z), mu = c == 0 ? mul.x : (c == 1 ? mul.y : mul.z);
      o[j] = c < C ? (src[((int64_t)n * C + c) * HW + p] - sh) * mu * scale : 0.f;
    }
    st8(dst + pix * ld + v * 8, pack8(o));
  }
}
// pixel-major (fp16 / fp32) -> fp32 NCHW, one thread per destination element (reads of a pixel's few channels hit one sector)
template <typename T>
__global__ void pm_to_nchw_kernel(const T* __restrict__ src, float* __restrict__ dst, int N, int C, int64_t HW, int64_t ld, float scale,
                                  int accumulate, float3 mul, const float* __restrict__ div) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t total = (int64_t)N * C * HW;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = idx % HW;
    const int64_t nc = idx / HW;
    const int c = (int)(nc % C);
    const int64_t n = nc / C;
    float v = (float)src[(n * HW + p) * ld + c] * scale * (c == 0 ? mul.x : (c == 1 ? mul.y : mul.z));
    if (div) v = v / div[n];
    dst[idx] = accumulate ? dst[idx] + v : v;
  }
}
int launch_nchw_to_pm(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], C = op.i[1], HW = op.i[2], ld = op.i[3];
  CGD_CHECK_ARG(N > 0 && C > 0 && HW > 0 && ld % 8 == 0 && C <= ld && op.p[0] && op.p[1], "nchw_to_pm: bad args");
  const bool aff = (op.flags & 4) != 0;  // f1..3 shift, f4..6 multiplier per channel
  CGD_CHECK_ARG(!aff || C <= 3, "nchw_to_pm: per-channel affine needs C <= 3");
  CGD_CUDA(launch_pdl(nchw_to_pm_kernel, dim3(ew_blocks(N * HW * (ld / 8))), dim3(256), 0, st, (const float*)op.p[0], (__half*)op.p[1], (int)N, (int)C, HW, ld, op.f[0],
                      aff ? make_float3(op.f[1], op.f[2], op.f[3]) : make_float3(0.f, 0.f, 0.f),
                      aff ? make_float3(op.f[4], op.f[5], op.f[6]) : make_float3(1.f, 1.f, 1.f)));
  CGD_LAUNCH_CHECK();
  return 0;
}
int launch_pm_to_nchw(const CgdOp& op, cudaStream_t st) {
  const int64_t N = op.i[0], C = op.i[1], HW = op.i[2], ld = op.i[3];
  CGD_CHECK_ARG(N > 0 && C > 0 && HW > 0 && C <= ld && op.p[0] && op.p[1], "pm_to_nchw: bad args");
  const int acc = (op.flags & 2) ? 1 : 0;
  CGD_CHECK_ARG(!(op.flags & 4) || C <= 3, "pm_to_nchw: per-channel scale needs C <= 3");
  const float3 mul = (op.flags & 4) ? make_float3(op.f[1], op.f[2], op.f[3]) : make_float3(1.f, 1.f, 1.f);  // per-channel multiplier
  // flags 8: image n divided by div[n] (p2, fp32 [N]; the per-image power-of-two scale of a seeded backward)
  CGD_CHECK_ARG(!(op.flags & 8) || (op.p[2] && ((uintptr_t)op.p[2] & 3) == 0), "pm_to_nchw: flags 8 needs a 4-byte aligned divisor vector p2");
  const float* div = (op.flags & 8) ? (const float*)op.p[2] : nullptr;
  if (op.flags & 1)
    CGD_CUDA(launch_pdl(pm_to_nchw_kernel<float>, dim3(ew_blocks(N * C * HW)), dim3(256), 0, st, (const float*)op.p[0], (float*)op.p[1], (int)N, (int)C, HW, ld, op.f[0], acc, mul, div));
  else
    CGD_CUDA(launch_pdl(pm_to_nchw_kernel<__half>, dim3(ew_blocks(N * C * HW)), dim3(256), 0, st, (const __half*)op.p[0], (float*)op.p[1], (int)N, (int)C, HW, ld, op.f[0], acc, mul, div));
  CGD_LAUNCH_CHECK();
  return 0;
}

// ---- timestep / class embeddings ([3P] guided_diffusion.nn.timestep_embedding, UNetModel.label_emb)
__global__ void timestep_emb_kernel(const float* __restrict__ t, float* __restrict__ out, int B, int dim, float tscale) {
  pdl_wait();
  pdl_launch_dependents();
  const int half = dim / 2;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * half) return;
  const int b = idx / half, i = idx % half;
  // fp32 like the reference: freqs = exp(-ln(10000) * i / half); args = t * freqs
  const float freq = expf(-9.210340371976184f * (float)i / (float)half);
  const float arg = t[b] * tscale * freq;
  out[(int64_t)b * dim + i] = cosf(arg);
  out[(int64_t)b * dim + half + i] = sinf(arg);
  if ((dim & 1) && i == 0) out[(int64_t)b * dim + dim - 1] = 0.f;
}
__global__ void label_add_kernel(float* __restrict__ emb, const float* __restrict__ table, const int64_t* __restrict__ y, int B, int D) {
  pdl_wait();
  pdl_launch_dependents();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * D) return;
  const int b = idx / D, d = idx % D;
  emb[idx] += table[y[b] * (int64_t)D + d];
}
int launch_timestep_emb(const CgdOp& op, cudaStream_t st) {
  const int64_t B = op.i[0], dim = op.i[1];
  CGD_CHECK_ARG(B > 0 && dim >= 2 && op.p[0] && op.p[1], "timestep_emb: bad args");
  CGD_CUDA(launch_pdl(timestep_emb_kernel, dim3((unsigned)ceil_div(B * (dim / 2), 128)), dim3(128), 0, st, (const float*)op.p[0], (float*)op.p[1], (int)B, (int)dim, op.f[0]));
  CGD_LAUNCH_CHECK();
  return 0;
}
int launch_label_add(const CgdOp& op, cudaStream_t st) {
  const int64_t B = op.i[0], D = op.i[1];
  CGD_CHECK_ARG(B > 0 && D > 0 && op.p[0] && op.p[1] && op.p[2], "label_add: bad args");
  CGD_CUDA(launch_pdl(label_add_kernel, dim3((unsigned)ceil_div(B * D, 256)), dim3(256), 0, st, (float*)op.p[0], (const float*)op.p[1], (const int64_t*)op.p[2], (int)B, (int)D));
  CGD_LAUNCH_CHECK();
  return 0;
}

// ---- QuickGELU ([3P] clip.model.QuickGELU): a = u * sigmoid(1.702 u); EXACT (QGELU_FWD flags 1, the OpenCLIP towers' nn.GELU):
// a = 0.5 u (1 + erf(u / sqrt 2)) = 0.5 u erfc(-u / sqrt 2) in fp32 from the fp16 u, rounded once to fp16
template <bool EXACT>
__global__ void qgelu_fwd_kernel(const __half* __restrict__ u, __half* __restrict__ a, int64_t nvec) {
  pdl_wait();
  pdl_launch_dependents();
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < nvec; idx += (int64_t)gridDim.x * blockDim.x) {
    float v[8];
    unpack8(ld8(u + idx * 8), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (EXACT) v[j] = 0.5f * v[j] * erfcf(v[j] * -0.70710678118654752f);  // Phi(u) = erfc(-u / sqrt 2) / 2: no cancellation for u << 0
      else v[j] = v[j] / (1.f + __expf(-1.702f * v[j]));
    }
    st8(a + idx * 8, pack8(v));
  }
}
__global__ void qgelu_bwd_kernel(const __half* __restrict__ da, const __half* __restrict__ u, __half* __restrict__ du, int64_t nvec) {
  pdl_wait();
  pdl_launch_dependents();
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < nvec; idx += (int64_t)gridDim.x * blockDim.x) {
    float v[8], d[8];
    unpack8(ld8(u + idx * 8), v);
    unpack8(ld8(da + idx * 8), d);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float s = 1.f / (1.f + __expf(-1.702f * v[j]));
      d[j] *= s * (1.f + 1.702f * v[j] * (1.f - s));
    }
    st8(du + idx * 8, pack8(d));
  }
}
int launch_qgelu_fwd(const CgdOp& op, cudaStream_t st) {
  const int64_t n = op.i[0];
  CGD_CHECK_ARG(n > 0 && n % 8 == 0 && op.p[0] && op.p[1], "qgelu: bad args");
  CGD_CHECK_ARG((op.flags & ~1) == 0, "qgelu: unknown flags %d (1 = exact GELU)", op.flags);
  if (op.flags & 1)
    CGD_CUDA(launch_pdl(qgelu_fwd_kernel<true>, dim3(ew_blocks(n / 8)), dim3(256), 0, st, (const __half*)op.p[0], (__half*)op.p[1], n / 8));
  else
    CGD_CUDA(launch_pdl(qgelu_fwd_kernel<false>, dim3(ew_blocks(n / 8)), dim3(256), 0, st, (const __half*)op.p[0], (__half*)op.p[1], n / 8));
  CGD_LAUNCH_CHECK();
  return 0;
}
int launch_qgelu_bwd(const CgdOp& op, cudaStream_t st) {
  const int64_t n = op.i[0];
  CGD_CHECK_ARG(n > 0 && n % 8 == 0 && op.p[0] && op.p[1] && op.p[2], "qgelu bwd: bad args");
  CGD_CUDA(launch_pdl(qgelu_bwd_kernel, dim3(ew_blocks(n / 8)), dim3(256), 0, st, (const __half*)op.p[0], (const __half*)op.p[1], (__half*)op.p[2], n / 8));
  CGD_LAUNCH_CHECK();
  return 0;
}

// ---- ViT token assembly ([3P] VisionTransformer.forward: cat(class_embedding, patches) + positional_embedding)
__global__ void vit_embed_kernel(__half* __restrict__ tok, const float* __restrict__ cls, const float* __restrict__ pos, int n, int T, int w) {
  pdl_wait();
  pdl_launch_dependents();
  const int V = w / 8;
  const int64_t total = (int64_t)n * T * V;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int v = (int)(idx % V);
    const int64_t row = idx / V;
    const int t = (int)(row % T);
    float a[8];
    if (t == 0) {
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] = cls[v * 8 + j];
      // the reference adds cls and pos in the model dtype; round cls to fp16 first like cat() of fp16 tensors does
      const half8 h = pack8(a);
      unpack8(h, a);
    } else {
      unpack8(ld8(tok + row * w + v * 8), a);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += pos[(int64_t)t * w + v * 8 + j];
    st8(tok + row * w + v * 8, pack8(a));
  }
}
int launch_vit_embed(const CgdOp& op, cudaStream_t st) {
  const int64_t n = op.i[0], T = op.i[1], w = op.i[2];
  CGD_CHECK_ARG(n > 0 && T > 0 && w % 8 == 0 && op.p[0] && op.p[1] && op.p[2], "vit_embed: bad args");
  CGD_CUDA(launch_pdl(vit_embed_kernel, dim3(ew_blocks(n * T * (w / 8))), dim3(256), 0, st, (__half*)op.p[0], (const float*)op.p[1], (const float*)op.p[2], (int)n, (int)T, (int)w));
  CGD_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------- CLIP ModifiedResNet AttentionPool2d token assembly
// y[n,0,:] = mean_t x[n,t,:] + pos[0,:] ; y[n,1+t,:] = x[n,t,:] + pos[1+t,:]  ([3P] clip/model.py AttentionPool2d.forward: cat of the mean
// token, then the positional embedding; the mean is rounded to fp16 before the add like the reference's fp16 tensors)
__global__ void attnpool_embed_fwd_kernel(const __half* __restrict__ x, const float* __restrict__ pos, __half* __restrict__ y, int n, int HW,
                                          int C, int64_t ldx) {
  pdl_wait();
  pdl_launch_dependents();
  const int V = C / 8;
  const int64_t total = (int64_t)n * (HW + 1) * V;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int v = (int)(idx % V);
    const int64_t row = idx / V;
    const int t = (int)(row % (HW + 1));
    const int64_t img = row / (HW + 1);
    const __half* xi = x + img * HW * ldx + v * 8;
    float a[8];
    if (t == 0) {
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] = 0.f;
      for (int u = 0; u < HW; ++u) {
        float f[8];
        unpack8(ld8(xi + (int64_t)u * ldx), f);
#pragma unroll
        for (int j = 0; j < 8; ++j) a[j] += f[j];
      }
      const float inv = 1.f / (float)HW;
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] *= inv;
      const half8 h = pack8(a);
      unpack8(h, a);
    } else {
      unpack8(ld8(xi + (int64_t)(t - 1) * ldx), a);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += pos[(int64_t)t * C + v * 8 + j];
    st8(y + row * C + v * 8, pack8(a));
  }
}
// dx[n,t,:] (=|+=) dy[n,1+t,:] + dy[n,0,:] / HW
__global__ void attnpool_embed_bwd_kernel(const __half* __restrict__ dy, __half* __restrict__ dx, int n, int HW, int C, int64_t ld_dx, int accumulate) {
  pdl_wait();
  pdl_launch_dependents();
  const int V = C / 8;
  const int64_t total = (int64_t)n * HW * V;
  const float inv = 1.f / (float)HW;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int v = (int)(idx % V);
    const int64_t row = idx / V;
    const int t = (int)(row % HW);
    const int64_t img = row / HW;
    float a[8], m[8];
    unpack8(ld8(dy + (img * (HW + 1) + 1 + t) * C + v * 8), a);
    unpack8(ld8(dy + (img * (HW + 1)) * C + v * 8), m);
    __half* o = dx + (img * HW + t) * ld_dx + v * 8;
    if (accumulate) {
      float c[8];
      unpack8(ld8(o), c);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] += c[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = fmaf(m[j], inv, a[j]);
    st8(o, pack8(a));
  }
}
int launch_attnpool_embed_fwd(const CgdOp& op, cudaStream_t st) {
  const int64_t n = op.i[0], HW = op.i[1], C = op.i[2], ldx = op.i[3];
  CGD_CHECK_ARG(n > 0 && HW > 0 && C % 8 == 0 && ldx % 8 == 0 && ldx >= C && op.p[0] && op.p[1] && op.p[2], "attnpool_embed_fwd: bad args");
  CGD_CUDA(launch_pdl(attnpool_embed_fwd_kernel, dim3(ew_blocks(n * (HW + 1) * (C / 8))), dim3(256), 0, st, (const __half*)op.p[0],
                      (const float*)op.p[1], (__half*)op.p[2], (int)n, (int)HW, (int)C, ldx));
  CGD_LAUNCH_CHECK();
  return 0;
}
int launch_attnpool_embed_bwd(const CgdOp& op, cudaStream_t st) {
  const int64_t n = op.i[0], HW = op.i[1], C = op.i[2], ld_dx = op.i[3];
  CGD_CHECK_ARG(n > 0 && HW > 0 && C % 8 == 0 && ld_dx % 8 == 0 && ld_dx >= C && op.p[0] && op.p[1], "attnpool_embed_bwd: bad args");
  CGD_CUDA(launch_pdl(attnpool_embed_bwd_kernel, dim3(ew_blocks(n * HW * (C / 8))), dim3(256), 0, st, (const __half*)op.p[0], (__half*)op.p[1], (int)n,
                      (int)HW, (int)C, ld_dx, (int)((op.flags & 2) ? 1 : 0)));
  CGD_LAUNCH_CHECK();
  return 0;
}

}  // namespace cgd
