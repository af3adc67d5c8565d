// augs.cu -- MakeCutouts with use_augs=True (cgd/modules.py:12-24, 60-64): the torchvision pipeline
//     RandomHorizontalFlip -> +noise -> RandomAffine(15 deg, translate .1; NEAREST, fill 0) -> +noise
//     -> RandomPerspective(.4, p = .7; BILINEAR, fill 0) -> +noise -> RandomGrayscale(.15) -> +noise -> adaptive_avg_pool2d
// applied to every crop, + CLIP_NORMALIZE (cgd/clip_util.py:45), as ONE gather kernel forward and ONE scatter kernel backward.
// The random decisions and geometric parameters are drawn on the host in torchvision's order (clip_guided_diffusion_b200/augs.py,
// 20 floats per cutout); the four noise fields come from torch.randn in the reference's shapes.  Everything between the crop and the
// pooled cutout is linear in the image, so the input gradient is the transposed gather (fp32 atomics: several cutouts and several
// taps hit the same source pixel; the reference's grid_sample backward on CUDA accumulates with atomics as well).
//
// Coordinate conventions are torchvision's (transforms/_functional_tensor.py): _gen_affine_grid / _perspective_grid build a
// normalised grid that grid_sample(align_corners=False) un-normalises; composed, a destination pixel (j, i) of a w x h image samples
//     affine:       sx = m0*bx + m1*by + m2 + (w-1)/2,  sy = m3*bx + m4*by + m5 + (h-1)/2,  bx = j - w/2 + .5, by = i - h/2 + .5, NEAREST
//     perspective:  sx = (c0*x + c1*y + c2) / (c6*x + c7*y + 1) - .5, sy = (c3*x + c4*y + c5) / (...) - .5, x = j + .5, y = i + .5, BILINEAR
// with zero padding, and with `fill` given (torchvision passes [0, 0, 0]) the bilinear result is additionally multiplied by the
// interpolated all-ones mask (_apply_grid_transform: img * mask + (1 - mask) * fill).
#include <algorithm>

#include "common.cuh"
#include "ops.cuh"
#include "pdl.cuh"

namespace cgd {

constexpr int AUG_NP = 20;  // floats per cutout, layout in augs.py

__device__ __forceinline__ void aug_pool_bin(int o, int S, int cs, int& s, int& e) {
  s = (int)(((unsigned)o * (unsigned)S) / (unsigned)cs);
  e = (int)((((unsigned)(o + 1)) * (unsigned)S + (unsigned)cs - 1u) / (unsigned)cs);
}

struct AugGeom {
  const float* prm;
  int Sx, Sy, offx, offy;
  bool flip, persp, gray;
};

// nearest source pixel of destination (tx, ty) under the inverse affine matrix; false = outside (fill 0)
__device__ __forceinline__ bool aug_affine_src(const AugGeom& g, int tx, int ty, int& sx, int& sy) {
  const float w = (float)g.Sx, h = (float)g.Sy;
  const float bx = (float)tx - w * 0.5f + 0.5f, by = (float)ty - h * 0.5f + 0.5f;
  // same operation order as torchvision: theta / (0.5 * size), grid = base . theta, then ((grid + 1) * size - 1) / 2
  const float gx = bx * (g.prm[1] / (0.5f * w)) + by * (g.prm[2] / (0.5f * w)) + g.prm[3] / (0.5f * w);
  const float gy = bx * (g.prm[4] / (0.5f * h)) + by * (g.prm[5] / (0.5f * h)) + g.prm[6] / (0.5f * h);
  const float fx = ((gx + 1.f) * w - 1.f) * 0.5f, fy = ((gy + 1.f) * h - 1.f) * 0.5f;
  sx = (int)nearbyintf(fx);  // grid_sample 'nearest' rounds half to even
  sy = (int)nearbyintf(fy);
  return sx >= 0 && sx < g.Sx && sy >= 0 && sy < g.Sy;
}

// bilinear taps of destination (xx, yy) under the perspective coefficients: base tap (x0, y0), weights of the four corners
__device__ __forceinline__ void aug_persp_taps(const AugGeom& g, int xx, int yy, int& x0, int& y0, float& wx1, float& wy1) {
  const float* c = g.prm + 8;
  const float w = (float)g.Sx, h = (float)g.Sy;
  const float x = (float)xx + 0.5f, y = (float)yy + 0.5f;
  const float den = c[6] * x + c[7] * y + 1.f;
  const float gx = (x * (c[0] / (0.5f * w)) + y * (c[1] / (0.5f * w)) + c[2] / (0.5f * w)) / den - 1.f;
  const float gy = (x * (c[3] / (0.5f * h)) + y * (c[4] / (0.5f * h)) + c[5] / (0.5f * h)) / den - 1.f;
  const float fx = ((gx + 1.f) * w - 1.f) * 0.5f, fy = ((gy + 1.f) * h - 1.f) * 0.5f;
  const float flx = floorf(fx), fly = floorf(fy);
  x0 = (int)flx;
  y0 = (int)fly;
  wx1 = fx - flx;
  wy1 = fy - fly;
}

__device__ __forceinline__ AugGeom aug_geom(const float* params, const int* coords, int k, int H, int W) {
  AugGeom gm;
  gm.prm = params + (int64_t)k * AUG_NP;
  gm.offx = coords[k * 3 + 0];
  gm.offy = coords[k * 3 + 1];
  const int S = coords[k * 3 + 2];
  gm.Sy = min(S, H - gm.offy);
  gm.Sx = min(S, W - gm.offx);
  gm.flip = gm.prm[0] != 0.f;
  gm.persp = gm.prm[7] != 0.f;
  gm.gray = gm.prm[16] != 0.f;
  return gm;
}

// the noise fields of one (cutout, image): plane c of stage s at nz + s * nstage + c * nplane, row stride Smax; nz null = no noise
struct AugNoise {
  const float* nz;
  int64_t nstage, nplane;
  int Smax;
};

// I4[c](tx, ty): the affine-transformed (flipped, noised) crop plus the second noise field; (tx, ty) inside the frame.  xb = image b
__device__ __forceinline__ void aug_i4(const AugGeom& gm, const float* xb, int64_t HW, int W, const AugNoise& n, int tx, int ty, float v[3]) {
  int sx, sy;
  const bool in = aug_affine_src(gm, tx, ty, sx, sy);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float a = 0.f;
    if (in) {
      const int cx = gm.flip ? gm.Sx - 1 - sx : sx;
      a = (xb[c * HW + (int64_t)(gm.offy + sy) * W + gm.offx + cx] + 1.f) * 0.5f;
      if (n.nz) a += n.nz[c * n.nplane + (int64_t)sy * n.Smax + sx];
    }
    if (n.nz) a += n.nz[n.nstage + c * n.nplane + (int64_t)ty * n.Smax + tx];
    v[c] = a;
  }
}

// I8[c](xx, yy): the whole pipeline at crop pixel (xx, yy) -- perspective, third noise field, grayscale, fourth noise field
__device__ __forceinline__ void aug_pixel(const AugGeom& gm, const float* xb, int64_t HW, int W, const AugNoise& n, int xx, int yy, float v[3]) {
  if (gm.persp) {
    int x0, y0;
    float wx1, wy1;
    aug_persp_taps(gm, xx, yy, x0, y0, wx1, wy1);
    float s[3] = {0.f, 0.f, 0.f}, m = 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int tx = x0 + (t & 1), ty = y0 + (t >> 1);
      if (tx < 0 || tx >= gm.Sx || ty < 0 || ty >= gm.Sy) continue;
      const float wt = ((t & 1) ? wx1 : 1.f - wx1) * ((t >> 1) ? wy1 : 1.f - wy1);
      float u[3];
      aug_i4(gm, xb, HW, W, n, tx, ty, u);
      s[0] += wt * u[0];
      s[1] += wt * u[1];
      s[2] += wt * u[2];
      m += wt;
    }
    v[0] = s[0] * m;
    v[1] = s[1] * m;
    v[2] = s[2] * m;
  } else {
    aug_i4(gm, xb, HW, W, n, xx, yy, v);
  }
  if (n.nz) {
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] += n.nz[2 * n.nstage + c * n.nplane + (int64_t)yy * n.Smax + xx];
  }
  if (gm.gray) {
    const float l = 0.2989f * v[0] + 0.587f * v[1] + 0.114f * v[2];
    v[0] = v[1] = v[2] = l;
  }
  if (n.nz) {
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] += n.nz[3 * n.nstage + c * n.nplane + (int64_t)yy * n.Smax + xx];
  }
}

__device__ __forceinline__ AugNoise aug_noise(const float* noise, int k, int b, int B, int Smax) {
  const int64_t nplane = (int64_t)Smax * Smax;
  return AugNoise{noise ? noise + (((int64_t)k * 4) * B + b) * 3 * nplane : nullptr, (int64_t)B * 3 * nplane, nplane, Smax};
}

// ---------------------------------------------------------------- forward: one thread per (cutout, image, output pixel), 3 channels
// x [B,3,H,W] in [-1, 1]; noise [cutn][4][B][3][Smax][Smax] (already scaled by 0.01) or null; out in ViT patch order like cutouts_fwd
__global__ void cutouts_aug_fwd_kernel(const float* __restrict__ x, const int* __restrict__ coords, const float* __restrict__ params,
                                       const float* __restrict__ noise, __half* __restrict__ out, int B, int H, int W, int cutn, int cs, int P,
                                       int Kpad, int Smax, float3 mean, float3 stdv) {
  pdl_wait();
  pdl_launch_dependents();
  const int g = cs / P, G2 = g * g, PP = P * P;
  const int64_t total = (int64_t)cutn * B * cs * cs;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int ox = (int)(idx % cs);
    int64_t r = idx / cs;
    const int oy = (int)(r % cs);
    r /= cs;
    const int b = (int)(r % B), k = (int)(r / B);
    const AugGeom gm = aug_geom(params, coords, k, H, W);
    const float* xb = x + (int64_t)b * 3 * H * W;
    const int64_t HW = (int64_t)H * W;
    const AugNoise nz = aug_noise(noise, k, b, B, Smax);
    int ys, ye, xs, xe;
    aug_pool_bin(oy, gm.Sy, cs, ys, ye);
    aug_pool_bin(ox, gm.Sx, cs, xs, xe);
    float acc[3] = {0.f, 0.f, 0.f};
    for (int yy = ys; yy < ye; ++yy)
      for (int xx = xs; xx < xe; ++xx) {
        float v[3];
        aug_pixel(gm, xb, HW, W, nz, xx, yy, v);
        acc[0] += v[0];
        acc[1] += v[1];
        acc[2] += v[2];
      }
    const float inv = 1.f / (float)((ye - ys) * (xe - xs));
    const int patch = (oy / P) * g + (ox / P), ky = oy % P, kx = ox % P;
    __half* o = out + (((int64_t)k * B + b) * G2 + patch) * Kpad;
    o[0 * PP + ky * P + kx] = __float2half_rn((acc[0] * inv - mean.x) / stdv.x);
    o[1 * PP + ky * P + kx] = __float2half_rn((acc[1] * inv - mean.y) / stdv.y);
    o[2 * PP + ky * P + kx] = __float2half_rn((acc[2] * inv - mean.z) / stdv.z);
    if (ky == 0 && kx == 0)
      for (int kk = 3 * PP; kk < Kpad; ++kk) o[kk] = __float2half_rn(0.f);
  }
}

// flags 1: the augmented crop itself, fp32 [cutn][B][3][Smax][Smax] in [0, 1] (top-left Sy x Sx of every plane written), for the
// ResizeRight cutouts (CUTOUTS_RR_FWD flags 2) to resample
__global__ void cutouts_aug_crop_kernel(const float* __restrict__ x, const int* __restrict__ coords, const float* __restrict__ params,
                                        const float* __restrict__ noise, float* __restrict__ crop, int B, int H, int W, int cutn, int Smax) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t nplane = (int64_t)Smax * Smax, total = (int64_t)cutn * B * nplane;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int xx = (int)(idx % Smax);
    int64_t r = idx / Smax;
    const int yy = (int)(r % Smax);
    r /= Smax;
    const int b = (int)(r % B), k = (int)(r / B);
    const AugGeom gm = aug_geom(params, coords, k, H, W);
    if (xx >= gm.Sx || yy >= gm.Sy) continue;
    float v[3];
    aug_pixel(gm, x + (int64_t)b * 3 * H * W, (int64_t)H * W, W, aug_noise(noise, k, b, B, Smax), xx, yy, v);
    float* o = crop + ((int64_t)k * B + b) * 3 * nplane + (int64_t)yy * Smax + xx;
    o[0] = v[0];
    o[nplane] = v[1];
    o[2 * nplane] = v[2];
  }
}

// ---------------------------------------------------------------- backward: the transposed gather, scattered with fp32 atomics
// d I8 = d of crop pixel (xx, yy) (already through grayscale) -> dx of image b (db) through perspective, nearest affine, flip, crop
__device__ __forceinline__ void aug_scatter_pixel(const AugGeom& gm, float* db, int64_t HW, int W, int xx, int yy, const float d[3]) {
  auto scatter = [&](int tx, int ty, float wgt) {  // d I4(tx, ty) += wgt * d  ->  through the nearest affine sample, flip, crop
    int sx, sy;
    if (!aug_affine_src(gm, tx, ty, sx, sy)) return;
    const int cx = gm.flip ? gm.Sx - 1 - sx : sx;
    float* q = db + (int64_t)(gm.offy + sy) * W + gm.offx + cx;
    atomicAdd(q, wgt * d[0]);
    atomicAdd(q + HW, wgt * d[1]);
    atomicAdd(q + 2 * HW, wgt * d[2]);
  };
  if (gm.persp) {
    int x0, y0;
    float wx1, wy1;
    aug_persp_taps(gm, xx, yy, x0, y0, wx1, wy1);
    float wts[4], m = 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int tx = x0 + (t & 1), ty = y0 + (t >> 1);
      const bool in = tx >= 0 && tx < gm.Sx && ty >= 0 && ty < gm.Sy;
      wts[t] = in ? ((t & 1) ? wx1 : 1.f - wx1) * ((t >> 1) ? wy1 : 1.f - wy1) : 0.f;
      m += wts[t];
    }
#pragma unroll
    for (int t = 0; t < 4; ++t)
      if (wts[t] != 0.f) scatter(x0 + (t & 1), y0 + (t >> 1), wts[t] * m);  // I5 = (sum_t w_t I4[t]) * mask, mask = sum of in-bounds w
  } else {
    scatter(xx, yy, 1.f);
  }
}

__device__ __forceinline__ void aug_gray_bwd(const AugGeom& gm, float d[3]) {
  if (gm.gray) {  // I7[c] = L(I6) for every c  =>  d I6[c'] = weight[c'] * sum_c d I7[c]
    const float t = d[0] + d[1] + d[2];
    d[0] = 0.2989f * t;
    d[1] = 0.587f * t;
    d[2] = 0.114f * t;
  }
}

// dx must be zero on entry (CGD_OP_FILL before this op); dx += d loss / d x_in of the CLIP path.  InT = float (flags 4): fp32 d cutouts
// [cutn*B, 3, cs, cs] of the stand-alone MakeCutouts backward (the patch layout with P = cs, Kpad = 3 cs^2)
__device__ __forceinline__ float aug_in(const __half* p) { return __half2float(*p); }
__device__ __forceinline__ float aug_in(const float* p) { return *p; }
template <typename InT>
__global__ void cutouts_aug_bwd_kernel(const InT* __restrict__ dpatch, const int* __restrict__ coords, const float* __restrict__ params,
                                       float* __restrict__ dx, int B, int H, int W, int cutn, int cs, int P, int Kpad, float3 stdv, float scale) {
  pdl_wait();
  pdl_launch_dependents();
  const int g = cs / P, G2 = g * g, PP = P * P;
  const int64_t total = (int64_t)cutn * B * cs * cs;
  const int64_t HW = (int64_t)H * W;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int ox = (int)(idx % cs);
    int64_t r = idx / cs;
    const int oy = (int)(r % cs);
    r /= cs;
    const int b = (int)(r % B), k = (int)(r / B);
    const AugGeom gm = aug_geom(params, coords, k, H, W);
    int ys, ye, xs, xe;
    aug_pool_bin(oy, gm.Sy, cs, ys, ye);
    aug_pool_bin(ox, gm.Sx, cs, xs, xe);
    const int patch = (oy / P) * g + (ox / P), ky = oy % P, kx = ox % P;
    const InT* dp = dpatch + (((int64_t)k * B + b) * G2 + patch) * Kpad + ky * P + kx;
    // d / d I8[c] of every pixel of the bin: pooled mean, CLIP normalisation, (x + 1) / 2, the tower's gradient scale
    const float inv = 0.5f * scale / (float)((ye - ys) * (xe - xs));
    float d[3] = {aug_in(dp) * inv / stdv.x, aug_in(dp + PP) * inv / stdv.y, aug_in(dp + 2 * PP) * inv / stdv.z};
    aug_gray_bwd(gm, d);
    if (d[0] == 0.f && d[1] == 0.f && d[2] == 0.f) continue;
    float* db = dx + (int64_t)b * 3 * HW;
    for (int yy = ys; yy < ye; ++yy)
      for (int xx = xs; xx < xe; ++xx) aug_scatter_pixel(gm, db, HW, W, xx, yy, d);
  }
}

// flags 1: d crop fp32 [cutn][B][3][Smax][Smax] (what CUTOUTS_RR_BWD flags 2 stores: d / d I8) -> dx, one thread per crop pixel
__global__ void cutouts_aug_crop_bwd_kernel(const float* __restrict__ dcrop, const int* __restrict__ coords, const float* __restrict__ params,
                                            float* __restrict__ dx, int B, int H, int W, int cutn, int Smax, float scale) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t nplane = (int64_t)Smax * Smax, total = (int64_t)cutn * B * nplane, HW = (int64_t)H * W;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int xx = (int)(idx % Smax);
    int64_t r = idx / Smax;
    const int yy = (int)(r % Smax);
    r /= Smax;
    const int b = (int)(r % B), k = (int)(r / B);
    const AugGeom gm = aug_geom(params, coords, k, H, W);
    if (xx >= gm.Sx || yy >= gm.Sy) continue;
    const float* q = dcrop + ((int64_t)k * B + b) * 3 * nplane + (int64_t)yy * Smax + xx;
    const float s = 0.5f * scale;  // (x + 1) / 2 and the gradient scale
    float d[3] = {q[0] * s, q[nplane] * s, q[2 * nplane] * s};
    aug_gray_bwd(gm, d);
    if (d[0] == 0.f && d[1] == 0.f && d[2] == 0.f) continue;
    aug_scatter_pixel(gm, dx + (int64_t)b * 3 * HW, HW, W, xx, yy, d);
  }
}

static inline int aug_blocks(int64_t items) {
  int64_t b = ceil_div(items, 256);
  return (int)std::max<int64_t>(1, std::min<int64_t>(b, 132 * 16));
}

// op tables: include/cgd_b200.h CGD_OP_CUTOUTS_AUG_FWD / _BWD
int launch_cutouts_aug_fwd(const CgdOp& op, cudaStream_t st) {
  const int64_t B = op.i[0], H = op.i[1], W = op.i[2], cutn = op.i[3], cs = op.i[4], P = op.i[5], Kpad = op.i[6], Smax = op.i[7];
  CGD_CHECK_ARG(B > 0 && H > 0 && W > 0 && cutn > 0 && cs > 0 && P > 0 && cs % P == 0 && Kpad >= 3 * P * P && Smax >= std::min(H, W),
                "cutouts_aug_fwd: bad dims");
  CGD_CHECK_ARG(op.p[0] && op.p[1] && op.p[2] && op.p[3], "cutouts_aug_fwd: null pointer (x, coords, patches, params)");
  CGD_CHECK_ARG(op.flags == 0 || op.flags == 1, "cutouts_aug_fwd: flags must be 0 (pooled patches) or 1 (augmented crops), got %d", op.flags);
  if (op.flags & 1) {
    CGD_CHECK_ARG(Smax <= 16384, "cutouts_aug_fwd: Smax <= 16384");
    CGD_CUDA(launch_pdl(cutouts_aug_crop_kernel, dim3(aug_blocks(cutn * B * Smax * Smax)), dim3(256), 0, st, (const float*)op.p[0],
                        (const int*)op.p[1], (const float*)op.p[3], (const float*)op.p[4], (float*)op.p[2], (int)B, (int)H, (int)W, (int)cutn,
                        (int)Smax));
  } else {
    CGD_CUDA(launch_pdl(cutouts_aug_fwd_kernel, dim3(aug_blocks(cutn * B * cs * cs)), dim3(256), 0, st, (const float*)op.p[0], (const int*)op.p[1],
                        (const float*)op.p[3], (const float*)op.p[4], (__half*)op.p[2], (int)B, (int)H, (int)W, (int)cutn, (int)cs, (int)P, (int)Kpad,
                        (int)Smax, make_float3(op.f[0], op.f[1], op.f[2]), make_float3(op.f[3], op.f[4], op.f[5])));
  }
  CGD_LAUNCH_CHECK();
  return 0;
}

int launch_cutouts_aug_bwd(const CgdOp& op, cudaStream_t st) {
  const int64_t B = op.i[0], H = op.i[1], W = op.i[2], cutn = op.i[3], cs = op.i[4], P = op.i[5], Kpad = op.i[6];
  CGD_CHECK_ARG(B > 0 && H > 0 && W > 0 && cutn > 0 && cs > 0 && P > 0 && cs % P == 0 && Kpad >= 3 * P * P, "cutouts_aug_bwd: bad dims");
  CGD_CHECK_ARG(op.p[0] && op.p[1] && op.p[2] && op.p[3], "cutouts_aug_bwd: null pointer (d_patches, coords, dx, params)");
  CGD_CHECK_ARG(op.flags == 0 || op.flags == 4 || op.flags == 1,
                "cutouts_aug_bwd: flags must be 0 (fp16 d patches), 4 (fp32 d cutouts) or 1 (fp32 d crops), got %d", op.flags);
  if (op.flags & 1) {
    const int64_t Smax = op.i[7];
    CGD_CHECK_ARG(Smax >= std::min(H, W) && Smax <= 16384, "cutouts_aug_bwd: flags 1 needs i7 Smax >= min(H, W)");
    CGD_CUDA(launch_pdl(cutouts_aug_crop_bwd_kernel, dim3(aug_blocks(cutn * B * Smax * Smax)), dim3(256), 0, st, (const float*)op.p[0],
                        (const int*)op.p[1], (const float*)op.p[3], (float*)op.p[2], (int)B, (int)H, (int)W, (int)cutn, (int)Smax, op.f[6]));
  } else if (op.flags & 4) {
    CGD_CHECK_ARG(P == cs && Kpad == 3 * cs * cs,
                  "cutouts_aug_bwd: flags 4 reads fp32 d cutouts [cutn*B, 3, cs, cs]: patch must equal cut_size and Kpad 3 * cut_size^2");
    CGD_CUDA(launch_pdl(cutouts_aug_bwd_kernel<float>, dim3(aug_blocks(cutn * B * cs * cs)), dim3(256), 0, st, (const float*)op.p[0],
                        (const int*)op.p[1], (const float*)op.p[3], (float*)op.p[2], (int)B, (int)H, (int)W, (int)cutn, (int)cs, (int)P, (int)Kpad,
                        make_float3(op.f[3], op.f[4], op.f[5]), op.f[6]));
  } else {
    CGD_CUDA(launch_pdl(cutouts_aug_bwd_kernel<__half>, dim3(aug_blocks(cutn * B * cs * cs)), dim3(256), 0, st, (const __half*)op.p[0],
                        (const int*)op.p[1], (const float*)op.p[3], (float*)op.p[2], (int)B, (int)H, (int)W, (int)cutn, (int)cs, (int)P, (int)Kpad,
                        make_float3(op.f[3], op.f[4], op.f[5]), op.f[6]));
  }
  CGD_LAUNCH_CHECK();
  return 0;
}

}  // namespace cgd
