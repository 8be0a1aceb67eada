// Small kernels around the cost volume: camera constants, source repack, sampler, Gaussian update.
#include "common.cuh"
#include "launchers.h"
#include "gaussian_common.cuh"
#include "upsample_common.cuh"

namespace magnet {

// homography.py:98-102 — a = K t, A = K R, one thread per (b, v).  fp32, products accumulated in
// index order (the reference uses a 3x3 fp32 matmul; any order differs by <= 1 ulp).
__global__ void pack_cameras_kernel(const float* __restrict__ intM, const float* __restrict__ R, int64_t r_sb,
                                    int64_t r_sv, int64_t r_si, int64_t r_sj, const float* __restrict__ t,
                                    int64_t t_sb, int64_t t_sv, int64_t t_si,
                                    const int32_t* __restrict__ is_valid, int B, int V,
                                    magnet_camera* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * V) return;
  const int b = idx / V, v = idx % V;
  const float* K = intM + (size_t)b * 9;
  const float* Rp = R + b * r_sb + v * r_sv;
  const float* tp = t + b * t_sb + v * t_sv;
  magnet_camera c;
  c.valid = (is_valid[idx] == 1) ? 1.0f : 0.0f;
  const float t0 = tp[0], t1 = tp[t_si], t2 = tp[2 * t_si];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float k0 = K[i * 3 + 0], k1 = K[i * 3 + 1], k2 = K[i * 3 + 2];
    c.a[i] = __fmaf_rn(k2, t2, __fmaf_rn(k1, t1, __fmul_rn(k0, t0)));
#pragma unroll
    for (int j = 0; j < 3; ++j)
      c.A[i * 3 + j] = __fmaf_rn(k2, Rp[2 * r_si + j * r_sj],
                                 __fmaf_rn(k1, Rp[1 * r_si + j * r_sj], __fmul_rn(k0, Rp[0 * r_si + j * r_sj])));
  }
  c.pad[0] = c.pad[1] = c.pad[2] = 0.0f;
  out[idx] = c;
}

// (N, C, H, W) -> TILED32 (N, H, XB, C/4, 32, 4), XB = ceil(W/32).  One thread per (n, y, xb, c4, xi):
// 4 coalesced 4-byte reads (stride HW) along x, one coalesced 16-byte write; padding pixels get zeros.
__global__ void repack_tiled32_kernel(const float* __restrict__ src, float4* __restrict__ dst, int C4, int H,
                                      int W, int XB) {
  const int xi = threadIdx.x, c4 = threadIdx.y + blockIdx.z % ((C4 + 3) / 4) * 4;
  const int xb = blockIdx.x, y = blockIdx.y;
  const size_t img = blockIdx.z / ((C4 + 3) / 4);
  if (c4 >= C4) return;
  const int x = xb * 32 + xi;
  const size_t HW = (size_t)H * W;
  float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
  if (x < W) {
    const float* s = src + (img * C4 * 4 + (size_t)c4 * 4) * HW + (size_t)y * W + x;
    o.x = s[0];
    o.y = s[HW];
    o.z = s[2 * HW];
    o.w = s[3 * HW];
  }
  dst[(((img * H + y) * XB + xb) * C4 + c4) * 32 + xi] = o;
}

struct KParams {
  float k[MAGNET_MAX_PLANES];
};

// MAGNET.py:154-156
__global__ void sample_depths_kernel(const float* __restrict__ gmm, const __grid_constant__ KParams kp, int D,
                                     int HW, float* __restrict__ dvol) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= HW) return;
  const size_t b = blockIdx.y;
  const float mu = gmm[(b * 2 + 0) * HW + n], sg = gmm[(b * 2 + 1) * HW + n];
  float* o = dvol + b * D * HW + n;
  for (int j = 0; j < D; ++j) o[(size_t)j * HW] = __fadd_rn(mu, __fmul_rn(sg, kp.k[j]));
}

// MAGNET.py:60,65-69 (gaussian_update, gaussian_common.cuh)
__global__ void gaussian_update_fwd_kernel(const float* __restrict__ dout, const float* __restrict__ gmm0,
                                           int HW, float* __restrict__ out) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= HW) return;
  const size_t b = blockIdx.y;
  const float mu1 = dout[(b * 2 + 0) * HW + n], s1 = dout[(b * 2 + 1) * HW + n];
  const float mu0 = gmm0[(b * 2 + 0) * HW + n], s0 = gmm0[(b * 2 + 1) * HW + n];
  float mu, sg;
  gaussian_update(mu1, s1, mu0, s0, mu, sg);
  out[(b * 2 + 0) * HW + n] = mu;
  out[(b * 2 + 1) * HW + n] = sg;
}

__global__ void gaussian_update_bwd_kernel(const float* __restrict__ gout, const float* __restrict__ dout,
                                           const float* __restrict__ gmm0, int HW, float* __restrict__ gin) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= HW) return;
  const size_t b = blockIdx.y;
  const float s1 = dout[(b * 2 + 1) * HW + n];
  const float s0 = gmm0[(b * 2 + 1) * HW + n];
  const float g_mu = gout[(b * 2 + 0) * HW + n], g_sg = gout[(b * 2 + 1) * HW + n];
  float d_mu1, d_s1;
  gaussian_update_bwd(g_mu, g_sg, s1, s0, d_mu1, d_s1);
  gin[(b * 2 + 0) * HW + n] = d_mu1;
  gin[(b * 2 + 1) * HW + n] = d_s1;
}

// Learned convex upsampling (upsample_depth_via_mask, MAGNET.py:15-27) without the (B,C,9,k,k,H,W) temporaries.
// One thread per output pixel (b, Y = y*k+ky, X = x*k+kx), all channels: softmax over the 9 mask logits
// mask[b, (i*k+ky)*k+kx, y, x], weighted sum of the zero-padded 3x3 neighbourhood of depth[b, c, y, x].
template <int CH>
__global__ void convex_upsample_fwd_kernel(const float* __restrict__ depth, const float* __restrict__ mask, int H,
                                           int W, int k, float* __restrict__ out) {
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y;
  const size_t b = blockIdx.z;
  if (X >= W * k) return;
  const int x = X / k, kx = X % k, y = Y / k, ky = Y % k;
  const size_t HW = (size_t)H * W;
  const float* mp = mask + (b * 9 * k * k + (size_t)ky * k + kx) * HW + (size_t)y * W + x;
  float w[9], m = -INFINITY;
#pragma unroll
  for (int i = 0; i < 9; ++i) { w[i] = mp[(size_t)i * k * k * HW]; m = fmaxf(m, w[i]); }
  float s = 0.0f;
#pragma unroll
  for (int i = 0; i < 9; ++i) { w[i] = expf(w[i] - m); s += w[i]; }
  const float inv = 1.0f / s;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const float* dp = depth + (b * CH + c) * HW;
    float acc = 0.0f;
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      const int yy = y + i / 3 - 1, xx = x + i % 3 - 1;
      const float v = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? dp[(size_t)yy * W + xx] : 0.0f;
      acc = __fmaf_rn(w[i] * inv, v, acc);
    }
    out[((b * CH + c) * H * k + Y) * (size_t)(W * k) + X] = acc;
  }
}

// Backward of the above w.r.t. the mask logits (softmax backward, written) and the low-resolution map
// (scatter-add with red.add into grad_depth, which the caller zeroes).
template <int CH>
__global__ void convex_upsample_bwd_kernel(const float* __restrict__ gout, const float* __restrict__ depth,
                                           const float* __restrict__ mask, int H, int W, int k,
                                           float* __restrict__ gdepth, float* __restrict__ gmask) {
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y;
  const size_t b = blockIdx.z;
  if (X >= W * k) return;
  const int x = X / k, kx = X % k, y = Y / k, ky = Y % k;
  const size_t HW = (size_t)H * W;
  const size_t moff = (b * 9 * k * k + (size_t)ky * k + kx) * HW + (size_t)y * W + x;
  float w[9], m = -INFINITY;
#pragma unroll
  for (int i = 0; i < 9; ++i) { w[i] = mask[moff + (size_t)i * k * k * HW]; m = fmaxf(m, w[i]); }
  float s = 0.0f;
#pragma unroll
  for (int i = 0; i < 9; ++i) { w[i] = expf(w[i] - m); s += w[i]; }
  const float inv = 1.0f / s;
  float t[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) { w[i] *= inv; t[i] = 0.0f; }
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const float g = gout[((b * CH + c) * H * k + Y) * (size_t)(W * k) + X];
    const float* dp = depth + (b * CH + c) * HW;
    float* gd = gdepth + (b * CH + c) * HW;
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      const int yy = y + i / 3 - 1, xx = x + i % 3 - 1;
      if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
        t[i] = __fmaf_rn(g, dp[(size_t)yy * W + xx], t[i]);
        atomicAdd(gd + (size_t)yy * W + xx, g * w[i]);
      }
    }
  }
  float dot = 0.0f;
#pragma unroll
  for (int i = 0; i < 9; ++i) dot = __fmaf_rn(w[i], t[i], dot);
#pragma unroll
  for (int i = 0; i < 9; ++i) gmask[moff + (size_t)i * k * k * HW] = w[i] * (t[i] - dot);
}

// SURVEY §8 f-4 — caller-side camera prep on the device.
// utils/utils.py:72-98 (data_preprocess): nghbr_pose = ext_nghbr * inv(ext_ref); a view is invalid when either
// extrinsic or the product contains a NaN (then its pose stays zero).  One thread per (b, v); the 4x4 inverse is
// Gauss-Jordan with partial pivoting in fp32 (the reference: LAPACK sgetri on the fp32 matrix).
__global__ void relative_poses_kernel(const float* __restrict__ ext_ref, const float* __restrict__ ext_nghbr, int B,
                                      int V, float* __restrict__ poses, int32_t* __restrict__ valid) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * V) return;
  const int b = idx / V, v = idx % V;
  float a[4][8];
  bool nan_ref = false, nan_n = false;
  const float* R = ext_ref + (size_t)b * 16;
  const float* N = ext_nghbr + ((size_t)v * B + b) * 16;           // list over views of (B,4,4), view-major
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      a[i][j] = R[i * 4 + j];
      a[i][4 + j] = i == j ? 1.0f : 0.0f;
      nan_ref |= isnan(R[i * 4 + j]);
      nan_n |= isnan(N[i * 4 + j]);
    }
  for (int c = 0; c < 4; ++c) {
    int piv = c;
    for (int r = c + 1; r < 4; ++r)
      if (fabsf(a[r][c]) > fabsf(a[piv][c])) piv = r;
    for (int j = 0; j < 8; ++j) { const float t = a[c][j]; a[c][j] = a[piv][j]; a[piv][j] = t; }
    const float inv = 1.0f / a[c][c];
    for (int j = 0; j < 8; ++j) a[c][j] *= inv;
    for (int r = 0; r < 4; ++r)
      if (r != c) {
        const float f = a[r][c];
        for (int j = 0; j < 8; ++j) a[r][j] = __fmaf_rn(-f, a[c][j], a[r][j]);
      }
  }
  float out[16];
  bool nan_p = false;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      float acc = 0.0f;
      for (int k = 0; k < 4; ++k) acc = __fmaf_rn(N[i * 4 + k], a[k][4 + j], acc);
      out[i * 4 + j] = acc;
      nan_p |= isnan(acc);
    }
  const bool ok = !(nan_ref || nan_n || nan_p);
  valid[idx] = ok ? 1 : 0;
  for (int e = 0; e < 16; ++e) poses[(size_t)idx * 16 + e] = ok ? out[e] : 0.0f;
}

// data/dataloader_scannet.py:113-153 and data/dataloader_kitti.py:94-127 (get_ray_array + get_cam_intrinsics):
// grid-resolution intrinsics and the per-pixel rays K_raw^-1 (pixel centre) — evaluated in fp64 like the numpy originals
// and rounded to fp32 once, so the result is bit-identical to the reference's arrays.
// raw (B,8) doubles: fx, fy, cx, cy of the raw image; img_W, img_H = size of the (cropped) image the H x W grid spans;
// left_margin, top_margin = crop offsets (KITTI: raw_W-1216 over 2, raw_H-352; ScanNet: img = raw image, margins 0).
//   intM:  fx*(W/img_W), fy*(H/img_H), (cx-left)*(W/img_W), (cy-top)*(H/img_H)
//   ray_x: (((x+0.5)*(img_W/W) - cx) + left) / fx      (with left == 0 the "+ left" is exact: ScanNet's formula)
__global__ void camera_rays_kernel(const double* __restrict__ raw, int H, int W, float* __restrict__ intM,
                                   float* __restrict__ rays) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const size_t b = blockIdx.y;
  const double fx = raw[b * 8 + 0], fy = raw[b * 8 + 1], cx = raw[b * 8 + 2], cy = raw[b * 8 + 3];
  const double iw = raw[b * 8 + 4], ih = raw[b * 8 + 5], left = raw[b * 8 + 6], top = raw[b * 8 + 7];
  if (n == 0) {
    float* K = intM + b * 9;
    for (int e = 0; e < 9; ++e) K[e] = 0.0f;
    K[0] = (float)(fx * ((double)W / iw));
    K[4] = (float)(fy * ((double)H / ih));
    K[2] = (float)((cx - left) * ((double)W / iw));
    K[5] = (float)((cy - top) * ((double)H / ih));
    K[8] = 1.0f;
  }
  if (n >= H * W) return;
  const int x = n % W, y = n / W;
  const size_t HW = (size_t)H * W;
  // the product is rounded before cx is subtracted, as numpy does: a contracted fma would differ from the reference
  // wherever the pixel-centre position is not exact in fp64 (by far more than an ulp where it cancels against cx)
  rays[(b * 3 + 0) * HW + n] = (float)((__dadd_rn(__dmul_rn((double)x + 0.5, iw / (double)W), -cx) + left) / fx);
  rays[(b * 3 + 1) * HW + n] = (float)((__dadd_rn(__dmul_rn((double)y + 0.5, ih / (double)H), -cy) + top) / fy);
  rays[(b * 3 + 2) * HW + n] = 1.0f;
}

// ---- SURVEY §8 f-2: convex upsampling fused with the Gaussian NLL (utils/losses.py:34-50) ---------------------------
// One thread per full-resolution pixel: softmax over the 9 mask logits, the upsampled (mu, sigma) of
// upsample_depth_via_mask (MAGNET.py:15-27) and, where gt_mask is set, nll = (mu-gt)^2 / (2 var) + 0.5 log(var),
// var = max(sigma^2, 1e-10).  The (B,2,kH,kW) prediction is never written: forward emits one partial sum per CTA
// (summed by the caller: deterministic), backward scatters straight into grad_depth / grad_mask.
// The upsampled (mu, sigma) come from upsampled_gaussian (upsample_common.cuh), shared with the depth metrics.
//
// NllForm::DNET is DnetLoss (utils/losses.py:13-22) on D-Net's output (DESIGN §3.19): the second channel is the raw v
// of the depth head, upsampled the same way, and var = activation_G(v_up) (DNET.py:56-60, activation_g) before the same
// clamp var[var < 1e-10] = 1e-10 (dnet_var).
enum class NllForm { MAGNET, DNET };

// DnetLoss's variance of the upsampled raw v.  The clamp cannot fire unless v is NaN (which passes, as in torch):
// expm1f is within 1 ulp, so expm1f(v) >= -1 (the float below -1 is 2 ulps of [-1, -0.5) away from any e^v - 1 > -1);
// then expm1f(v) + 1 >= +0 exactly and activation_g(v) >= 0 + 1e-10f = 1e-10f, while torch compares the fp32 var with
// the fp32 1e-10f.  For v <= -17.4 expm1f(v) is -1 and var is exactly 1e-10f, unclamped, with its gradient.
__device__ __forceinline__ float dnet_var(float v) {
  const float a = activation_g(v);
  return a < 1e-10f ? 1e-10f : a;
}

template <NllForm F>
__global__ void __launch_bounds__(128) upsample_nll_fwd_kernel(const float* __restrict__ depth, const float* __restrict__ mask,
                                                                const float* __restrict__ gt, const uint8_t* __restrict__ gtm,
                                                                int H, int W, int k, float* __restrict__ partial) {
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y;
  const size_t b = blockIdx.z;
  float nll = 0.0f;
  if (X < W * k) {
    const size_t o = (b * H * k + Y) * (size_t)(W * k) + X;
    if (gtm[o]) {
      float w[9], mu, sg;                                   // sg: sigma (MAGNET) or the raw v (DNET)
      upsampled_gaussian(depth, mask, b, H, W, k, X / k, Y / k, X % k, Y % k, w, mu, sg);
      const float var = F == NllForm::MAGNET ? fmaxf(sg * sg, 1e-10f) : dnet_var(sg), d = mu - gt[o];
      nll = (d * d) / (2.0f * var) + 0.5f * logf(var);
    }
  }
  __shared__ float red[4];
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) nll += __shfl_xor_sync(0xffffffffu, nll, s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = nll;
  __syncthreads();
  if (threadIdx.x == 0)
    partial[(b * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = (red[0] + red[1]) + (red[2] + red[3]);
}

// scale = upstream gradient * iteration weight / number of supervised pixels: the argument, or with DEV_SCALE the
// device float *scale_dev (read at run time, so a captured graph takes it from memory)
template <NllForm F, bool DEV_SCALE>
__global__ void __launch_bounds__(128) upsample_nll_bwd_kernel(const float* __restrict__ depth, const float* __restrict__ mask,
                                                                const float* __restrict__ gt, const uint8_t* __restrict__ gtm,
                                                                float scale_arg, const float* __restrict__ scale_dev, int H,
                                                                int W, int k, float* __restrict__ gdepth,
                                                                float* __restrict__ gmask) {
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y;
  const size_t b = blockIdx.z;
  if (X >= W * k) return;
  const int x = X / k, kx = X % k, y = Y / k, ky = Y % k;
  const size_t HW = (size_t)H * W;
  const size_t moff = (b * 9 * k * k + (size_t)ky * k + kx) * HW + (size_t)y * W + x;
  const size_t o = (b * H * k + Y) * (size_t)(W * k) + X;
  if (!gtm[o]) {
#pragma unroll
    for (int i = 0; i < 9; ++i) gmask[moff + (size_t)i * k * k * HW] = 0.0f;
    return;
  }
  const float scale = DEV_SCALE ? __ldg(scale_dev) : scale_arg;
  float w[9], mu, sg;                                       // sg: sigma (MAGNET) or the raw v (DNET)
  upsampled_gaussian(depth, mask, b, H, W, k, x, y, kx, ky, w, mu, sg);
  float g_mu, g_sg;
  if constexpr (F == NllForm::MAGNET) {
    const float var = fmaxf(sg * sg, 1e-10f), d = mu - gt[o];
    g_mu = scale * d / var;
    // var[var < 1e-10] = 1e-10 (losses.py:45) cuts the gradient to sigma where it clamps
    g_sg = (sg * sg < 1e-10f) ? 0.0f : scale * (1.0f / sg - (d * d) / (var * sg));
  } else {
    const float var = dnet_var(sg), d = mu - gt[o];
    g_mu = scale * d / var;
    // d nll / d var times elu'(v) as ATen's elu backward forms it (exp(v) for v <= 0); zero where the clamp of
    // losses.py:20 fires (never for a non-NaN v, dnet_var)
    const float delu = sg <= 0.0f ? expf(sg) : 1.0f;
    g_sg = (activation_g(sg) < 1e-10f) ? 0.0f : scale * (0.5f / var - (d * d) / (2.0f * var * var)) * delu;
  }
  float t[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    t[i] = 0.0f;
    const int yy = y + i / 3 - 1, xx = x + i % 3 - 1;
    if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
      const size_t q = (size_t)yy * W + xx;
      t[i] = __fmaf_rn(g_sg, depth[(b * 2 + 1) * HW + q], g_mu * depth[(b * 2 + 0) * HW + q]);
      atomicAdd(gdepth + (b * 2 + 0) * HW + q, g_mu * w[i]);
      atomicAdd(gdepth + (b * 2 + 1) * HW + q, g_sg * w[i]);
    }
  }
  float dot = 0.0f;
#pragma unroll
  for (int i = 0; i < 9; ++i) dot = __fmaf_rn(w[i], t[i], dot);
#pragma unroll
  for (int i = 0; i < 9; ++i) gmask[moff + (size_t)i * k * k * HW] = w[i] * (t[i] - dot);
}

cudaError_t launch_upsample_nll_fwd(bool dnet, const float* depth, const float* mask, const float* gt, const uint8_t* gtm,
                                    int B, int H, int W, int k, float* partial, cudaStream_t st) {
  dim3 grid((W * k + 127) / 128, H * k, B);
  if (dnet)
    upsample_nll_fwd_kernel<NllForm::DNET><<<grid, 128, 0, st>>>(depth, mask, gt, gtm, H, W, k, partial);
  else
    upsample_nll_fwd_kernel<NllForm::MAGNET><<<grid, 128, 0, st>>>(depth, mask, gt, gtm, H, W, k, partial);
  return cudaGetLastError();
}

template <NllForm F>
static void upsample_nll_bwd(dim3 grid, const float* depth, const float* mask, const float* gt, const uint8_t* gtm,
                             float scale, const float* scale_dev, int H, int W, int k, float* gdepth, float* gmask,
                             cudaStream_t st) {
  if (scale_dev)
    upsample_nll_bwd_kernel<F, true><<<grid, 128, 0, st>>>(depth, mask, gt, gtm, 0.0f, scale_dev, H, W, k, gdepth, gmask);
  else
    upsample_nll_bwd_kernel<F, false><<<grid, 128, 0, st>>>(depth, mask, gt, gtm, scale, nullptr, H, W, k, gdepth, gmask);
}

cudaError_t launch_upsample_nll_bwd(bool dnet, const float* depth, const float* mask, const float* gt, const uint8_t* gtm,
                                    float scale, const float* scale_dev, int B, int H, int W, int k, float* gdepth,
                                    float* gmask, cudaStream_t st) {
  dim3 grid((W * k + 127) / 128, H * k, B);
  if (dnet)
    upsample_nll_bwd<NllForm::DNET>(grid, depth, mask, gt, gtm, scale, scale_dev, H, W, k, gdepth, gmask, st);
  else
    upsample_nll_bwd<NllForm::MAGNET>(grid, depth, mask, gt, gtm, scale, scale_dev, H, W, k, gdepth, gmask, st);
  return cudaGetLastError();
}

cudaError_t launch_relative_poses(const float* ext_ref, const float* ext_nghbr, int B, int V, float* poses,
                                  int32_t* valid, cudaStream_t st) {
  relative_poses_kernel<<<(B * V + 63) / 64, 64, 0, st>>>(ext_ref, ext_nghbr, B, V, poses, valid);
  return cudaGetLastError();
}

cudaError_t launch_camera_rays(const double* raw, int B, int H, int W, float* intM, float* rays, cudaStream_t st) {
  camera_rays_kernel<<<dim3((H * W + 255) / 256, B), 256, 0, st>>>(raw, H, W, intM, rays);
  return cudaGetLastError();
}

cudaError_t launch_upsample_fwd(const float* depth, const float* mask, int B, int CH, int H, int W, int k, float* out,
                                cudaStream_t st) {
  dim3 grid((W * k + 127) / 128, H * k, B);
  if (CH == 1) convex_upsample_fwd_kernel<1><<<grid, 128, 0, st>>>(depth, mask, H, W, k, out);
  else if (CH == 2) convex_upsample_fwd_kernel<2><<<grid, 128, 0, st>>>(depth, mask, H, W, k, out);
  else return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_upsample_bwd(const float* gout, const float* depth, const float* mask, int B, int CH, int H, int W,
                                int k, float* gdepth, float* gmask, cudaStream_t st) {
  dim3 grid((W * k + 127) / 128, H * k, B);
  if (CH == 1) convex_upsample_bwd_kernel<1><<<grid, 128, 0, st>>>(gout, depth, mask, H, W, k, gdepth, gmask);
  else if (CH == 2) convex_upsample_bwd_kernel<2><<<grid, 128, 0, st>>>(gout, depth, mask, H, W, k, gdepth, gmask);
  else return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_pack_cameras(const float* intM, const float* R, int64_t r_sb, int64_t r_sv, int64_t r_si,
                                int64_t r_sj, const float* t, int64_t t_sb, int64_t t_sv, int64_t t_si,
                                const int32_t* is_valid, int B, int V, magnet_camera* out, cudaStream_t st) {
  const int n = B * V;
  pack_cameras_kernel<<<(n + 63) / 64, 64, 0, st>>>(intM, R, r_sb, r_sv, r_si, r_sj, t, t_sb, t_sv, t_si,
                                                    is_valid, B, V, out);
  return cudaGetLastError();
}

cudaError_t launch_repack(const float* src, float* dst, int N, int C, int H, int W, cudaStream_t st) {
  const int C4 = C / 4, XB = (W + 31) / 32;
  dim3 grid(XB, H, N * ((C4 + 3) / 4)), block(32, 4);
  repack_tiled32_kernel<<<grid, block, 0, st>>>(src, reinterpret_cast<float4*>(dst), C4, H, W, XB);
  return cudaGetLastError();
}

cudaError_t launch_sample(const float* gmm, const float* k_host, int B, int D, int HW, float* dvol,
                          cudaStream_t st) {
  KParams kp;
  for (int j = 0; j < MAGNET_MAX_PLANES; ++j) kp.k[j] = j < D ? k_host[j] : 0.0f;
  sample_depths_kernel<<<dim3((HW + 255) / 256, B), 256, 0, st>>>(gmm, kp, D, HW, dvol);
  return cudaGetLastError();
}

cudaError_t launch_update_fwd(const float* dout, const float* gmm0, int B, int HW, float* out, cudaStream_t st) {
  gaussian_update_fwd_kernel<<<dim3((HW + 255) / 256, B), 256, 0, st>>>(dout, gmm0, HW, out);
  return cudaGetLastError();
}

cudaError_t launch_update_bwd(const float* gout, const float* dout, const float* gmm0, int B, int HW, float* gin,
                              cudaStream_t st) {
  gaussian_update_bwd_kernel<<<dim3((HW + 255) / 256, B), 256, 0, st>>>(gout, dout, gmm0, HW, gin);
  return cudaGetLastError();
}

// The frame table's range check on the device (magnet_check_src_index): one CTA per row b.  Each entry is compared in
// its own width, so an int64 entry >= 2^31 is out of range rather than wrapped; out-of-range entries become 0 in `out`
// and set bad[b].  Every entry and every bad[b] is written, so no memset precedes the launch.
template <class T>
__global__ void __launch_bounds__(128) check_src_index_kernel(const T* __restrict__ idx, int V, int n_src,
                                                              int32_t* __restrict__ out, int32_t* __restrict__ bad) {
  const size_t row = (size_t)blockIdx.x * V;
  int any = 0;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    const T e = idx[row + v];
    const bool ok = e >= 0 && e < (T)n_src;
    out[row + v] = ok ? (int32_t)e : 0;
    any |= !ok;
  }
  any = __syncthreads_or(any);
  if (threadIdx.x == 0) bad[blockIdx.x] = any;
}

cudaError_t launch_check_src_index(const void* idx, bool wide, int B, int V, int n_src, int32_t* out, int32_t* bad,
                                   cudaStream_t st) {
  const int threads = V >= 128 ? 128 : (V + 31) / 32 * 32;
  if (wide)
    check_src_index_kernel<int64_t><<<B, threads, 0, st>>>(static_cast<const int64_t*>(idx), V, n_src, out, bad);
  else
    check_src_index_kernel<int32_t><<<B, threads, 0, st>>>(static_cast<const int32_t*>(idx), V, n_src, out, bad);
  return cudaGetLastError();
}

}  // namespace magnet
