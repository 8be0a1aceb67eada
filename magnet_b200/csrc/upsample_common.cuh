// Device code of the learned convex upsampling shared by the fused kernels that never materialise the
// full-resolution prediction: the upsample + NLL loss (aux_kernels.cu) and the depth metrics (depth_metrics.cu), which
// load the mask logits (upsampled_gaussian), and the fused mask head (mask_head.cu), which has them in registers
// (convex_gaussian).  Both forms run the same operations in the same order, so equal logits give equal bits; the
// loading form is kept as its own text so that the kernels which use it compile exactly as before.
#pragma once
#include <cstddef>
#include <cmath>

namespace magnet {

// upsample_depth_via_mask (MAGNET.py:15-27) at one full-resolution pixel (X = x*k+kx, Y = y*k+ky) of image b:
// softmax over the 9 mask logits mask[b, (i*k+ky)*k+kx, y, x] (written to w), weighted sum of the zero-padded 3x3
// neighbourhood of the quarter-resolution [mu, sigma] in depth (B,2,H,W).
__device__ __forceinline__ void upsampled_gaussian(const float* __restrict__ depth, const float* __restrict__ mask,
                                                   size_t b, int H, int W, int k, int x, int y, int kx, int ky,
                                                   float (&w)[9], float& mu, float& sg) {
  const size_t HW = (size_t)H * W;
  const float* mp = mask + (b * 9 * k * k + (size_t)ky * k + kx) * HW + (size_t)y * W + x;
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < 9; ++i) { w[i] = mp[(size_t)i * k * k * HW]; m = fmaxf(m, w[i]); }
  float s = 0.0f;
#pragma unroll
  for (int i = 0; i < 9; ++i) { w[i] = expf(w[i] - m); s += w[i]; }
  const float inv = 1.0f / s;
  mu = sg = 0.0f;
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    w[i] *= inv;
    const int yy = y + i / 3 - 1, xx = x + i % 3 - 1;
    if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
      mu = __fmaf_rn(w[i], depth[(b * 2 + 0) * HW + (size_t)yy * W + xx], mu);
      sg = __fmaf_rn(w[i], depth[(b * 2 + 1) * HW + (size_t)yy * W + xx], sg);
    }
  }
}

// The register form of upsampled_gaussian: the 9 logits of one full-resolution pixel are in w (tap i at dy = i/3 - 1,
// dx = i%3 - 1).  Max, exp, sum, one reciprocal; then tap by tap the scaled weight (left in w) and, when tap(i, a, c)
// finds the neighbour inside the image (a, c = its quarter-resolution [mu, sigma]), one FMA each into mu and sg.
template <class Tap>
__device__ __forceinline__ void convex_gaussian(float (&w)[9], Tap tap, float& mu, float& sg) {
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < 9; ++i) m = fmaxf(m, w[i]);
  float s = 0.0f;
#pragma unroll
  for (int i = 0; i < 9; ++i) { w[i] = expf(w[i] - m); s += w[i]; }
  const float inv = 1.0f / s;
  mu = sg = 0.0f;
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    w[i] *= inv;
    float a, c;
    if (tap(i, a, c)) {
      mu = __fmaf_rn(w[i], a, mu);
      sg = __fmaf_rn(w[i], c, sg);
    }
  }
}

// The combination alone, with the weights convex_gaussian left in w: another prediction under the same mask.
template <class Tap>
__device__ __forceinline__ void convex_combine(const float (&w)[9], Tap tap, float& mu, float& sg) {
  mu = sg = 0.0f;
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    float a, c;
    if (tap(i, a, c)) {
      mu = __fmaf_rn(w[i], a, mu);
      sg = __fmaf_rn(w[i], c, sg);
    }
  }
}

}  // namespace magnet
