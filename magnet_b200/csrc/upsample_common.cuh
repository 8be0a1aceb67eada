// Device code of the learned convex upsampling shared by the fused kernels that never materialise the
// full-resolution prediction: the upsample + NLL loss (aux_kernels.cu) and the depth metrics (depth_metrics.cu).
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

}  // namespace magnet
