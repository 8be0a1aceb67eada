// The consistency test of the CW volume (homography.py:143-158) in the operation sequence of the tensor-core forward
// (cost_mma.cu), shared with the CW backward (cost_cw_bwd.cu): both evaluate these helpers on the same inputs, so the
// backward applies exactly the mask of the forward call that produced the volume.
//   sample position (ix, iy) = project2 / project of common.cuh / cells_common.cuh, clamped by clamp_coord;
//   cell origin x0 = floor(ix), fraction fx = ix - x0 (cell_split);
//   (mu~, sigma~) = lerp2d over the four (mu, sigma) taps, zero outside the image (lerp2d_x2 on the paired table);
//   keep <=> |z - mu~| < sigma~ * kappa, strict (cw_keep).
#pragma once
#include "common.cuh"

namespace magnet {

// Anything left of -1 / right of W (above / below likewise) has all four taps out of the image: clamp so that cells stay
// near the image; NaN (fmaxf drops it) maps to "out of bounds".  xmax = W + 1 (ymax = H + 1).
__device__ __forceinline__ float clamp_coord(float x, float xmax) { return fminf(fmaxf(x, -2.0f), xmax); }

// cell origin and fraction: x - floor(x) is exact, written as fma(x0, -1, x)
__device__ __forceinline__ void cell_split(float x, float& x0, float& f) {
  x0 = floorf(x);
  f = __fmaf_rn(x0, -1.0f, x);
}

// bilinear interpolation v00 + fx (v01 - v00), then along y; v01 - v00 as fma(v00, -1, v01) (exact product, one
// rounding = the subtraction)
__device__ __forceinline__ float lerp2d(float v00, float v01, float v10, float v11, float fx, float fy) {
  const float t = __fmaf_rn(fx, __fmaf_rn(v00, -1.0f, v01), v00);
  const float u = __fmaf_rn(fx, __fmaf_rn(v10, -1.0f, v11), v10);
  return __fmaf_rn(fy, __fmaf_rn(t, -1.0f, u), t);
}

// a (mu, sigma) pair from the paired table: top = (mu, sigma) of taps (x0, y0), (x0 + 1, y0); bot likewise at y0 + 1
__device__ __forceinline__ float2 lerp2d_x2(float4 top, float4 bot, float fx, float fy) {
  return make_float2(lerp2d(top.x, top.z, bot.x, bot.z, fx, fy), lerp2d(top.y, top.w, bot.y, bot.w, fx, fy));
}

// homography.py:157-158: |z - mu~| < sigma~ * kappa, strict
__device__ __forceinline__ bool cw_keep(float z, float2 ms, float kappa) {
  return fabsf(__fsub_rn(z, ms.x)) < __fmul_rn(ms.y, kappa);
}

}  // namespace magnet
