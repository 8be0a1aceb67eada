// Soft-argmin over the D planes of one pixel, shared by the F-Net training loss (fnet_l1.cu) and the F-Net depth map
// (plane_depth.cu), so that the evaluated prediction is bit for bit the one the loss supervises.
//   prob_j = softmax_j(s_j) (homography.py:46), pred = sum_j prob_j d_j
// s points at the pixel's first plane, consecutive planes are `stride` floats apart; d holds the D plane depths.
// A row with a NaN, or whose maximum is infinite, gives NaN (as torch.softmax: exp(inf - inf) = NaN).  Full-precision
// expf: the library is compiled without fast-math.
#pragma once

namespace magnet {

// softmax statistics of one pixel: max, 1 / sum exp(s - max) and the soft-argmin prediction
__device__ __forceinline__ void soft_argmin(const float* s, int stride, int D, const float* d, float& m, float& inv_z,
                                            float& pred) {
  m = -INFINITY;
  for (int j = 0; j < D; ++j) m = fmaxf(m, s[(size_t)j * stride]);
  float z = 0.0f, num = 0.0f;
  for (int j = 0; j < D; ++j) {
    const float e = expf(s[(size_t)j * stride] - m);
    z += e;
    num = __fmaf_rn(e, d[j], num);
  }
  inv_z = 1.0f / z;
  pred = num * inv_z;
}

}  // namespace magnet
