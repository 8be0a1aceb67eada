// F-Net depth map: the soft-argmin prediction sum_j prob_j d_j of train_FNet.py:96 / :180 from a (B,D,H,W) plane
// volume, written as (B,1,H,W).  One thread per (b, pixel); consecutive threads read consecutive pixels of a plane.
//   scores form: the 1/V-averaged scores of magnet_cost_volume_f32 (softmax == 0); the softmax over the planes is
//     fused in (soft_argmin.cuh, the same code as the training loss), the probability volume is never written.
//   probabilities form: the output of est_costvolume_F / MAGNET_F.forward; pred = sum_j p_j d_j in plane order.
#include "common.cuh"
#include "launchers.h"
#include "soft_argmin.cuh"

namespace magnet {

constexpr int PD_THREADS = 128;

struct PlaneDepthParams {
  int D, HW;
  const float* __restrict__ vol;   // (B,D,H,W)
  float* __restrict__ out;         // (B,1,H,W)
  float d[MAGNET_MAX_PLANES];      // plane depths
};

template <bool SCORES>
__global__ void __launch_bounds__(PD_THREADS) plane_depth_kernel(const __grid_constant__ PlaneDepthParams p) {
  const int n = blockIdx.x * PD_THREADS + threadIdx.x;
  if (n >= p.HW) return;
  const size_t b = blockIdx.y;
  const float* s = p.vol + b * p.D * p.HW + n;
  float pred;
  if (SCORES) {
    float m, inv_z;
    soft_argmin(s, p.HW, p.D, p.d, m, inv_z, pred);
  } else {
    pred = 0.0f;
    for (int j = 0; j < p.D; ++j) pred = __fmaf_rn(s[(size_t)j * p.HW], p.d[j], pred);
  }
  p.out[b * p.HW + n] = pred;
}

cudaError_t launch_plane_depth(const float* vol, const float* planes, int B, int D, int HW, bool scores, float* out,
                               cudaStream_t st) {
  PlaneDepthParams p;
  p.D = D; p.HW = HW; p.vol = vol; p.out = out;
  for (int j = 0; j < MAGNET_MAX_PLANES; ++j) p.d[j] = j < D ? planes[j] : 0.0f;
  const dim3 grid((HW + PD_THREADS - 1) / PD_THREADS, B);
  if (scores)
    plane_depth_kernel<true><<<grid, PD_THREADS, 0, st>>>(p);
  else
    plane_depth_kernel<false><<<grid, PD_THREADS, 0, st>>>(p);
  return cudaGetLastError();
}

}  // namespace magnet
