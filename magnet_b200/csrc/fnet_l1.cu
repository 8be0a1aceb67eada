// F-Net training loss, fused: soft-argmin over the D planes + masked L1 — replaces train_FNet.py:96-108
//   prob = softmax_j(score) (homography.py:46), pred = sum_j prob_j d_j, loss = mean over mask of |pred - gt|
// on the 1/V-averaged scores of the plane-sweep volume (magnet_cost_volume_f32 with softmax == 0).  One thread per
// (b, pixel); neither the (B,D,H,W) probability volume nor the (B,1,H,W) prediction is written.
//   forward: one partial sum of |pred - gt| per CTA of 128 pixels (the caller adds them and divides by the count)
//   backward: dL/dscore_j = prob_j (d_j - pred) sign(pred - gt) mask scale, sign(0) = 0 (torch's abs backward)
#include "common.cuh"
#include "launchers.h"
#include "soft_argmin.cuh"

namespace magnet {

constexpr int L1_THREADS = 128;

struct FnetL1Params {
  int D, HW;
  float scale;                          // backward: upstream gradient / number of supervised pixels
  const float* __restrict__ scores;     // (B,D,H,W)
  const float* __restrict__ gt;         // (B,1,H,W)
  const uint8_t* __restrict__ mask;     // (B,1,H,W)
  const float* __restrict__ grad_scale; // device scalar multiplying `scale`, or NULL
  float* __restrict__ out;              // partials (forward) / dL/dscores (backward)
  float d[MAGNET_MAX_PLANES];           // plane depths
};

__global__ void __launch_bounds__(L1_THREADS) fnet_l1_fwd_kernel(const __grid_constant__ FnetL1Params p) {
  const int n = blockIdx.x * L1_THREADS + threadIdx.x;
  const size_t b = blockIdx.y;
  float l1 = 0.0f;
  if (n < p.HW && p.mask[b * p.HW + n]) {
    float m, inv_z, pred;
    soft_argmin(p.scores + b * p.D * p.HW + n, p.HW, p.D, p.d, m, inv_z, pred);
    l1 = fabsf(pred - p.gt[b * p.HW + n]);
  }
  __shared__ float red[L1_THREADS / 32];
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) l1 += __shfl_xor_sync(0xffffffffu, l1, s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = l1;
  __syncthreads();
  if (threadIdx.x == 0) p.out[b * gridDim.x + blockIdx.x] = (red[0] + red[1]) + (red[2] + red[3]);
}

__global__ void __launch_bounds__(L1_THREADS) fnet_l1_bwd_kernel(const __grid_constant__ FnetL1Params p) {
  const int n = blockIdx.x * L1_THREADS + threadIdx.x;
  if (n >= p.HW) return;
  const size_t b = blockIdx.y;
  const float* s = p.scores + b * p.D * p.HW + n;
  float* g = p.out + b * p.D * p.HW + n;
  float coef = 0.0f, m = 0.0f, inv_z = 0.0f, pred = 0.0f;
  if (p.mask[b * p.HW + n]) {
    soft_argmin(s, p.HW, p.D, p.d, m, inv_z, pred);
    const float d = pred - p.gt[b * p.HW + n];
    const float sgn = d > 0.0f ? 1.0f : (d < 0.0f ? -1.0f : 0.0f);
    coef = sgn * p.scale * (p.grad_scale != nullptr ? *p.grad_scale : 1.0f);
  }
  if (coef == 0.0f) {
    for (int j = 0; j < p.D; ++j) g[(size_t)j * p.HW] = 0.0f;
    return;
  }
  for (int j = 0; j < p.D; ++j) {
    const float pj = expf(s[(size_t)j * p.HW] - m) * inv_z;
    g[(size_t)j * p.HW] = pj * (p.d[j] - pred) * coef;
  }
}

int fnet_l1_partials(int B, int HW) { return B * ((HW + L1_THREADS - 1) / L1_THREADS); }

static FnetL1Params l1_params(const float* scores, const float* planes, const float* gt, const uint8_t* mask, int D,
                              int HW, float scale, const float* grad_scale, float* out) {
  FnetL1Params p;
  p.D = D; p.HW = HW; p.scale = scale;
  p.scores = scores; p.gt = gt; p.mask = mask; p.grad_scale = grad_scale; p.out = out;
  for (int j = 0; j < MAGNET_MAX_PLANES; ++j) p.d[j] = j < D ? planes[j] : 0.0f;
  return p;
}

cudaError_t launch_fnet_l1_fwd(const float* scores, const float* planes, const float* gt, const uint8_t* mask, int B,
                               int D, int HW, float* partial, cudaStream_t st) {
  const FnetL1Params p = l1_params(scores, planes, gt, mask, D, HW, 0.0f, nullptr, partial);
  fnet_l1_fwd_kernel<<<dim3((HW + L1_THREADS - 1) / L1_THREADS, B), L1_THREADS, 0, st>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_fnet_l1_bwd(const float* scores, const float* planes, const float* gt, const uint8_t* mask,
                               float scale, const float* grad_scale, int B, int D, int HW, float* grad_scores,
                               cudaStream_t st) {
  const FnetL1Params p = l1_params(scores, planes, gt, mask, D, HW, scale, grad_scale, grad_scores);
  fnet_l1_bwd_kernel<<<dim3((HW + L1_THREADS - 1) / L1_THREADS, B), L1_THREADS, 0, st>>>(p);
  return cudaGetLastError();
}

}  // namespace magnet
