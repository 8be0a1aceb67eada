// Shared device helpers for the MaGNet matching kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/magnet_b200.h"

namespace magnet {

// Kernel-side view of magnet_cost_args; k values travel in the launch parameters
// (constant bank, uniform loads) so that no __constant__ symbol / extra copy is needed.
struct CostParams {
  int B, V, D, H, W, HW;
  int k_sorted;       // 1 when k[0..D) is non-decreasing (enables the analytic cell walk)
  float kappa;
  float inv_v_exact;  // 1/V when V is a power of two (exact), else 0 -> use IEEE division
  float vf;           // float(V)
  const float* __restrict__ ref_feat;
  const float* __restrict__ src_feat;
  const float* __restrict__ src_gmm;
  const float* __restrict__ rays;
  const magnet_camera* __restrict__ cams;
  const float* __restrict__ d_volume;
  const float* __restrict__ ref_gmm;
  float* __restrict__ out;
  float k[MAGNET_MAX_PLANES];
};

// Kernel-side arguments of the F-volume backward (magnet_cost_f_bwd_args + the geometry of its forward call).
struct BwdParams {
  int B, V, D, C, H, W, HW;
  int softmax;
  float vf;
  const float* __restrict__ ref_feat;   // (B,C,H,W)
  const float* __restrict__ src_feat;   // (V*B,C,H,W) NCHW
  const float* __restrict__ rays;
  const magnet_camera* __restrict__ cams;
  const float* __restrict__ prob;       // (B,D,H,W) forward output (softmax == 1) or unused
  const float* __restrict__ grad_out;   // (B,D,H,W)
  float* __restrict__ g_score;          // (B,D,H,W) workspace
  float* __restrict__ grad_ref;         // (B,C,H,W), written
  float* __restrict__ grad_src;         // (V*B,C,H,W), accumulated with atomics (caller zeroes it)
  float k[MAGNET_MAX_PLANES];
};

// Kernel-side arguments of the CW-volume backward (magnet_cost_bwd_args + the geometry of its forward call).
struct CwBwdParams {
  int B, V, D, H, W, HW;
  int cw;                                  // 1: consistency-weighted (the mask is applied), 0: plain sweep
  float kappa;
  const float* __restrict__ ref_feat;      // (B,C,H,W) NCHW
  const float* __restrict__ src_feat;      // (V*B,C,H,W) NCHW
  const float* __restrict__ src_gmm;       // (V*B,2,H,W)
  const float* __restrict__ rays;
  const magnet_camera* __restrict__ cams;
  const float* __restrict__ d_volume;      // (B,D,H,W), MAGNET_DEPTH_VOLUME
  const float* __restrict__ ref_gmm;       // (B,2,H,W), MAGNET_DEPTH_GAUSS
  const float* __restrict__ g_score;       // (B,D,H,W) = grad_out / V
  float* __restrict__ grad_ref;            // (B,C,H,W) written, or NULL
  float* __restrict__ grad_src;            // (V*B,C,H,W) accumulated with atomics, or NULL
  float* __restrict__ grad_depth;          // VOLUME (B,D,H,W) / GAUSS (B,2,H,W) written, or NULL
  float k[MAGNET_MAX_PLANES];
};

// 1/x to <1 ulp: MUFU.RCP + one Newton step.  x == 0 -> NaN/inf, which the callers'
// coordinate clamp turns into "out of bounds" (same outcome as the reference's +-10 clamp).
__device__ __forceinline__ float rcp_nr(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return __fmaf_rn(r, __fmaf_rn(-x, r, 1.0f), r);
}

__device__ __forceinline__ float ldg_f(const float* p) { return __ldg(p); }

// SPLIT16 scale rule: the power-of-two shift that maps absmax into [2^14, 2^15); 0 (scale 1) for an all-zero or
// non-finite tensor
__device__ __forceinline__ int split16_shift(unsigned absmax_bits) {
  const int e = (int)(absmax_bits >> 23) & 0xff;
  if (e == 0 || e == 255) return 0;
  return max(-100, min(100, 14 - (e - 127)));
}

// Element-wise float2 arithmetic, each element one IEEE round-to-nearest operation (sm_90 has no packed f32x2 FMA):
// the kernels evaluate two hypotheses / two channel partial sums side by side with these.
__device__ __forceinline__ float2 ffma2_rn(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fadd2_rn(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }

// Two hypotheses at once: continuous sample position (ix, iy) = projected pixel - 0.5 (SURVEY A.2 / A.5 #1) and z =
// depth in the source camera.  Element by element the same IEEE operations as the scalar project() of cells_common.cuh
// (z = a2 + q2*d separately rounded, 1/(z + 1e-10) = MUFU.RCP + one Newton step), so results are bit-identical to
// evaluating the two hypotheses one after the other.
__device__ __forceinline__ void project2(const float2 d, float a0, float a1, float a2, float q0, float q1, float q2,
                                         float2& ix, float2& iy, float2& z) {
  const float2 P0 = ffma2_rn(make_float2(q0, q0), d, make_float2(a0, a0));
  const float2 P1 = ffma2_rn(make_float2(q1, q1), d, make_float2(a1, a1));
  // the products are rounded by __fmul_rn, never contracted into an FMA: z is rounded twice, as in the reference
  z = fadd2_rn(make_float2(a2, a2), make_float2(__fmul_rn(q2, d.x), __fmul_rn(q2, d.y)));
  const float2 zp = fadd2_rn(z, make_float2(1e-10f, 1e-10f));
  float2 r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r.x) : "f"(zp.x));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r.y) : "f"(zp.y));
  const float2 e = ffma2_rn(make_float2(-zp.x, -zp.y), r, make_float2(1.0f, 1.0f));
  r = ffma2_rn(r, e, r);
  ix = ffma2_rn(P0, r, make_float2(-0.5f, -0.5f));
  iy = ffma2_rn(P1, r, make_float2(-0.5f, -0.5f));
}

}  // namespace magnet
