// Shared device helpers for the MaGNet matching kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <mutex>
#include <type_traits>

#include "../../include/magnet_b200.h"

namespace magnet {

inline size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

// Opt-in shared memory (and, with max_carveout, the largest carveout): set once per (kernel, device), not on every
// launch.  `flags` belongs to the kernel; dev, when given, receives the current device.
template <typename K>
cudaError_t set_smem_once(K kern, std::once_flag (&flags)[64], int bytes, bool max_carveout, int* dev = nullptr) {
  int d = 0;
  cudaError_t e = cudaGetDevice(&d);
  if (e != cudaSuccess) return e;
  if (dev) *dev = d;
  std::call_once(flags[d & 63], [&] {
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess && max_carveout)
      e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  });
  return e;
}

// Runtime value -> compile-time constant.  A Choice<T, Vs...> holds a value that is one of Vs; dispatch(f, c...) calls
// f(std::integral_constant<T, V>{}...) with the V that each choice holds, and returns cudaErrorInvalidValue when one
// holds none of its Vs.  Every combination of the Vs is instantiated: a launcher whose kernel exists for only part of
// the product says so with `if constexpr` in f.
template <class T, T... Vs>
struct Choice {
  T value;
};
using DepthMode = Choice<int, MAGNET_DEPTH_VOLUME, MAGNET_DEPTH_GAUSS, MAGNET_DEPTH_PLANES>;
using Flag = Choice<bool, false, true>;

template <class F>
cudaError_t dispatch(F&& f) {
  return f();
}
template <class F, class T, T... Vs, class... Rest>
cudaError_t dispatch(F&& f, Choice<T, Vs...> c, Rest... rest);
template <class T, T V, class F, class... Rest>
cudaError_t dispatch_fixed(F& f, Rest... rest) {   // f with its first argument bound to V
  return dispatch([&f](auto... cs) { return f(std::integral_constant<T, V>{}, cs...); }, rest...);
}
template <class F, class T, T... Vs, class... Rest>
cudaError_t dispatch(F&& f, Choice<T, Vs...> c, Rest... rest) {
  cudaError_t e = cudaErrorInvalidValue;
  (void)((c.value == Vs && ((e = dispatch_fixed<T, Vs>(f, rest...)), true)) || ...);
  return e;
}

// Work slots of the persistent kernels: each launch takes one slot of its family's arrays (host ticket, work_slot() in
// launchers.h); `next` counts the work items handed out, `done` the CTAs that finished, and the launch's last CTA
// re-arms the slot, so a captured launch can be replayed and no memset precedes a launch.  Launches that share a slot
// must not run concurrently: WORK_SLOTS / 2 eager launches or as many captured ones would have to be in flight at once.
constexpr int WORK_SLOTS = 1024;

// the next work item of the launch (0, 1, ... in claim order)
__device__ __forceinline__ unsigned slot_claim(unsigned* next, int slot) { return atomicAdd(&next[slot], 1u); }

// once per CTA, after its last global write: true in the launch's last CTA to finish
__device__ __forceinline__ bool slot_last_cta(unsigned* done, int slot) {
  __threadfence();
  return atomicAdd(&done[slot], 1u) == gridDim.x - 1;
}

// once per CTA at exit: the last CTA re-arms the work counter
__device__ __forceinline__ void slot_finish(unsigned* next, unsigned* done, int slot) {
  if (slot_last_cta(done, slot)) {
    next[slot] = 0u;
    done[slot] = 0u;
    __threadfence();
  }
}

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

// Source image of view (b, v) of a cost-volume forward: the view-major slot v*B + b (homography.py:105), or with IDX
// the entry b*V + v of the caller's frame table (magnet_cost_volume_indexed_f32).  IDX is a template flag, so the
// view-major instantiations compile to the code they had before the table existed.
template <bool IDX>
__device__ __forceinline__ int src_image(const int32_t* __restrict__ src_index, int b, int v, int B, int V) {
  if constexpr (IDX) return __ldg(src_index + b * V + v);
  else return v * B + b;
}

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
