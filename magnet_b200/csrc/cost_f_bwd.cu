// Backward of the fronto-parallel plane-sweep volume (homography.est_costvolume_F, homography.py:10-75) w.r.t.
// both feature maps — SURVEY §8 row f-1 (F-Net training, train_FNet.py:95-114).
//
//   score[b,j,p] = 1/V * sum_v sum_t w_t(v,j,p) * <ref[b,:,p], src_v[:, tap_t]> ;  prob = softmax_j(score)
//   g_score = prob * (g_prob - sum_j prob * g_prob) / V                                   (kernel 1)
//   g_ref[b,c,p]   += sum_{v,j,t} g_score * w_t * src_v[c, tap_t]                        (kernel 2, registers)
//   g_src[v,c,tap] += sum_{p,j: tap_t(p,j)=tap} g_score * w_t * ref[b,c,p]                (kernel 2, atomics)
// Tap sharing as in the forward: the planes of one pixel that fall into the same bilinear cell are first
// reduced to 4 corner coefficients G_t = sum_j g_score_j * w_t(j); only a change of cell touches the C channels
// (4 gathers + 4 red.add per channel).  One thread per (b, pixel); exact per-plane walk (any plane order).
// Correctness-first implementation: it is not on the frames/s path (F-Net training only).
#include "cells_common.cuh"

namespace magnet {

__global__ void score_grad_kernel(const __grid_constant__ BwdParams p) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= p.HW) return;
  const size_t base = (size_t)blockIdx.y * p.D * p.HW + n;
  const float inv_v = 1.0f / p.vf;
  if (p.softmax) {
    float dot = 0.0f;
    for (int j = 0; j < p.D; ++j) dot += p.prob[base + (size_t)j * p.HW] * p.grad_out[base + (size_t)j * p.HW];
    for (int j = 0; j < p.D; ++j) {
      const float pr = p.prob[base + (size_t)j * p.HW];
      p.g_score[base + (size_t)j * p.HW] = pr * (p.grad_out[base + (size_t)j * p.HW] - dot) * inv_v;
    }
  } else {
    for (int j = 0; j < p.D; ++j) p.g_score[base + (size_t)j * p.HW] = p.grad_out[base + (size_t)j * p.HW] * inv_v;
  }
}

template <int C>
__global__ void __launch_bounds__(128)
cost_f_bwd_kernel(const __grid_constant__ BwdParams p) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= p.HW) return;
  const int b = blockIdx.y, H = p.H, W = p.W, HW = p.HW;
  float ref[C], gref[C];
#pragma unroll
  for (int c = 0; c < C; ++c) {
    ref[c] = ldg_f(p.ref_feat + ((size_t)b * C + c) * HW + n);
    gref[c] = 0.0f;
  }
  const float r0 = ldg_f(p.rays + ((size_t)b * 3 + 0) * HW + n);
  const float r1 = ldg_f(p.rays + ((size_t)b * 3 + 1) * HW + n);
  const float r2 = ldg_f(p.rays + ((size_t)b * 3 + 2) * HW + n);
  const float* gs = p.g_score + (size_t)b * p.D * HW + n;
  const float xmax = (float)W + 1.0f, ymax = (float)H + 1.0f;

  for (int v = 0; v < p.V; ++v) {
    const magnet_camera* cam = p.cams + (b * p.V + v);
    if (cam->valid != 1.0f) continue;
    const float a0 = cam->a[0], a1 = cam->a[1], a2 = cam->a[2];
    const float q0 = __fmaf_rn(cam->A[2], r2, __fmaf_rn(cam->A[1], r1, __fmul_rn(cam->A[0], r0)));
    const float q1 = __fmaf_rn(cam->A[5], r2, __fmaf_rn(cam->A[4], r1, __fmul_rn(cam->A[3], r0)));
    const float q2 = __fmaf_rn(cam->A[8], r2, __fmaf_rn(cam->A[7], r1, __fmul_rn(cam->A[6], r0)));
    const int vb = v * p.B + b;
    const float* src = p.src_feat + (size_t)vb * C * HW;
    float* gsrc = p.grad_src + (size_t)vb * C * HW;

    float cx = -1e30f, cy = -1e30f;
    float G00 = 0.f, G01 = 0.f, G10 = 0.f, G11 = 0.f;
    auto flush = [&]() {
      if (cx < -1e29f) return;
      const int x0 = (int)cx, y0 = (int)cy, x1 = x0 + 1, y1 = y0 + 1;
      const bool i00 = x0 >= 0 && x0 < W && y0 >= 0 && y0 < H, i01 = x1 >= 0 && x1 < W && y0 >= 0 && y0 < H;
      const bool i10 = x0 >= 0 && x0 < W && y1 >= 0 && y1 < H, i11 = x1 >= 0 && x1 < W && y1 >= 0 && y1 < H;
      if (!(i00 | i01 | i10 | i11)) return;
      if (G00 == 0.f && G01 == 0.f && G10 == 0.f && G11 == 0.f) return;
      const int o00 = y0 * W + x0, o01 = o00 + 1, o10 = o00 + W, o11 = o10 + 1;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const float* s = src + (size_t)c * HW;
        float* g = gsrc + (size_t)c * HW;
        float acc = gref[c];
        if (i00) { acc = __fmaf_rn(G00, ldg_f(s + o00), acc); atomicAdd(g + o00, G00 * ref[c]); }
        if (i01) { acc = __fmaf_rn(G01, ldg_f(s + o01), acc); atomicAdd(g + o01, G01 * ref[c]); }
        if (i10) { acc = __fmaf_rn(G10, ldg_f(s + o10), acc); atomicAdd(g + o10, G10 * ref[c]); }
        if (i11) { acc = __fmaf_rn(G11, ldg_f(s + o11), acc); atomicAdd(g + o11, G11 * ref[c]); }
        gref[c] = acc;
      }
    };
    for (int j = 0; j < p.D; ++j) {
      float ix, iy, z;
      project(p.k[j], a0, a1, a2, q0, q1, q2, ix, iy, z);
      clamp_pos(ix, iy, xmax, ymax);
      float fx = ix - cx, fy = iy - cy;
      if (!(fx >= 0.0f && fx < 1.0f && fy >= 0.0f && fy < 1.0f)) {
        flush();
        cx = floorf(ix);
        cy = floorf(iy);
        fx = ix - cx;
        fy = iy - cy;
        G00 = G01 = G10 = G11 = 0.f;
      }
      const float g = gs[(size_t)j * HW];
      const float wx1 = fx, wx0 = 1.0f - fx, wy1 = fy, wy0 = 1.0f - fy;
      G00 = __fmaf_rn(g, wx0 * wy0, G00);
      G01 = __fmaf_rn(g, wx1 * wy0, G01);
      G10 = __fmaf_rn(g, wx0 * wy1, G10);
      G11 = __fmaf_rn(g, wx1 * wy1, G11);
    }
    flush();
  }
#pragma unroll
  for (int c = 0; c < C; ++c) p.grad_ref[((size_t)b * C + c) * HW + n] = gref[c];
}

// g_score into the workspace (also the first launch of the tensor-core backward, cost_f_bwd_mma.cu)
cudaError_t launch_score_grad(const BwdParams& p, cudaStream_t st) {
  score_grad_kernel<<<dim3((p.HW + 127) / 128, p.B), 128, 0, st>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_cost_f_bwd(const BwdParams& p, cudaStream_t st, int* launches) {
  cudaError_t e = launch_score_grad(p, st);
  if (e != cudaSuccess) return e;
  dim3 grid((p.HW + 127) / 128, p.B);
  switch (p.C) {
    case 8: cost_f_bwd_kernel<8><<<grid, 128, 0, st>>>(p); break;
    case 16: cost_f_bwd_kernel<16><<<grid, 128, 0, st>>>(p); break;
    case 32: cost_f_bwd_kernel<32><<<grid, 128, 0, st>>>(p); break;
    case 64: cost_f_bwd_kernel<64><<<grid, 128, 0, st>>>(p); break;
    default: return cudaErrorInvalidValue;
  }
  *launches = 2;
  return cudaGetLastError();
}

}  // namespace magnet
