// MAGNET_VARIANT_DIRECT — one thread per output element, reference operation order.
//
// This is the plain fused formulation of homography.py:124-161: for every (b, j, pixel) and every
// valid view it projects, unnormalises exactly like grid_sample (align_corners=False), gathers the
// 4 bilinear taps of all C channels, forms the channel dot product, applies the consistency test
// and accumulates over views in fp64 (the reference's accidental `.double()`, homography.py:158).
// It never materialises a D x C x H x W tensor, but it shares nothing between hypotheses, so it is
// on-chip bound (4*C FMAs and 4*C gathers per hypothesis).  It exists as (1) the in-library
// cross-check for the tap-sharing kernel, (2) the fallback for channel counts the tap-sharing
// kernel is not instantiated for.
#include "common.cuh"
#include "launchers.h"

namespace magnet {

template <bool CW, bool IDX>
__global__ void __launch_bounds__(128)
cost_direct_kernel(const CostParams p, const int depth_mode, const int src_layout, const int C,
                   const int32_t* __restrict__ src_index) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= p.HW) return;
  const int j = blockIdx.y, b = blockIdx.z;
  const int H = p.H, W = p.W, HW = p.HW;

  float d;
  if (depth_mode == MAGNET_DEPTH_VOLUME) {
    d = p.d_volume[((size_t)b * p.D + j) * HW + n];
  } else if (depth_mode == MAGNET_DEPTH_GAUSS) {
    const float mu = p.ref_gmm[((size_t)b * 2 + 0) * HW + n];
    const float sg = p.ref_gmm[((size_t)b * 2 + 1) * HW + n];
    d = __fadd_rn(mu, __fmul_rn(sg, p.k[j]));          // MAGNET.py:155: mul, then add
  } else {
    d = p.k[j];
  }
  const float r0 = p.rays[((size_t)b * 3 + 0) * HW + n];
  const float r1 = p.rays[((size_t)b * 3 + 1) * HW + n];
  const float r2 = p.rays[((size_t)b * 3 + 2) * HW + n];
  const float* ref = p.ref_feat + (size_t)b * C * HW + n;
  const float uc = (float)W / 2.0f, vc = (float)H / 2.0f;

  double acc64 = 0.0;
  float acc32 = 0.0f;
  for (int v = 0; v < p.V; ++v) {
    const magnet_camera cam = p.cams[b * p.V + v];
    if (cam.valid != 1.0f) continue;
    const float q0 = __fmaf_rn(cam.A[2], r2, __fmaf_rn(cam.A[1], r1, __fmul_rn(cam.A[0], r0)));
    const float q1 = __fmaf_rn(cam.A[5], r2, __fmaf_rn(cam.A[4], r1, __fmul_rn(cam.A[3], r0)));
    const float q2 = __fmaf_rn(cam.A[8], r2, __fmaf_rn(cam.A[7], r1, __fmul_rn(cam.A[6], r0)));
    // homography.py:132-133
    const float P0 = __fadd_rn(cam.a[0], __fmul_rn(q0, d));
    const float P1 = __fadd_rn(cam.a[1], __fmul_rn(q1, d));
    const float P2 = __fadd_rn(cam.a[2], __fmul_rn(q2, d));   // == z_cam (homography.py:137-138)
    const float Zp = __fadd_rn(P2, 1e-10f);
    const float u = __fdiv_rn(P0, Zp), w = __fdiv_rn(P1, Zp);
    // :143-148
    float gx = __fdiv_rn(__fsub_rn(u, uc), uc);
    float gy = __fdiv_rn(__fsub_rn(w, vc), vc);
    if (gx > 10.0f) gx = 10.0f;
    if (gx < -10.0f) gx = -10.0f;
    if (gy > 10.0f) gy = 10.0f;
    if (gy < -10.0f) gy = -10.0f;
    // grid_sampler_unnormalize (align_corners=False)
    const float ix = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.0f), (float)W), 1.0f), 2.0f);
    const float iy = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.0f), (float)H), 1.0f), 2.0f);
    if (!(fabsf(ix) < 1e30f) || !(fabsf(iy) < 1e30f)) continue;   // NaN: every tap out of bounds
    const float x0f = floorf(ix), y0f = floorf(iy);
    const float x1f = x0f + 1.0f, y1f = y0f + 1.0f;
    const float w_nw = __fmul_rn(x1f - ix, y1f - iy), w_ne = __fmul_rn(ix - x0f, y1f - iy);
    const float w_sw = __fmul_rn(x1f - ix, iy - y0f), w_se = __fmul_rn(ix - x0f, iy - y0f);
    const int x0 = (int)x0f, y0 = (int)y0f, x1 = x0 + 1, y1 = y0 + 1;
    const bool in_nw = x0 >= 0 && x0 < W && y0 >= 0 && y0 < H;
    const bool in_ne = x1 >= 0 && x1 < W && y0 >= 0 && y0 < H;
    const bool in_sw = x0 >= 0 && x0 < W && y1 >= 0 && y1 < H;
    const bool in_se = x1 >= 0 && x1 < W && y1 >= 0 && y1 < H;
    const int vb = src_image<IDX>(src_index, b, v, p.B, p.V);    // view-major (homography.py:105) or the frame table
    float cost = 0.0f;
    if (in_nw | in_ne | in_sw | in_se) {
      if (src_layout == MAGNET_SRC_NCHW) {
        const float* src = p.src_feat + (size_t)vb * C * HW;
        const int o_nw = y0 * W + x0, o_ne = o_nw + 1, o_sw = o_nw + W, o_se = o_sw + 1;
        for (int c = 0; c < C; ++c) {
          const float* s = src + (size_t)c * HW;
          float f = 0.0f;
          if (in_nw) f = __fmaf_rn(ldg_f(s + o_nw), w_nw, f);
          if (in_ne) f = __fmaf_rn(ldg_f(s + o_ne), w_ne, f);
          if (in_sw) f = __fmaf_rn(ldg_f(s + o_sw), w_sw, f);
          if (in_se) f = __fmaf_rn(ldg_f(s + o_se), w_se, f);
          cost = __fadd_rn(cost, __fmul_rn(ldg_f(ref + (size_t)c * HW), f));
        }
      } else {
        const int XB = (W + 31) >> 5, C4 = C / 4;
        const float4* src = reinterpret_cast<const float4*>(p.src_feat) + (size_t)vb * H * XB * C4 * 32;
        // TILED32: pixel (y,x) quad c4 at ((y*XB + x/32)*C4 + c4)*32 + x%32
        const int o_nw = (y0 * XB + (x0 >> 5)) * C4 * 32 + (x0 & 31), o_ne = (y0 * XB + (x1 >> 5)) * C4 * 32 + (x1 & 31);
        const int o_sw = (y1 * XB + (x0 >> 5)) * C4 * 32 + (x0 & 31), o_se = (y1 * XB + (x1 >> 5)) * C4 * 32 + (x1 & 31);
        for (int c4 = 0; c4 < C4; ++c4) {
          const float4* s = src + c4 * 32;
          float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
          if (in_nw) { const float4 t = __ldg(s + o_nw); f.x = __fmaf_rn(t.x, w_nw, f.x); f.y = __fmaf_rn(t.y, w_nw, f.y); f.z = __fmaf_rn(t.z, w_nw, f.z); f.w = __fmaf_rn(t.w, w_nw, f.w); }
          if (in_ne) { const float4 t = __ldg(s + o_ne); f.x = __fmaf_rn(t.x, w_ne, f.x); f.y = __fmaf_rn(t.y, w_ne, f.y); f.z = __fmaf_rn(t.z, w_ne, f.z); f.w = __fmaf_rn(t.w, w_ne, f.w); }
          if (in_sw) { const float4 t = __ldg(s + o_sw); f.x = __fmaf_rn(t.x, w_sw, f.x); f.y = __fmaf_rn(t.y, w_sw, f.y); f.z = __fmaf_rn(t.z, w_sw, f.z); f.w = __fmaf_rn(t.w, w_sw, f.w); }
          if (in_se) { const float4 t = __ldg(s + o_se); f.x = __fmaf_rn(t.x, w_se, f.x); f.y = __fmaf_rn(t.y, w_se, f.y); f.z = __fmaf_rn(t.z, w_se, f.z); f.w = __fmaf_rn(t.w, w_se, f.w); }
          const float* rc = ref + (size_t)(4 * c4) * HW;
          cost = __fadd_rn(cost, __fmul_rn(ldg_f(rc), f.x));
          cost = __fadd_rn(cost, __fmul_rn(ldg_f(rc + HW), f.y));
          cost = __fadd_rn(cost, __fmul_rn(ldg_f(rc + 2 * (size_t)HW), f.z));
          cost = __fadd_rn(cost, __fmul_rn(ldg_f(rc + 3 * (size_t)HW), f.w));
        }
      }
    }
    if (CW) {
      const float* gm = p.src_gmm + (size_t)vb * 2 * HW;
      const float* gs = gm + HW;
      const int o_nw = y0 * W + x0, o_ne = o_nw + 1, o_sw = o_nw + W, o_se = o_sw + 1;
      float mu = 0.0f, sg = 0.0f;
      if (in_nw) { mu = __fmaf_rn(ldg_f(gm + o_nw), w_nw, mu); sg = __fmaf_rn(ldg_f(gs + o_nw), w_nw, sg); }
      if (in_ne) { mu = __fmaf_rn(ldg_f(gm + o_ne), w_ne, mu); sg = __fmaf_rn(ldg_f(gs + o_ne), w_ne, sg); }
      if (in_sw) { mu = __fmaf_rn(ldg_f(gm + o_sw), w_sw, mu); sg = __fmaf_rn(ldg_f(gs + o_sw), w_sw, sg); }
      if (in_se) { mu = __fmaf_rn(ldg_f(gm + o_se), w_se, mu); sg = __fmaf_rn(ldg_f(gs + o_se), w_se, sg); }
      // homography.py:157-159: strict '<', fp64 product and accumulation
      const bool keep = fabsf(__fsub_rn(P2, mu)) < __fmul_rn(sg, p.kappa);
      acc64 += keep ? (double)cost : 0.0;
    } else {
      acc32 = __fadd_rn(acc32, cost);                              // homography.py:41 (fp32)
    }
  }
  const float s = CW ? (float)acc64 : acc32;                       // :118 store rounds to fp32
  p.out[((size_t)b * p.D + j) * HW + n] = __fdiv_rn(s, p.vf);      // :120 / float(n_views)
}

// softmax over the D planes, in place (homography.py:46), after any cost-volume forward that asks for it
__global__ void softmax_planes_kernel(float* __restrict__ vol, int D, int HW) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= HW) return;
  float* col = vol + (size_t)blockIdx.y * D * HW + n;
  float m = -INFINITY;
  for (int j = 0; j < D; ++j) m = fmaxf(m, col[(size_t)j * HW]);
  float s = 0.0f;
  for (int j = 0; j < D; ++j) s += expf(col[(size_t)j * HW] - m);
  for (int j = 0; j < D; ++j) col[(size_t)j * HW] = __fdiv_rn(expf(col[(size_t)j * HW] - m), s);
}

cudaError_t launch_softmax_planes(float* vol, int B, int D, int HW, cudaStream_t st) {
  softmax_planes_kernel<<<dim3((HW + 127) / 128, B), 128, 0, st>>>(vol, D, HW);
  return cudaGetLastError();
}

cudaError_t launch_cost_direct(const CostParams& p, int depth_mode, int src_layout, int C, bool cw,
                               const int32_t* src_index, cudaStream_t st, int* launches) {
  *launches = 1;
  return dispatch(
      [&](auto w, auto idx) {
        cost_direct_kernel<w, idx><<<dim3((p.HW + 127) / 128, p.D, p.B), 128, 0, st>>>(p, depth_mode, src_layout, C,
                                                                                       src_index);
        return cudaGetLastError();
      },
      Flag{cw}, Flag{src_index != nullptr});
}

}  // namespace magnet
