// Backward of the consistency-weighted cost volume (homography.est_costvolume_CW, homography.py:79-161) w.r.t. both
// feature maps and the depth hypotheses, on the CUDA cores.
//
//   out[b,j,p] = 1/V sum_v m(b,v,j,p) sum_t w_t <ref[b,:,p], src_v[:, tap_t]>        (m: consistency mask, 0 / 1)
//   g_score    = grad_out / V                                                           (kernel 1, score_grad_kernel)
//   grad_ref[b,c,p]   = sum_{v,j,t} g_score m w_t src_v[c, tap_t]                       (kernel 2, registers)
//   grad_src[v,c,tap] += sum_{p,j: tap_t = tap} g_score m w_t ref[b,c,p]                 (kernel 2, atomics)
//   grad_d[b,j,p]     = sum_v g_score m (dcost/dix du/dd + dcost/diy dv/dd)             (kernel 2)
// with dcost/dix the derivative of the bilinear interpolant of the four per-cell dot products f_t = <ref_p, src_t> and
// du/dd = (q0 Zp - P0 q2) / Zp^2 (likewise v).  The mask is piecewise constant: the source Gaussians get no gradient.
// In MAGNET_DEPTH_GAUSS mode d_j = mu + sigma k_j, so grad_mu = sum_j grad_d_j and grad_sigma = sum_j k_j grad_d_j.
//
// The mask must be the one the forward applied, bit for bit, or a gradient would flow through a hypothesis the forward
// dropped.  MASK selects the arithmetic of the forward kernel that produced the volume:
//   MASK_MMA    — cost_mma.cu (tensor cores, SPLIT16 forward): the position of common.cuh/cells_common.cuh project(),
//                 clamped, and the helpers of cw_mask.cuh, which cost_mma.cu calls as well;
//   MASK_DIRECT — cost_direct.cu (the reference's operation order: IEEE divisions, +-10 grid clamp, fma chain over
//                 the in-image taps).
// The tap-sharing kernels (cells / TMA) walk cells analytically and interpolate with a polynomial; their mask is not
// reproduced here, so a differentiable forward never runs on them.
//
// Tap sharing as in cost_f_bwd.cu: consecutive hypotheses of one pixel that fall into the same bilinear cell are reduced
// to 4 corner coefficients G_t before the C channels are touched.  Four lanes per (b, pixel); any hypothesis order.
// After a tensor-core forward the feature gradients come from the tensor-core kernel on the forward's split buffers
// (cost_f_bwd_mma.cu, same mask helpers) and this kernel computes the depth gradient only.
//
// Camera gradients (GEOM, DESIGN §3.11): the same walk takes the position derivative one step further.  With
// gx = g m dcost/dix, gy = g m dcost/diy, P = a + q d (q = A r), Zp = P2 + 1e-10, u = P0/Zp, w = P1/Zp:
//   g_P = (gx, gy, -(gx u + gy w)) / Zp;   grad_a[b,v] = sum_{p,j} g_P;   grad_A[b,v] = sum_p (sum_j g_P d_j) r_p^T;
//   grad_ray[b,:,p] = sum_v A_v^T sum_j g_P d_j.
// Per (pixel, view) 6 accumulators, per pixel 3 ray accumulators; per view each block reduces its pixels' 12-vectors
// in a fixed order into a caller-owned workspace, and geom_reduce_kernel adds the blocks in a fixed order: no atomics,
// bit-identical from run to run.  MAGNET_DEPTH_PLANES (the F volume, no mask) uses the position arithmetic of project().
// The GEOM flag sits on the shared body so that the existing kernels keep their parameter block and their code.
#include "cells_common.cuh"
#include "cw_mask.cuh"
#include "launchers.h"

namespace magnet {

constexpr int MASK_MMA = 0, MASK_DIRECT = 1;

// Four lanes per (b, pixel): lane q of the quad holds channels [q*CPL, q*CPL + CPL) of ref and grad_ref (channels >= C
// are idle), so at C = 64 a thread keeps 2 x 16 channel values instead of 2 x 64.  The four lanes walk the same
// hypotheses with the same data, hence in lockstep; the per-cell dot products are reduced across the quad by shuffles.
// Outputs of a GEOM launch: per-block partials [(b*V + v)*12 + k][block] and the ray gradient (B,3,HW) or NULL.
struct GeomOut {
  float* __restrict__ partials;
  float* __restrict__ grad_rays;
};

template <int CPL, int MODE, int MASK, bool GEOM>
__device__ __forceinline__ void cw_bwd_body(const CwBwdParams& p, const int C, const GeomOut* go) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int n0 = t >> 2, q = t & 3;
  // whole quads leave together (HW quads per row of blocks); a GEOM block keeps them for its per-view reductions,
  // walking the last pixel again without writing anything
  if (!GEOM && n0 >= p.HW) return;
  const bool active = n0 < p.HW;
  const int n = GEOM && !active ? p.HW - 1 : n0;
  const unsigned qmask = 0xfu << (threadIdx.x & 28);
  const int b = blockIdx.y, H = p.H, W = p.W, HW = p.HW, D = p.D;
  const bool need_ref = !GEOM && p.grad_ref != nullptr, need_src = !GEOM && p.grad_src != nullptr;
  const bool need_d = p.grad_depth != nullptr;
  const int c0 = q * CPL;
  float ref[CPL], gref[CPL];
#pragma unroll
  for (int i = 0; i < CPL; ++i) {
    ref[i] = c0 + i < C ? ldg_f(p.ref_feat + ((size_t)b * C + c0 + i) * HW + n) : 0.0f;
    gref[i] = 0.0f;
  }
  const float r0 = ldg_f(p.rays + ((size_t)b * 3 + 0) * HW + n);
  const float r1 = ldg_f(p.rays + ((size_t)b * 3 + 1) * HW + n);
  const float r2 = ldg_f(p.rays + ((size_t)b * 3 + 2) * HW + n);
  const float* gs = p.g_score + (size_t)b * D * HW + n;
  float mu_p = 0.0f, sg_p = 0.0f, g_mu = 0.0f, g_sg = 0.0f;
  if (MODE == MAGNET_DEPTH_GAUSS) {
    mu_p = ldg_f(p.ref_gmm + ((size_t)b * 2 + 0) * HW + n);
    sg_p = ldg_f(p.ref_gmm + ((size_t)b * 2 + 1) * HW + n);
  }
  float* gd = p.grad_depth + (size_t)b * D * HW + n;       // VOLUME: this pixel's column, accumulated over the views
  const bool writer = GEOM ? q == 0 && active : q == 0;   // lane 0 of the quad owns the depth gradient
  if (MODE == MAGNET_DEPTH_VOLUME && need_d && writer)
    for (int j = 0; j < D; ++j) gd[(size_t)j * HW] = 0.0f;
  const float xmax = (float)W + 1.0f, ymax = (float)H + 1.0f;
  const float uc = (float)W / 2.0f, vc = (float)H / 2.0f;
  float gr0 = 0.f, gr1 = 0.f, gr2 = 0.f;                  // GEOM: the ray gradient, summed over the views

  for (int v = 0; v < p.V; ++v) {
    const magnet_camera* cam = p.cams + (b * p.V + v);
    if (cam->valid != 1.0f) continue;
    const float a0 = cam->a[0], a1 = cam->a[1], a2 = cam->a[2];
    const float q0 = __fmaf_rn(cam->A[2], r2, __fmaf_rn(cam->A[1], r1, __fmul_rn(cam->A[0], r0)));
    const float q1 = __fmaf_rn(cam->A[5], r2, __fmaf_rn(cam->A[4], r1, __fmul_rn(cam->A[3], r0)));
    const float q2 = __fmaf_rn(cam->A[8], r2, __fmaf_rn(cam->A[7], r1, __fmul_rn(cam->A[6], r0)));
    const int vb = v * p.B + b;
    const float* src = p.src_feat + ((size_t)vb * C + c0) * HW;
    const float* gm = p.src_gmm + (size_t)vb * 2 * HW;
    float* gsrc = need_src ? p.grad_src + ((size_t)vb * C + c0) * HW : nullptr;
    float sa0 = 0.f, sa1 = 0.f, sa2 = 0.f, sd0 = 0.f, sd1 = 0.f, sd2 = 0.f;   // GEOM: sum_j g_P, sum_j g_P d_j

    // the current cell: origin, which taps are inside, their (mu, sigma), their dot products, the coefficients G_t
    float cx = -1e30f, cy = -1e30f;
    bool i00 = false, i01 = false, i10 = false, i11 = false;
    int o00 = 0;
    float m00 = 0.f, m01 = 0.f, m10 = 0.f, m11 = 0.f, s00 = 0.f, s01 = 0.f, s10 = 0.f, s11 = 0.f;
    float f00 = 0.f, f01 = 0.f, f10 = 0.f, f11 = 0.f;
    float G00 = 0.f, G01 = 0.f, G10 = 0.f, G11 = 0.f;
    auto flush = [&]() {
      if (!(i00 | i01 | i10 | i11)) return;
      if (G00 == 0.f && G01 == 0.f && G10 == 0.f && G11 == 0.f) return;
      if (!need_ref && !need_src) return;
      const int o01 = o00 + 1, o10 = o00 + W, o11 = o10 + 1;
#pragma unroll
      for (int i = 0; i < CPL; ++i) {
        if (c0 + i >= C) break;
        const float* s = src + (size_t)i * HW;
        if (need_ref) {
          float acc = gref[i];
          if (i00) acc = __fmaf_rn(G00, ldg_f(s + o00), acc);
          if (i01) acc = __fmaf_rn(G01, ldg_f(s + o01), acc);
          if (i10) acc = __fmaf_rn(G10, ldg_f(s + o10), acc);
          if (i11) acc = __fmaf_rn(G11, ldg_f(s + o11), acc);
          gref[i] = acc;
        }
        if (need_src) {
          float* g = gsrc + (size_t)i * HW;
          if (i00) atomicAdd(g + o00, G00 * ref[i]);
          if (i01) atomicAdd(g + o01, G01 * ref[i]);
          if (i10) atomicAdd(g + o10, G10 * ref[i]);
          if (i11) atomicAdd(g + o11, G11 * ref[i]);
        }
      }
    };
    auto open = [&](float nx, float ny) {
      cx = nx;
      cy = ny;
      const int x0 = (int)nx, y0 = (int)ny, x1 = x0 + 1, y1 = y0 + 1;
      i00 = x0 >= 0 && x0 < W && y0 >= 0 && y0 < H; i01 = x1 >= 0 && x1 < W && y0 >= 0 && y0 < H;
      i10 = x0 >= 0 && x0 < W && y1 >= 0 && y1 < H; i11 = x1 >= 0 && x1 < W && y1 >= 0 && y1 < H;
      o00 = y0 * W + x0;
      const int o01 = o00 + 1, o10 = o00 + W, o11 = o10 + 1;
      if (p.cw) {                                         // without consistency src_gmm may be NULL (the C ABI allows it)
        m00 = i00 ? ldg_f(gm + o00) : 0.f; s00 = i00 ? ldg_f(gm + HW + o00) : 0.f;
        m01 = i01 ? ldg_f(gm + o01) : 0.f; s01 = i01 ? ldg_f(gm + HW + o01) : 0.f;
        m10 = i10 ? ldg_f(gm + o10) : 0.f; s10 = i10 ? ldg_f(gm + HW + o10) : 0.f;
        m11 = i11 ? ldg_f(gm + o11) : 0.f; s11 = i11 ? ldg_f(gm + HW + o11) : 0.f;
      }
      f00 = f01 = f10 = f11 = 0.f;
      if ((need_d || GEOM) && (i00 | i01 | i10 | i11)) {
#pragma unroll
        for (int i = 0; i < CPL; ++i) {
          if (c0 + i >= C) break;
          const float* s = src + (size_t)i * HW;
          if (i00) f00 = __fmaf_rn(ref[i], ldg_f(s + o00), f00);
          if (i01) f01 = __fmaf_rn(ref[i], ldg_f(s + o01), f01);
          if (i10) f10 = __fmaf_rn(ref[i], ldg_f(s + o10), f10);
          if (i11) f11 = __fmaf_rn(ref[i], ldg_f(s + o11), f11);
        }
#pragma unroll
        for (int m = 1; m < 4; m <<= 1) {                 // quad butterfly: every lane ends with the full sums
          f00 += __shfl_xor_sync(qmask, f00, m, 4);
          f01 += __shfl_xor_sync(qmask, f01, m, 4);
          f10 += __shfl_xor_sync(qmask, f10, m, 4);
          f11 += __shfl_xor_sync(qmask, f11, m, 4);
        }
      }
      G00 = G01 = G10 = G11 = 0.f;
    };

    for (int j = 0; j < D; ++j) {
      float d;
      if (MODE == MAGNET_DEPTH_VOLUME) d = ldg_f(p.d_volume + ((size_t)b * D + j) * HW + n);
      else if (MODE == MAGNET_DEPTH_PLANES) d = p.k[j];
      else d = __fadd_rn(mu_p, __fmul_rn(sg_p, p.k[j]));  // MAGNET.py:155: mul, then add
      // sample position, source depth z, du/dd, dv/dd in the forward kernel's arithmetic
      float ix, iy, z, dudd, dvdd;
      float u_g = 0.f, w_g = 0.f, rz_g = 0.f;             // GEOM: u, w, 1/Zp
      bool clx = false, cly = false;                      // GEOM, DIRECT: the axis hit the +-10 clamp
      if (MASK == MASK_MMA) {
        project(d, a0, a1, a2, q0, q1, q2, ix, iy, z);    // element by element == project2 of cost_mma.cu
        ix = clamp_coord(ix, xmax);
        iy = clamp_coord(iy, ymax);
        const float r = rcp_nr(__fadd_rn(z, 1e-10f));
        dudd = (q0 - __fmaf_rn(q0, d, a0) * r * q2) * r;
        dvdd = (q1 - __fmaf_rn(q1, d, a1) * r * q2) * r;
        if (GEOM) {
          u_g = __fmaf_rn(q0, d, a0) * r;
          w_g = __fmaf_rn(q1, d, a1) * r;
          rz_g = r;
        }
      } else {                                            // cost_direct.cu, homography.py:132-148
        const float P0 = __fadd_rn(a0, __fmul_rn(q0, d));
        const float P1 = __fadd_rn(a1, __fmul_rn(q1, d));
        z = __fadd_rn(a2, __fmul_rn(q2, d));
        const float Zp = __fadd_rn(z, 1e-10f);
        const float u = __fdiv_rn(P0, Zp), w = __fdiv_rn(P1, Zp);
        float gx = __fdiv_rn(__fsub_rn(u, uc), uc);
        float gy = __fdiv_rn(__fsub_rn(w, vc), vc);
        dudd = (q0 - u * q2) / Zp;
        dvdd = (q1 - w * q2) / Zp;
        if (GEOM) {
          u_g = u;
          w_g = w;
          rz_g = __fdiv_rn(1.0f, Zp);
          clx = !(fabsf(gx) <= 10.0f);
          cly = !(fabsf(gy) <= 10.0f);
        }
        if (gx > 10.0f) { gx = 10.0f; dudd = 0.0f; }      // the masked assignment passes no gradient
        if (gx < -10.0f) { gx = -10.0f; dudd = 0.0f; }
        if (gy > 10.0f) { gy = 10.0f; dvdd = 0.0f; }
        if (gy < -10.0f) { gy = -10.0f; dvdd = 0.0f; }
        ix = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.0f), (float)W), 1.0f), 2.0f);
        iy = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.0f), (float)H), 1.0f), 2.0f);
        if (!(fabsf(ix) < 1e30f) || !(fabsf(iy) < 1e30f)) continue;   // NaN: every tap out of bounds
      }
      float x0f, y0f, fx, fy;
      cell_split(ix, x0f, fx);
      cell_split(iy, y0f, fy);
      if (x0f != cx || y0f != cy) {
        flush();
        open(x0f, y0f);
      }
      if (!(i00 | i01 | i10 | i11)) continue;             // no tap inside: no cost, no gradient (and mu~ = sigma~ = 0)
      bool keep = true;
      if (p.cw) {
        if (MASK == MASK_MMA) {
          keep = cw_keep(z, make_float2(lerp2d(m00, m01, m10, m11, fx, fy), lerp2d(s00, s01, s10, s11, fx, fy)), p.kappa);
        } else {                                          // cost_direct.cu: weights, fma chain over the in-image taps
          const float x1f = x0f + 1.0f, y1f = y0f + 1.0f;
          const float w_nw = __fmul_rn(x1f - ix, y1f - iy), w_ne = __fmul_rn(ix - x0f, y1f - iy);
          const float w_sw = __fmul_rn(x1f - ix, iy - y0f), w_se = __fmul_rn(ix - x0f, iy - y0f);
          float mu = 0.0f, sg = 0.0f;
          if (i00) { mu = __fmaf_rn(m00, w_nw, mu); sg = __fmaf_rn(s00, w_nw, sg); }
          if (i01) { mu = __fmaf_rn(m01, w_ne, mu); sg = __fmaf_rn(s01, w_ne, sg); }
          if (i10) { mu = __fmaf_rn(m10, w_sw, mu); sg = __fmaf_rn(s10, w_sw, sg); }
          if (i11) { mu = __fmaf_rn(m11, w_se, mu); sg = __fmaf_rn(s11, w_se, sg); }
          keep = fabsf(__fsub_rn(z, mu)) < __fmul_rn(sg, p.kappa);
        }
      }
      if (!keep) continue;
      const float g = gs[(size_t)j * HW];
      const float wx1 = fx, wx0 = 1.0f - fx, wy1 = fy, wy0 = 1.0f - fy;
      G00 = __fmaf_rn(g, wx0 * wy0, G00);
      G01 = __fmaf_rn(g, wx1 * wy0, G01);
      G10 = __fmaf_rn(g, wx0 * wy1, G10);
      G11 = __fmaf_rn(g, wx1 * wy1, G11);
      if (need_d) {
        const float dcdx = (f01 - f00) * wy0 + (f11 - f10) * wy1;
        const float dcdy = (f10 - f00) * wx0 + (f11 - f01) * wx1;
        const float gdv = g * (dcdx * dudd + dcdy * dvdd);
        if (MODE == MAGNET_DEPTH_VOLUME) {
          if (writer) gd[(size_t)j * HW] += gdv;
        } else {
          g_mu += gdv;
          g_sg = __fmaf_rn(p.k[j], gdv, g_sg);
        }
      }
      if (GEOM) {                                         // kept apart so that the block above compiles as before
        const float dcdx = (f01 - f00) * wy0 + (f11 - f10) * wy1;     // the same values as above
        const float dcdy = (f10 - f00) * wx0 + (f11 - f01) * wx1;
        const float gx = clx ? 0.f : __fmul_rn(g, dcdx), gy = cly ? 0.f : __fmul_rn(g, dcdy);
        const float gp0 = __fmul_rn(gx, rz_g), gp1 = __fmul_rn(gy, rz_g);
        const float gp2 = -__fmul_rn(__fmaf_rn(gy, w_g, __fmul_rn(gx, u_g)), rz_g);
        sa0 = __fadd_rn(sa0, gp0); sa1 = __fadd_rn(sa1, gp1); sa2 = __fadd_rn(sa2, gp2);
        sd0 = __fmaf_rn(gp0, d, sd0); sd1 = __fmaf_rn(gp1, d, sd1); sd2 = __fmaf_rn(gp2, d, sd2);
      }
    }
    flush();
    if (GEOM) {
      // ray gradient A^T h, h = sum_j g_P d_j
      gr0 = __fmaf_rn(cam->A[6], sd2, __fmaf_rn(cam->A[3], sd1, __fmaf_rn(cam->A[0], sd0, gr0)));
      gr1 = __fmaf_rn(cam->A[7], sd2, __fmaf_rn(cam->A[4], sd1, __fmaf_rn(cam->A[1], sd0, gr1)));
      gr2 = __fmaf_rn(cam->A[8], sd2, __fmaf_rn(cam->A[5], sd1, __fmaf_rn(cam->A[2], sd0, gr2)));
      // this pixel's 12-vector (A row-major: h_i r_k, then a: sum_j g_P), owner lanes only, reduced over the block
      __shared__ float red[4][12];
      float c[12] = {sd0 * r0, sd0 * r1, sd0 * r2, sd1 * r0, sd1 * r1, sd1 * r2, sd2 * r0, sd2 * r1, sd2 * r2,
                     sa0, sa1, sa2};
#pragma unroll
      for (int k = 0; k < 12; ++k) {
        c[k] = writer ? c[k] : 0.0f;                      // lanes 0, 4, .., 28 hold the warp's pixels
#pragma unroll
        for (int m = 16; m >= 4; m >>= 1) c[k] = __fadd_rn(c[k], __shfl_xor_sync(0xffffffffu, c[k], m));
      }
      if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 12; ++k) red[threadIdx.x >> 5][k] = c[k];
      }
      __syncthreads();
      if (threadIdx.x < 12) {
        const float s = __fadd_rn(__fadd_rn(red[0][threadIdx.x], red[1][threadIdx.x]),
                                  __fadd_rn(red[2][threadIdx.x], red[3][threadIdx.x]));
        go->partials[((size_t)(b * p.V + v) * 12 + threadIdx.x) * gridDim.x + blockIdx.x] = s;
      }
      __syncthreads();
    }
  }
  if (GEOM && writer && go->grad_rays != nullptr) {
    go->grad_rays[((size_t)b * 3 + 0) * HW + n] = gr0;
    go->grad_rays[((size_t)b * 3 + 1) * HW + n] = gr1;
    go->grad_rays[((size_t)b * 3 + 2) * HW + n] = gr2;
  }
  if (need_ref) {
#pragma unroll
    for (int i = 0; i < CPL; ++i)
      if (c0 + i < C) p.grad_ref[((size_t)b * C + c0 + i) * HW + n] = gref[i];
  }
  if (MODE == MAGNET_DEPTH_GAUSS && need_d && writer) {
    p.grad_depth[((size_t)b * 2 + 0) * HW + n] = g_mu;
    p.grad_depth[((size_t)b * 2 + 1) * HW + n] = g_sg;
  }
}

template <int CPL, int MODE, int MASK>
__global__ void __launch_bounds__(128)
cost_cw_bwd_kernel(const __grid_constant__ CwBwdParams p, const int C) {
  cw_bwd_body<CPL, MODE, MASK, false>(p, C, nullptr);
}

template <int CPL, int MODE, int MASK>
__global__ void __launch_bounds__(128)
cost_geom_bwd_kernel(const __grid_constant__ CwBwdParams p, const int C, const __grid_constant__ GeomOut go) {
  cw_bwd_body<CPL, MODE, MASK, true>(p, C, &go);
}

// grad_cams[bv, k] = sum over the blocks of the partials, in a fixed order: warp k, lane l adds blocks l, l + 32, ...,
// then a butterfly over the lanes.  Zero for an invalid view (its partials were never written).
__global__ void __launch_bounds__(384)
geom_reduce_kernel(const float* __restrict__ partials, const magnet_camera* __restrict__ cams, int nblk,
                   float* __restrict__ grad_cams) {
  const int bv = blockIdx.x, k = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float s = 0.0f;
  if (cams[bv].valid == 1.0f) {
    const float* src = partials + ((size_t)bv * 12 + k) * nblk;
    for (int i = lane; i < nblk; i += 32) s = __fadd_rn(s, src[i]);
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, m));
  }
  if (lane == 0) grad_cams[(size_t)bv * 12 + k] = s;
}

bool cw_bwd_supports(int C) { return C >= 1 && C <= 64; }

size_t geom_workspace_bytes(int B, int V, int H, int W) {
  const size_t nblk = ((size_t)H * W + 31) / 32;               // 32 pixels (128 threads, 4 lanes each) per block
  return (size_t)B * V * 12 * nblk * sizeof(float);
}

// channels per lane of C <= 64 channels (4 lanes per pixel)
static Choice<int, 1, 2, 4, 8, 16> channels_per_lane(int C) {
  return {C <= 4 ? 1 : C <= 8 ? 2 : C <= 16 ? 4 : C <= 32 ? 8 : C <= 64 ? 16 : 0};
}
using Mask = Choice<int, MASK_MMA, MASK_DIRECT>;

// Camera (and optionally ray and depth) gradients: g_score (softmax or not) into p.g_score, the GEOM walk with
// per-block partials into `partials`, then the fixed-order reduction into grad_cams (B*V, 12).  Three launches.
cudaError_t launch_cost_geom_bwd(const CwBwdParams& p, int C, int mode, bool mask_mma, int softmax, const float* prob,
                                 const float* grad_out, float* partials, float* grad_rays, float* grad_cams,
                                 cudaStream_t st, int* launches) {
  BwdParams s;
  s.B = p.B; s.V = p.V; s.D = p.D; s.C = C; s.H = p.H; s.W = p.W; s.HW = p.HW;
  s.softmax = softmax;
  s.vf = (float)p.V;
  s.ref_feat = s.src_feat = s.rays = nullptr;
  s.cams = nullptr;
  s.prob = prob;
  s.grad_out = grad_out;
  s.g_score = const_cast<float*>(p.g_score);
  s.grad_ref = s.grad_src = nullptr;
  cudaError_t e = launch_score_grad(s, st);
  if (e != cudaSuccess) return e;
  GeomOut go;
  go.partials = partials;
  go.grad_rays = grad_rays;
  const dim3 grid((4 * p.HW + 127) / 128, p.B);
  const int mask = mask_mma || mode == MAGNET_DEPTH_PLANES ? MASK_MMA : MASK_DIRECT;
  e = dispatch(
      [&](auto cpl, auto m, auto k) -> cudaError_t {
        // the F volume (PLANES) has no mask: its positions are the tensor-core forward's
        if constexpr (m == MAGNET_DEPTH_PLANES && k != MASK_MMA) {
          return cudaErrorInvalidValue;
        } else {
          cost_geom_bwd_kernel<cpl, m, k><<<grid, 128, 0, st>>>(p, C, go);
          return cudaGetLastError();
        }
      },
      channels_per_lane(C), DepthMode{mode}, Mask{mask});
  if (e != cudaSuccess) return e;
  geom_reduce_kernel<<<p.B * p.V, 384, 0, st>>>(partials, p.cams, (int)grid.x, grad_cams);
  *launches = 3;
  return cudaGetLastError();
}

// p: NCHW maps (CUDA-core kernel).  split: the same call with ref_feat / src_feat pointing to the forward's SPLIT16
// or HALF16 buffers (split_layout), or NULL.  With split, both feature gradients come from the tensor-core kernel and the CUDA-core kernel only
// computes the depth gradient; otherwise the CUDA-core kernel computes everything that is requested.  mask_mma:
// reproduce the mask of the tensor-core forward (else of the DIRECT forward).  First of all g_score = grad_out / V goes
// to the workspace (score_grad_kernel with softmax = 0).
cudaError_t launch_cost_cw_bwd(const CwBwdParams& p, const CwBwdParams* split, int split_layout, int C, int mode,
                               bool mask_mma, const float* grad_out, cudaStream_t st, int* launches) {
  BwdParams s;
  s.B = p.B; s.V = p.V; s.D = p.D; s.C = C; s.H = p.H; s.W = p.W; s.HW = p.HW;
  s.softmax = 0;
  s.vf = (float)p.V;
  s.ref_feat = s.src_feat = s.rays = s.prob = nullptr;
  s.cams = nullptr;
  s.grad_out = grad_out;
  s.g_score = const_cast<float*>(p.g_score);
  s.grad_ref = s.grad_src = nullptr;
  cudaError_t e = launch_score_grad(s, st);
  if (e != cudaSuccess) return e;
  *launches = 1;
  CwBwdParams cc = p;
  if (split != nullptr) {
    if (split->grad_ref != nullptr || split->grad_src != nullptr) {
      if ((e = launch_cost_cw_bwd_mma(*split, mode, split_layout, st)) != cudaSuccess) return e;
      ++*launches;
    }
    cc.grad_ref = cc.grad_src = nullptr;
  }
  if (cc.grad_ref == nullptr && cc.grad_src == nullptr && cc.grad_depth == nullptr) return cudaSuccess;
  const dim3 grid((4 * p.HW + 127) / 128, p.B);
  e = dispatch(
      [&](auto cpl, auto m, auto k) {
        cost_cw_bwd_kernel<cpl, m, k><<<grid, 128, 0, st>>>(cc, C);
        return cudaGetLastError();
      },
      channels_per_lane(C), Choice<int, MAGNET_DEPTH_VOLUME, MAGNET_DEPTH_GAUSS>{mode},
      Mask{mask_mma ? MASK_MMA : MASK_DIRECT});
  if (e == cudaSuccess) ++*launches;
  return e;
}

}  // namespace magnet
