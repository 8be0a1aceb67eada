// Device helpers shared by the tap-sharing kernels (cost_cells.cu: taps gathered from global memory;
// cost_window.cu: taps gathered from a shared-memory copy of the CTA's source window).
#pragma once
#include "common.cuh"

namespace magnet {

template <int MODE>
struct DepthSrc {
  float mu, sg;
  const float* dv;   // d_volume + b*D*HW + n
  int HW;
};

template <int MODE>
__device__ __forceinline__ float depth_of(const CostParams& p, const DepthSrc<MODE>& ds, int j) {
  if (MODE == MAGNET_DEPTH_VOLUME) return ldg_f(ds.dv + (size_t)j * ds.HW);
  if (MODE == MAGNET_DEPTH_GAUSS) return __fadd_rn(ds.mu, __fmul_rn(ds.sg, p.k[j]));   // MAGNET.py:155: mul, then add
  return p.k[j];
}

// Projection at depth d: continuous source-image sample position (ix, iy) = projected pixel - 0.5
// (SURVEY A.2 / A.5 #1) and z = depth in the source camera (exactly the reference's mul-then-add).
__device__ __forceinline__ void project(float d, float a0, float a1, float a2, float q0, float q1, float q2,
                                        float& ix, float& iy, float& z) {
  const float P0 = __fmaf_rn(q0, d, a0);
  const float P1 = __fmaf_rn(q1, d, a1);
  z = __fadd_rn(a2, __fmul_rn(q2, d));
  const float r = rcp_nr(__fadd_rn(z, 1e-10f));
  ix = __fmaf_rn(P0, r, -0.5f);
  iy = __fmaf_rn(P1, r, -0.5f);
}

// Anything left of -1 / right of W (above / below likewise) has all four taps out of bounds: clamp so
// that cell coordinates stay small and NaN (fmaxf drops it) maps to "out of bounds" (exact walk only).
__device__ __forceinline__ void clamp_pos(float& ix, float& iy, float xmax, float ymax) {
  ix = fminf(fmaxf(ix, -2.0f), xmax);
  iy = fminf(fmaxf(iy, -2.0f), ymax);
}

struct Tap {
  float f, m, s;   // <ref, src>, source mu, source sigma at one integer source pixel (0 when outside)
};

// <ref, src[tap]> over C channels: C/4 LDG.128 at immediate offsets from one address, two FMA chains (even / odd channels).
template <int C>
__device__ __forceinline__ float tap_dot(const float4* __restrict__ s, const float2 (&ref2)[C / 2]) {
  float2 s0 = make_float2(0.f, 0.f), s1 = make_float2(0.f, 0.f);
#pragma unroll
  for (int c4 = 0; c4 < C / 4; ++c4) {
    const float4 t = __ldg(s + c4 * 32);
    s0 = ffma2_rn(ref2[2 * c4 + 0], make_float2(t.x, t.y), s0);
    s1 = ffma2_rn(ref2[2 * c4 + 1], make_float2(t.z, t.w), s1);
  }
  return (s0.x + s0.y) + (s1.x + s1.y);
}


// Two dot products <ref, src[tapA]>, <ref, src[tapB]> at once, loads issued in batches of 2 x QB channel quads
// before their FMAs so that 2*QB LDG.128 per lane are in flight (the gathers mostly miss L1).
template <int C, int QB>
__device__ __forceinline__ void tap_dot2(const float4* __restrict__ sa, const float4* __restrict__ sb,
                                         const float2 (&ref2)[C / 2], float& fa, float& fb) {
  float2 a0 = make_float2(0.f, 0.f), a1 = a0, b0 = a0, b1 = a0;
#pragma unroll
  for (int q0 = 0; q0 < C / 4; q0 += QB) {
    float4 ta[QB], tb[QB];
#pragma unroll
    for (int q = 0; q < QB; ++q) {
      ta[q] = __ldg(sa + (q0 + q) * 32);
      tb[q] = __ldg(sb + (q0 + q) * 32);
    }
#pragma unroll
    for (int q = 0; q < QB; ++q) {
      a0 = ffma2_rn(ref2[2 * (q0 + q) + 0], make_float2(ta[q].x, ta[q].y), a0);
      a1 = ffma2_rn(ref2[2 * (q0 + q) + 1], make_float2(ta[q].z, ta[q].w), a1);
      b0 = ffma2_rn(ref2[2 * (q0 + q) + 0], make_float2(tb[q].x, tb[q].y), b0);
      b1 = ffma2_rn(ref2[2 * (q0 + q) + 1], make_float2(tb[q].z, tb[q].w), b1);
    }
  }
  fa = (a0.x + a0.y) + (a1.x + a1.y);
  fb = (b0.x + b0.y) + (b1.x + b1.y);
}

// Two taps at once (see load_tap for the clamping convention).
template <int C, bool CW>
__device__ __forceinline__ void load_tap2(const float4* __restrict__ src_img, const float* __restrict__ gm,
                                          const float2 (&ref2)[C / 2], int xa, int ya, int xb, int yb, int W, int H,
                                          int XB, int HW, Tap& ta, Tap& tb) {
  const bool ina = xa >= 0 && xa < W && ya >= 0 && ya < H, inb = xb >= 0 && xb < W && yb >= 0 && yb < H;
  const int xac = min(max(xa, 0), W - 1), yac = min(max(ya, 0), H - 1);
  const int xbc = min(max(xb, 0), W - 1), ybc = min(max(yb, 0), H - 1);
  float ma = 0.f, sga = 0.f, mb = 0.f, sgb = 0.f;
  if (CW) {
    ma = ldg_f(gm + yac * W + xac); sga = ldg_f(gm + HW + yac * W + xac);
    mb = ldg_f(gm + ybc * W + xbc); sgb = ldg_f(gm + HW + ybc * W + xbc);
  }
  float fa, fb;
  tap_dot2<C, (C / 4 < 8 ? C / 4 : 8)>(src_img + ((yac * XB + (xac >> 5)) * (C / 4) * 32 + (xac & 31)),
                                       src_img + ((ybc * XB + (xbc >> 5)) * (C / 4) * 32 + (xbc & 31)), ref2, fa, fb);
  ta.f = ina ? fa : 0.0f; ta.m = ina ? ma : 0.0f; ta.s = ina ? sga : 0.0f;
  tb.f = inb ? fb : 0.0f; tb.m = inb ? mb : 0.0f; tb.s = inb ? sgb : 0.0f;
}

// Branch-free: out-of-image taps are gathered from the clamped position and zeroed afterwards, so that the
// loads of several taps can be in flight together (a per-tap `if` puts a reconvergence point between them).
template <int C, bool CW>
__device__ __forceinline__ Tap load_tap(const float4* __restrict__ src_img, const float* __restrict__ gm,
                                        const float2 (&ref2)[C / 2], int x, int y, int W, int H, int XB, int HW) {
  const bool inb = x >= 0 && x < W && y >= 0 && y < H;
  const int xc = min(max(x, 0), W - 1), yc = min(max(y, 0), H - 1);
  Tap t;
  const float f = tap_dot<C>(src_img + ((yc * XB + (xc >> 5)) * (C / 4) * 32 + (xc & 31)), ref2);
  t.f = inb ? f : 0.0f;
  t.m = t.s = 0.0f;
  if (CW) {
    const float m = ldg_f(gm + yc * W + xc), sg = ldg_f(gm + HW + yc * W + xc);
    t.m = inb ? m : 0.0f;
    t.s = inb ? sg : 0.0f;
  }
  return t;
}

__device__ __forceinline__ float4 bilinear_poly(float v00, float v01, float v10, float v11) {
  // v(fx,fy) = c0 + fx*cx + fy*(cy + fx*cxy)
  return make_float4(v00, v01 - v00, v10 - v00, (v00 - v01) - (v10 - v11));
}

// Depth at which the projected sample crosses the vertical grid line ix == m (horizontal: swap the
// roles of (a0,q0) and (a1,q1)):  (a0 + q0 d) / (a2 + q2 d) - 0.5 = m  =>  d = (c a2 - a0) / (q0 - c q2).
// The position is a Moebius function of depth: a grid line beyond its asymptote is only "crossed" on the other
// branch (behind the current depth) — such a line is never reached, so anything not ahead of `dcur` is +inf.
__device__ __forceinline__ float crossing_depth(float m, float a_num, float q_num, float a2, float q2, float dcur) {
  const float c = m + 0.5f;
  const float num = __fmaf_rn(c, a2, -a_num);
  const float den = __fmaf_rn(-c, q2, q_num);
  const float d = den != 0.0f ? num * rcp_nr(den) : INFINITY;
  return d >= __fmaf_rn(-1e-5f, fabsf(dcur), dcur) - 1e-12f ? d : INFINITY;
}

// Cell-list header: the cell origin (as floats).  Which hypotheses belong to which cell is carried by the
// start mask that cell_list returns.


// Phase A for one lane: the list of bilinear cells the hypotheses [j_lo, jc_end) of this (pixel, view) fall
// into, at most NCELLS per call.  Headers (cell origins) go to hdr[i * STRIDE]; returns the number of cells, the first hypothesis that is NOT covered (j_stop), the
// bounding box of the cell origins and a bit mask of the hypotheses that start a cell (chunks of <= 32).
//   walk == true : analytic walk from grid line to grid line in depth space (the sample path is a straight
//     line, monotone in depth when every hypothesis is in front of the source camera); the first hypothesis
//     of the next cell is found by binary search in the sorted k table `ks`.  The bilinear interpolant is
//     continuous across cell edges, so a hypothesis that rounding puts on the "wrong" side of an edge changes
//     the result by O(1e-6).  All lanes of the warp must call with the same `walk`.
//   walk == false: evaluate every hypothesis and record each change of cell (any depth order, any sign of z).
struct CellBox {
  int x_lo, x_hi, y_lo, y_hi;   // min / max cell origin over the recorded cells
};

template <int MODE, int NCELLS, int STRIDE>
__device__ __forceinline__ void cell_list(const CostParams& p, const DepthSrc<MODE>& ds, const float* __restrict__ ks,
                                          float2* __restrict__ hdr, bool walk, int jc, int j_lo, int jc_end,
                                          float a0, float a1, float a2, float q0, float q1, float q2, int sx, int sy,
                                          int W, int H, int& ncell, int& j_stop, CellBox& box, unsigned& startmask) {
  const unsigned FULL = 0xffffffffu;
  const float xmax = (float)W + 1.0f, ymax = (float)H + 1.0f;
  ncell = 0;
  j_stop = jc_end;
  startmask = 0u;                       // bit (j - jc) set <=> hypothesis j is the first one of a recorded cell
  box.x_lo = box.y_lo = 1 << 30;
  box.x_hi = box.y_hi = -(1 << 30);
  if (walk) {
    float ix, iy, z;
    const float d_lo = depth_of<MODE>(p, ds, j_lo);
    project(d_lo, a0, a1, a2, q0, q1, q2, ix, iy, z);
    clamp_pos(ix, iy, xmax, ymax);
    int x0 = min((int)floorf(ix), W), y0 = min((int)floorf(iy), H);            // in [-2, W] x [-2, H]
    // next grid line in the direction of travel; lines exist only at -1..W (x) / -1..H (y)
    int mx = sx > 0 ? x0 + 1 : x0, my = sy > 0 ? y0 + 1 : y0;
    float dX = (sx != 0 && mx >= -1 && mx <= W) ? crossing_depth((float)mx, a0, q0, a2, q2, d_lo) : INFINITY;
    float dY = (sy != 0 && my >= -1 && my <= H) ? crossing_depth((float)my, a1, q1, a2, q2, d_lo) : INFINITY;
    const float inv_sg = MODE == MAGNET_DEPTH_GAUSS ? rcp_nr(ds.sg) : 1.0f;
    int jcur = j_lo;
    bool done = false;
    int guard = 0;                                        // a step either records a cell, moves one grid line or ends:
    const int guard_max = 2 * (W + H) + 2 * NCELLS + 64;   // more than any walk across the image can take
    while (__any_sync(FULL, !done)) {
      if (++guard > guard_max && !done) { j_stop = jcur > j_lo ? jcur : j_lo + 1; done = true; }   // never spin, always advance
      if (!done) {
        const float dn = fminf(dX, dY);
        // first j in [jcur, jc_end) with depth_j >= dn  <=>  k_j >= kc
        const float kc = MODE == MAGNET_DEPTH_GAUSS ? (dn - ds.mu) * inv_sg : dn;
        int lo = jcur, hi = jc_end;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (ks[mid - jc] < kc) lo = mid + 1; else hi = mid;
        }
        if (lo > jcur) {                                                   // the cell holds hypotheses
          hdr[ncell * STRIDE] = make_float2((float)x0, (float)y0);
          startmask |= 1u << ((jcur - jc) & 31);
          box.x_lo = min(box.x_lo, x0); box.x_hi = max(box.x_hi, x0);
          box.y_lo = min(box.y_lo, y0); box.y_hi = max(box.y_hi, y0);
          ++ncell;
          jcur = lo;
        }
        if (jcur >= jc_end) {
          done = true;
        } else if (ncell == NCELLS) {
          j_stop = jcur;
          done = true;
        } else if (dX <= dY) {
          x0 += sx;
          mx += sx;
          dX = (mx >= -1 && mx <= W) ? crossing_depth((float)mx, a0, q0, a2, q2, dX) : INFINITY;
        } else {
          y0 += sy;
          my += sy;
          dY = (my >= -1 && my <= H) ? crossing_depth((float)my, a1, q1, a2, q2, dY) : INFINITY;
        }
      }
    }
  } else {
    float cx = -1e30f, cy = -1e30f;
    for (int j = j_lo; j < jc_end; ++j) {
      float ix, iy, z;
      project(depth_of<MODE>(p, ds, j), a0, a1, a2, q0, q1, q2, ix, iy, z);
      clamp_pos(ix, iy, xmax, ymax);
      const float fx = ix - cx, fy = iy - cy;
      if (!(fx >= 0.0f && fx < 1.0f && fy >= 0.0f && fy < 1.0f)) {
        if (ncell == NCELLS) { j_stop = j; break; }
        cx = floorf(ix);
        cy = floorf(iy);
        hdr[ncell * STRIDE] = make_float2(cx, cy);
        startmask |= 1u << ((j - jc) & 31);
        box.x_lo = min(box.x_lo, (int)cx); box.x_hi = max(box.x_hi, (int)cx);
        box.y_lo = min(box.y_lo, (int)cy); box.y_hi = max(box.y_hi, (int)cy);
        ++ncell;
      }
    }
  }
}

// Whether the analytic walk may be used for this (lane, view, chunk): depths increase with j and every
// hypothesis is in front of the source camera (z is linear in depth, so both ends suffice).
template <int MODE>
__device__ __forceinline__ bool walk_ok(const CostParams& p, const DepthSrc<MODE>& ds, int jc, int jc_end, float a2,
                                        float q2) {
  if (MODE == MAGNET_DEPTH_VOLUME || p.k_sorted == 0) return false;
  // sigma must be a NORMAL positive number: rcp.approx.ftz of a denormal is inf, the crossing depths become NaN and
  // the walk would never advance (a Gaussian update can shrink sigma by 1e-10 per iteration) -> exact walk instead
  const bool sorted = MODE == MAGNET_DEPTH_PLANES ? true : (ds.sg >= 1e-30f && ds.sg < 1e30f && fabsf(ds.mu) < 1e30f);
  const float zA = __fadd_rn(a2, __fmul_rn(q2, depth_of<MODE>(p, ds, jc)));
  const float zB = __fadd_rn(a2, __fmul_rn(q2, depth_of<MODE>(p, ds, jc_end - 1)));
  return sorted && zA > 1e-6f && zB > 1e-6f && zA < 1e30f && zB < 1e30f;
}

}  // namespace magnet
