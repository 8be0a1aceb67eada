// MAGNET_VARIANT_CELLS — tap-sharing fused warp + sample + consistency + view-fusion kernel.
//
// Replaces homography.py:79-161 (and :10-75 with CW == false) without materialising any
// D x C x H x W tensor.  Key identity (SURVEY §7 hard part 1):
//     sum_c ref_c * (sum_t w_t * src_{t,c})  ==  sum_t w_t * <ref, src_t>
// The D hypotheses of one reference pixel project onto a short epipolar segment of the source
// view, so they fall into only a handful of bilinear cells (about 6 at 640x480 / D=64).  Each
// distinct cell needs 4 channel dot products <ref[p], src[tap]> (plus 4 taps of source mu and
// sigma); every hypothesis inside the cell is then a 3-FMA bilinear polynomial per quantity.
//
// Mapping: one thread per reference pixel; a CTA is a 16x8 pixel tile (a warp = 2 rows x 16 pixels, so the
// gathers of neighbouring lanes hit neighbouring addresses and the CTA's source footprint stays compact)
// and owns ONE chunk of JCHUNK = 32 hypotheses (the chunks of a tile are adjacent CTAs).  Per view the work is
// split into three phases that every lane of a warp executes in LOCKSTEP — a run-per-cell loop would diverge
// on the bench workload, where neighbouring pixels cross different numbers of cells:
//   A  cell list: analytic walk from grid line to grid line in depth space + binary search for the first
//      hypothesis of each cell (cells_common.cuh: cell_list); exact per-hypothesis walk as the fallback
//      (d_volume mode, points behind the camera, unsorted k).  Headers in shared memory, at most NCELL per
//      round, plus a bit mask of the hypotheses that start a cell;
//   B  for cell i = 0..warp-max: channel dot products + mu/sigma of the taps that are NEW with respect to
//      the lane's previous cell (an edge-adjacent cell shares two taps, kept in registers), loads clamped
//      instead of predicated and batched (16 LDG.128 in flight) -> 12 polynomial coefficients per cell,
//      3 float4 per lane in shared memory;
//   C  walk the hypotheses; where the mask says a cell starts reload the record (3 LDS.128, the only
//      divergent code), evaluate cost / mu~ / sigma~, apply the consistency test and accumulate over views
//      in a shared-memory column owned by the lane.
// If a lane needs more than NCELL cells (incoherent depth, e.g. random test inputs) the warp processes the
// hypotheses in several rounds [j_lo, j_end), j_end = warp-min of the first hypothesis a lane could not
// cover — always correct, no separate slow path.  52 KB shared memory and 168 registers -> 3 CTAs per SM.
//
// Source features are gathered from the TILED32 layout (N, H, W/32, C/4, 32, 4): the 16 channel
// quads of one pixel sit at a compile-time stride (512 B), so one base address + immediates serve
// the whole dot product, and 32 neighbouring pixels form one contiguous 512-byte segment per quad.
//
// Numerics (DESIGN.md "parity"): same formulas as the reference, but (i) 1/Zp via MUFU.RCP + one
// Newton step and ix = P0/Zp - 0.5 folded into one FMA instead of the normalise / clamp /
// unnormalise round trip, (ii) channel sums re-associated (dot-then-blend, even / odd channel FMA chains),
// (iii) bilinear polynomial instead of 4 explicit weights, (iv) fp32 view accumulation.  Each
// changes results at the 1e-6 relative level; the hard consistency threshold can flip for elements
// within ~1e-5 of it (the reference's own fp32-vs-fp64 flips have the same margins).
#include <mutex>

#include "cells_common.cuh"
#include "launchers.h"

namespace magnet {

#ifndef MAGNET_NCELL
#define MAGNET_NCELL 5
#endif
#ifndef MAGNET_JCHUNK
#define MAGNET_JCHUNK 32
#endif
#ifndef MAGNET_TILE_W
#define MAGNET_TILE_W 16
#endif
constexpr int NT = 128;                // threads per CTA = reference pixels per CTA
constexpr int TILE_W = MAGNET_TILE_W;  // CTA tile = TILE_W x (NT / TILE_W) reference pixels (2-D keeps the
constexpr int TILE_H = NT / TILE_W;    // source footprint of a CTA compact enough for L1 to capture tap reuse)
constexpr int NCELL = MAGNET_NCELL;    // cell records per lane per round
constexpr int JCHUNK = MAGNET_JCHUNK;  // hypotheses per CTA (accumulation chunk)

__host__ __device__ inline int cells_chunk(int D) { return D < JCHUNK ? D : JCHUNK; }
// dynamic shared memory: rec[NCELL][3][NT] float4 | hdr[NCELL][NT] float2 | acc[chunk][NT] float | ks[chunk]
// (kept as small as possible: what the CTAs do not take stays L1, and the tap gathers live on L1 hits)
__host__ __device__ inline size_t cells_smem_bytes(int D) {
  return (size_t)NCELL * 3 * NT * 16 + (size_t)NCELL * NT * 8 + (size_t)cells_chunk(D) * NT * 4 +
         (size_t)cells_chunk(D) * 4;
}
static_assert(JCHUNK <= 32, "the cell start mask of a chunk is one 32-bit word");

#ifndef MAGNET_MIN_CTAS
#define MAGNET_MIN_CTAS 3   // 168 registers: more tap loads in flight per thread beats a 4th resident CTA
#endif
template <int C, int MODE, bool CW, bool REUSE, bool IDX>
__global__ void __launch_bounds__(NT, MAGNET_MIN_CTAS)
cost_cells_kernel(const __grid_constant__ CostParams p, const int chunk, const int grid_chunks,
                  const int32_t* __restrict__ src_index) {
  extern __shared__ float4 smem4[];
  float4* rec = smem4;                                                   // [NCELL][3][NT]
  float2* hdr = reinterpret_cast<float2*>(smem4 + NCELL * 3 * NT);       // [NCELL][NT]
  float* acc = reinterpret_cast<float*>(hdr + NCELL * NT);               // [chunk][NT]
  float* ks = acc + chunk * NT;                                          // [chunk] k (or plane depth) table

  const int tid = threadIdx.x;
  const int b = blockIdx.y;
  const int H = p.H, W = p.W, HW = p.HW, D = p.D;
  const int XB = (W + 31) >> 5;
  const int tiles_x = (W + TILE_W - 1) / TILE_W;
  // grid_chunks == number of chunks: one CTA per (tile, chunk), chunks of a tile adjacent (L2);
  // grid_chunks == 1: one CTA per tile that loops over the chunks (source lines of chunk c are re-used from
  // L1 / L2 by chunk c+1 of the same CTA).
  const int tile = blockIdx.x / grid_chunks;
  const int jc_first = (blockIdx.x % grid_chunks) * chunk;
  const int jc_last = grid_chunks == 1 ? D : min(jc_first + chunk, D);
  const int px = (tile % tiles_x) * TILE_W + tid % TILE_W;
  const int py = (tile / tiles_x) * TILE_H + tid / TILE_W;
  const bool live = px < W && py < H;
  const int n = live ? py * W + px : HW - 1;    // dead lanes shadow the last pixel, never store
  const unsigned FULL = 0xffffffffu;

  float2 ref2[C / 2];
  {
    const float* rp = p.ref_feat + (size_t)b * C * HW + n;
#pragma unroll
    for (int c = 0; c < C / 2; ++c) ref2[c] = make_float2(ldg_f(rp + (size_t)(2 * c) * HW), ldg_f(rp + (size_t)(2 * c + 1) * HW));
  }
  const float r0 = ldg_f(p.rays + ((size_t)b * 3 + 0) * HW + n);
  const float r1 = ldg_f(p.rays + ((size_t)b * 3 + 1) * HW + n);
  const float r2 = ldg_f(p.rays + ((size_t)b * 3 + 2) * HW + n);

  DepthSrc<MODE> ds;
  ds.HW = HW;
  ds.dv = nullptr;
  ds.mu = ds.sg = 0.0f;
  if (MODE == MAGNET_DEPTH_VOLUME) ds.dv = p.d_volume + (size_t)b * D * HW + n;
  if (MODE == MAGNET_DEPTH_GAUSS) {
    ds.mu = ldg_f(p.ref_gmm + ((size_t)b * 2 + 0) * HW + n);
    ds.sg = ldg_f(p.ref_gmm + ((size_t)b * 2 + 1) * HW + n);
  }
  const size_t img_stride4 = (size_t)H * XB * (C / 4) * 32;             // float4 per source image

  for (int jc = jc_first; jc < jc_last; jc += chunk) {
  const int jc_end = min(jc + chunk, D);
  for (int j = 0; j < jc_end - jc; ++j) acc[j * NT + tid] = 0.0f;
  if (MODE != MAGNET_DEPTH_VOLUME) {
    __syncthreads();                                                     // previous chunk done with ks
    for (int j = tid; j < jc_end - jc; j += NT) ks[j] = p.k[jc + j];
    __syncthreads();
  }

  for (int v = 0; v < p.V; ++v) {
    const magnet_camera* cam = p.cams + (b * p.V + v);
    if (cam->valid != 1.0f) continue;                                    // CTA-uniform
    const float a0 = cam->a[0], a1 = cam->a[1], a2 = cam->a[2];
    const float q0 = __fmaf_rn(cam->A[2], r2, __fmaf_rn(cam->A[1], r1, __fmul_rn(cam->A[0], r0)));
    const float q1 = __fmaf_rn(cam->A[5], r2, __fmaf_rn(cam->A[4], r1, __fmul_rn(cam->A[3], r0)));
    const float q2 = __fmaf_rn(cam->A[8], r2, __fmaf_rn(cam->A[7], r1, __fmul_rn(cam->A[6], r0)));
    const int vb = src_image<IDX>(src_index, b, v, p.B, p.V);
    const float4* src_img = reinterpret_cast<const float4*>(p.src_feat) + (size_t)vb * img_stride4;
    const float* gm = CW ? p.src_gmm + (size_t)vb * 2 * HW : nullptr;

    const bool walk = __all_sync(FULL, walk_ok<MODE>(p, ds, jc, jc_end, a2, q2));   // warp-uniform choice
    // direction of travel of the sample as depth grows: sign of d(ix)/dd = (q0 a2 - a0 q2) / z^2
    const float gx = __fmaf_rn(q0, a2, -__fmul_rn(a0, q2)), gy = __fmaf_rn(q1, a2, -__fmul_rn(a1, q2));
    const int sx = gx > 0.0f ? 1 : (gx < 0.0f ? -1 : 0), sy = gy > 0.0f ? 1 : (gy < 0.0f ? -1 : 0);

    // previous cell of this lane (taps kept in registers for reuse by an edge-adjacent next cell)
    int px0 = -1000000, py0 = -1000000;
    Tap p00, p01, p10, p11;
    p00.f = p00.m = p00.s = 0.f;
    p01 = p10 = p11 = p00;

    int j_lo = jc;
    while (j_lo < jc_end) {                                              // rounds; warp-uniform
      // ---------------- phase A: cell list ----------------------------------------------------
      int ncell, j_stop;
      CellBox box;
      unsigned startmask;
      cell_list<MODE, NCELL, NT>(p, ds, ks, hdr + tid, walk, jc, j_lo, jc_end, a0, a1, a2, q0, q1, q2, sx, sy, W, H,
                                 ncell, j_stop, box, startmask);
      const int j_end = __reduce_min_sync(FULL, j_stop);
      const int nmax = __reduce_max_sync(FULL, ncell);

      // ---------------- phase B: per-cell records ----------------------------------------------
      // (every lane computes the same tap slot per iteration: its gathers are issued together, which gives more
      // memory-level parallelism than each lane walking its own list of new taps)
      for (int i = 0; i < nmax; ++i) {
        if (i < ncell) {
          const float2 h = hdr[i * NT + tid];
          const int x0 = (int)h.x, y0 = (int)h.y;
          const int dx = x0 - px0, dy = y0 - py0;
          const bool mvx = REUSE && dy == 0 && (dx == 1 || dx == -1);
          const bool mvy = REUSE && dx == 0 && (dy == 1 || dy == -1);
          // two taps every lane computes: the new column (x move), the new row (y move), or the top row
          int ax = x0, ay = y0, bx = x0 + 1, by = y0;
          if (mvx) { ax = bx = (dx == 1) ? x0 + 1 : x0; by = y0 + 1; }
          if (mvy) { ay = by = (dy == 1) ? y0 + 1 : y0; }
          Tap tA, tB;
          load_tap2<C, CW>(src_img, gm, ref2, ax, ay, bx, by, W, H, XB, HW, tA, tB);
          Tap n00, n01, n10, n11;
          if (mvx) {
            if (dx == 1) { n00 = p01; n10 = p11; n01 = tA; n11 = tB; }
            else         { n01 = p00; n11 = p10; n00 = tA; n10 = tB; }
          } else if (mvy) {
            if (dy == 1) { n00 = p10; n01 = p11; n10 = tA; n11 = tB; }
            else         { n10 = p00; n11 = p01; n00 = tA; n01 = tB; }
          } else {                                                       // first cell / diagonal / jump
            n00 = tA; n01 = tB;
            load_tap2<C, CW>(src_img, gm, ref2, x0, y0 + 1, x0 + 1, y0 + 1, W, H, XB, HW, n10, n11);
          }
          p00 = n00; p01 = n01; p10 = n10; p11 = n11;
          px0 = x0; py0 = y0;
          rec[(i * 3 + 0) * NT + tid] = bilinear_poly(n00.f, n01.f, n10.f, n11.f);
          if (CW) {
            rec[(i * 3 + 1) * NT + tid] = bilinear_poly(n00.m, n01.m, n10.m, n11.m);
            rec[(i * 3 + 2) * NT + tid] = bilinear_poly(n00.s, n01.s, n10.s, n11.s);
          }
        }
      }

      // ---------------- phase C: evaluate hypotheses [j_lo, j_end) -----------------------------
      {
        float cx = 0.0f, cy = 0.0f;
        float4 rd = make_float4(0.f, 0.f, 0.f, 0.f), rm = rd, rs = rd;
        const float2* hp = hdr + tid - NT;
        const float4* rp = rec + tid - 3 * NT;
        float* ap = acc + (j_lo - jc) * NT + tid;
        unsigned starts = startmask >> (j_lo - jc);                      // bit 0 <=> hypothesis j starts a cell
        // one hypothesis: switch to the lane's next cell where the mask says so, blend, test, accumulate
        auto eval = [&](const float ix, const float iy, const float z, const bool start, float* __restrict__ a) {
          if (start) {                                                   // entering the lane's next cell
            hp += NT;
            rp += 3 * NT;
            const float2 h = *hp;
            cx = h.x;
            cy = h.y;
            rd = rp[0];
            if (CW) {
              rm = rp[NT];
              rs = rp[2 * NT];
            }
          }
          const float fx = ix - cx, fy = iy - cy;
          float cost = __fmaf_rn(fy, __fmaf_rn(fx, rd.w, rd.z), __fmaf_rn(fx, rd.y, rd.x));
          if (!(fabsf(cost) < 3.0e38f)) cost = 0.0f;                     // all-zero record x non-finite position
          float val = cost;
          if (CW) {
            const float mu = __fmaf_rn(fy, __fmaf_rn(fx, rm.w, rm.z), __fmaf_rn(fx, rm.y, rm.x));
            const float sg = __fmaf_rn(fy, __fmaf_rn(fx, rs.w, rs.z), __fmaf_rn(fx, rs.y, rs.x));
            // homography.py:157-158: |z - mu~| < sigma~ * kappa, strict
            val = (fabsf(__fsub_rn(z, mu)) < __fmul_rn(sg, p.kappa)) ? cost : 0.0f;
          }
          *a += val;
        };
        int j = j_lo;
#pragma unroll 2
        for (; j + 1 < j_end; j += 2, ap += 2 * NT, starts >>= 2) {      // two hypotheses per float2 projection
          float2 ix2, iy2, z2;
          project2(make_float2(depth_of<MODE>(p, ds, j), depth_of<MODE>(p, ds, j + 1)), a0, a1, a2, q0, q1, q2, ix2, iy2, z2);
          eval(ix2.x, iy2.x, z2.x, (starts & 1u) != 0u, ap);
          eval(ix2.y, iy2.y, z2.y, (starts & 2u) != 0u, ap + NT);
        }
        if (j < j_end) {
          float ix, iy, z;
          project(depth_of<MODE>(p, ds, j), a0, a1, a2, q0, q1, q2, ix, iy, z);
          eval(ix, iy, z, (starts & 1u) != 0u, ap);
        }
      }
      j_lo = j_end;
    }
  }

  // -------- epilogue: 1/V mean over ALL views (homography.py:120) ---------------------------------
  if (live) {
    float* outp = p.out + ((size_t)b * D + jc) * HW + n;
    const int cnt = jc_end - jc;
    if (p.inv_v_exact != 0.0f) {
      for (int j = 0; j < cnt; ++j) outp[(size_t)j * HW] = acc[j * NT + tid] * p.inv_v_exact;
    } else {
      for (int j = 0; j < cnt; ++j) outp[(size_t)j * HW] = __fdiv_rn(acc[j * NT + tid], p.vf);
    }
  }
  }   // chunk loop
}

static int cells_grid_x(int H, int W) { return ((W + TILE_W - 1) / TILE_W) * ((H + TILE_H - 1) / TILE_H); }

template <int C, int MODE, bool CW, bool REUSE, bool IDX>
static cudaError_t launch_cells(const CostParams& p, const int32_t* src_index, cudaStream_t st) {
  static std::once_flag flags[64];
  auto kern = cost_cells_kernel<C, MODE, CW, REUSE, IDX>;
  cudaError_t e = set_smem_once(kern, flags, (int)cells_smem_bytes(MAGNET_MAX_PLANES), false);
  if (e != cudaSuccess) return e;
  const size_t smem = cells_smem_bytes(p.D);
  const int chunk = cells_chunk(p.D), nchunks = (p.D + chunk - 1) / chunk;
  dim3 grid(cells_grid_x(p.H, p.W) * nchunks, p.B), block(NT);
  kern<<<grid, block, smem, st>>>(p, chunk, nchunks, src_index);
  return cudaGetLastError();
}

bool cells_supports(int C, int D, int layout) {
  return (C == 16 || C == 32 || C == 64) && layout == MAGNET_SRC_TILED32 && D >= 1;
}

void cells_launch_info(int B, int H, int W, int D, int* grid, int* block, int* smem) {
  const int chunk = cells_chunk(D);
  *grid = cells_grid_x(H, W) * ((D + chunk - 1) / chunk) * B;
  *block = NT;
  *smem = (int)cells_smem_bytes(D);
}

cudaError_t launch_cost_cells(const CostParams& p, int mode, int C, bool cw, bool reuse, const int32_t* src_index,
                              cudaStream_t st, int* launches) {
  *launches = 1;
  return dispatch(
      [&](auto c, auto m, auto w, auto r, auto idx) -> cudaError_t {
        // !REUSE is a diagnostic variant: only the bench configuration, GAUSS, is instantiated
        if constexpr (!r && m != MAGNET_DEPTH_GAUSS) return cudaErrorInvalidValue;
        else return launch_cells<c, m, w, r, idx>(p, src_index, st);
      },
      Choice<int, 16, 32, 64>{C}, DepthMode{mode}, Flag{cw}, Flag{reuse}, Flag{src_index != nullptr});
}

}  // namespace magnet
