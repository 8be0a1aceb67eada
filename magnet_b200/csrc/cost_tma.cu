// MAGNET_VARIANT_TMA — TMA-staged CUDA-core kernel (MAGNET_SRC_PIXC; AUTO uses it for the drop-in path with few
// hypotheses or C in {16, 32} — cost_mma.cu is the production kernel for C == 64): tap-sharing fused warp + sample + consistency + view fusion
// with the CTA's source window staged in shared memory by TMA (cp.async.bulk.tensor, mbarrier completion) and the
// per-hypothesis state held in a per-thread shared-memory scratch.
//
// Replaces homography.py:79-161 (and :10-75 with CW == false); absorbs the sampler of MAGNET.py:154-156.
// Same identity as cost_cells.cu — sum_c ref_c (sum_t w_t src_tc) = sum_t w_t <ref, src_t>, each bilinear cell of a
// (pixel, view) costs 4 channel dot products and every hypothesis inside it is a 3-FMA polynomial — but a different
// machine mapping, chosen from the round-1 profile (the gathers, not HBM, bound cost_cells: 3.4 GB L2->L1 per launch):
//
//   * source features live in MAGNET_SRC_PIXC: (N, H, W, C+4) = per pixel C channels + (mu, sigma, 0, 0), 272 B for
//     C = 64.  One rank-4 tensor map (box = 8 pixels x 1 row) describes it; per (CTA, view) the bounding box of the
//     CTA's bilinear cells is fetched by 8-pixel TMA boxes into a pixel-major window: every source byte crosses
//     L2 -> SM once per (tile, view), out-of-image taps are ZERO-FILLED by the copy engine (grid_sample's
//     padding_mode='zeros' for free, no bounds checks), and the 272-byte pixel pitch makes the 16-byte tap reads of 8
//     neighbouring pixels bank-conflict free.  The camera table of the batch element is staged by cp.async.bulk.
//   * FOUR lanes per reference pixel: lane h holds 16 of the 64 reference channels (16 registers instead of 64) and a
//     contiguous quarter of the hypotheses.  A tap is 4 LDS.128 + 16 FFMA per lane and a 2-step butterfly; the
//     hypothesis phases need no cross-lane traffic.  CTA = 16x4 pixel tile = 256 threads, two CTAs per SM = 16 warps.
//   * the lane's 16 depth hypotheses and 16 view accumulators live in a per-thread SHARED-MEMORY scratch (32 KB per
//     CTA, 16-byte groups interleaved across the threads: conflict-free): the index may be a run-time value, so the
//     per-hypothesis loops stay rolled (small code, no register arrays, no spills) — with the arrays in registers the
//     fully unrolled phases needed > 255 registers.
//   * per view: A  every lane walks ITS hypotheses exactly (no sortedness assumption, identical for d_volume /
//                  Gaussian / plane depths), flags the ones that enter a new bilinear cell; the 4 lanes of a pixel
//                  splice their lists (shuffles) into <= NORG cell origins in shared memory + the CTA bounding box;
//               -> TMA of the window (one elected warp), mbarrier wait;
//               then, NCP cells at a time (one pass for 87 % of the warps at cfg2):
//               B  lockstep over the pixel's cells: the two taps that are new w.r.t. the previous cell (4 for the first
//                  / a diagonal move) -> polynomial records (cost, mu~, sigma~) in shared memory;
//               C  every lane evaluates its hypotheses that fall into those cells (record reloaded only where the cell
//                  changes), applies |z - mu~| < kappa sigma~ and accumulates over the views.
//     More than NORG cells per pixel / KL per lane (incoherent depth) -> the walk restarts behind the last covered
//     hypothesis with taps gathered from global memory; a window that does not fit the buffer -> the same global path
//     for that view.  Always correct.
//
// Numerics: as cost_cells.cu (DESIGN.md "parity"); channel sums are additionally split over 4 lanes.
#include <mutex>

#include "common.cuh"
#include "launchers.h"
#include "tma_common.cuh"

namespace magnet {

constexpr int TNT = 256;               // threads per CTA
constexpr int TTW = 16, TTH = 4;       // CTA tile in reference pixels; a warp = 8 pixels of one row x 4 lanes
constexpr int TPX = TTW * TTH;         // 64 pixels
constexpr int NCP = 8;                 // cell records per pixel per B/C pass
constexpr int NORG = 16;               // cell origins per pixel per walk
constexpr int KL = 6;                  // cells one lane may contribute per walk (staging slots)
constexpr int TJL = 16;                // hypotheses per lane
constexpr int TCH = 4 * TJL;           // hypotheses per CTA (chunk)
constexpr int TMAXV = 16;              // views whose camera constants are staged in shared memory
constexpr int SCR_COLS = 32;           // scratch floats per thread: 16 depths + 16 accumulators

// shared-memory map (bytes)
constexpr int OFF_BAR = 0;                                   // mbarrier
constexpr int OFF_BBOX = 16;                                 // int[2][4]  x_lo, x_hi, y_lo, y_hi of the cell origins
constexpr int OFF_KS = 64;                                   // float[TCH] sampler offsets / plane depths of the chunk
constexpr int OFF_CAM = OFF_KS + TCH * 4;                    // magnet_camera[TMAXV]
constexpr int OFF_ORG = OFF_CAM + TMAXV * 64;                // float2[NORG][TPX]  cell origins
constexpr int OFF_REC = OFF_ORG + NORG * TPX * 8;            // float4[3][NCP][TPX] records; every warp's own rows double
constexpr int OFF_SCR = ((OFF_REC + 3 * NCP * TPX * 16 + 127) / 128) * 128;   //   as its float2 staging slots in phase A
constexpr int OFF_WIN = OFF_SCR + SCR_COLS * TNT * 4;        // float4[SCR_COLS / 4][TNT] per-thread scratch
constexpr int TMA_SMEM_TOTAL = (228 * 1024 - 2 * 1024) / 2;  // two CTAs per SM (1 KB per CTA is reserved by the driver)
static_assert(4 * KL <= 3 * NCP, "one staging slot per record row (see phase_a)");
static_assert(OFF_CAM % 16 == 0 && OFF_ORG % 16 == 0 && OFF_REC % 16 == 0 && OFF_SCR % 16 == 0, "alignment");

__host__ __device__ constexpr int pix_floats(int C) { return C + 4; }
__host__ __device__ constexpr int tma_box_bytes(int C) { return 8 * pix_floats(C) * 4; }
__host__ __device__ constexpr int tma_win_cap(int C) { return (TMA_SMEM_TOTAL - OFF_WIN) / tma_box_bytes(C); }

struct ViewGeom {
  float a0, a1, a2, q0, q1, q2;
};

__device__ __forceinline__ void project2(const float2 d, const ViewGeom& g, float2& ix, float2& iy, float2& z) {
  project2(d, g.a0, g.a1, g.a2, g.q0, g.q1, g.q2, ix, iy, z);   // common.cuh: two hypotheses side by side
}

// predicated shared-memory loads (the destination keeps its value when the predicate is false): phase C reloads the
// record only where the cell changes, without a branch per hypothesis
__device__ __forceinline__ void lds128_if(bool p, uint32_t addr, float4& v) {
  asm volatile("{\n.reg .pred q;\nsetp.ne.u32 q, %4, 0;\n@q ld.shared.v4.f32 {%0, %1, %2, %3}, [%5];\n}"
               : "+f"(v.x), "+f"(v.y), "+f"(v.z), "+f"(v.w) : "r"((unsigned)p), "r"(addr));
}
__device__ __forceinline__ void lds64_if(bool p, uint32_t addr, float& a, float& b) {
  asm volatile("{\n.reg .pred q;\nsetp.ne.u32 q, %2, 0;\n@q ld.shared.v2.f32 {%0, %1}, [%3];\n}"
               : "+f"(a), "+f"(b) : "r"((unsigned)p), "r"(addr));
}

__device__ __forceinline__ float4 bilinear_poly4(float v00, float v01, float v10, float v11) {
  // v(fx,fy) = c0 + fx*cx + fy*(cy + fx*cxy)
  return make_float4(v00, v01 - v00, v10 - v00, (v00 - v01) - (v10 - v11));
}

// Per-thread scratch: column c (a multiple of 4; columns 8q .. 8q+3 = depths 4q .. 4q+3, 8q+4 .. 8q+7 = their
// accumulators) is one float4 at scr[(c / 4) * TNT], scr = the thread's slot of the OFF_SCR array.
__device__ __forceinline__ float4& scr_at(float4* scr, int c) { return scr[(c >> 2) * TNT]; }

// Per-lane result of phase A (pixel-wide quantities are identical on the 4 lanes of a pixel).
struct LaneCells {
  unsigned mask;   // bit m: my hypothesis m starts a cell that this walk keeps
  int base;        // number of kept cells of the pixel that start before my range
  int ncell;       // kept cells of the pixel
  int jstop;       // first (chunk-local) hypothesis of the pixel that this walk does NOT cover
  int mlo;         // my first pending hypothesis (TJL: none)
};

// ---------------------------------------------------------------------------------------------------------------
// Phase A: hypotheses >= jlo of the pixel are pending.  Scratch columns 8q .. 8q+3 hold my depths 4q .. 4q+3;
// depths beyond my last hypothesis replicate it (so they never start a cell and need no predicate).
// Every lane projects each of its hypotheses and records the changes of cell: exact for any depth order and sign of z.
// (The analytic grid-line walk of cost_cells.cu over each lane's quarter of the hypotheses would walk 32 lanes in
// lockstep with a binary search per step; this loop has no data-dependent trip count.)
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ LaneCells phase_a(const ViewGeom& g, float4* __restrict__ scr, const int mend, const int nj,
                                             const int jb, const int jlo, const int Dc, const int W, const int H,
                                             const int lane, const int pxl, float2* __restrict__ stg,
                                             float2* __restrict__ org, int (&box)[4]) {
  const unsigned FULL = 0xffffffffu;
  const int h = lane >> 3;
  const float xmax = (float)W + 1.0f, ymax = (float)H + 1.0f;
  int mlo = min(max(jlo - jb, 0), TJL);
  if (mlo >= nj) mlo = TJL;
  __syncwarp();                                           // the staging area aliases the records phase C just read
  unsigned mask = 0u;
  int k = 0;
  int lane_stop = nj;                                     // first of MY hypotheses that this walk does not cover
  float pcx = 0.0f, pcy = 0.0f;
  // staging slot (h, k) of pixel p lives in the first half of the 128-byte segment that record row h*KL + k holds for
  // this warp's 8 pixels: staging never touches bytes that belong to another warp's records (which that warp may
  // still be reading in phase C of the previous view)
  float2* mystg = stg + ((h * KL) * TPX + (pxl & ~7)) * 2 + (lane & 7);
  constexpr int SK = 2 * TPX;                             // float2 stride between consecutive staging slots
  {
#pragma unroll 1
    for (int m = 0; m < mend; m += 4) {                   // 4 hypotheses per trip: two independent float2 projections
      const float4 d = scr_at(scr, 2 * m);
      float2 ixa, iya, za, ixb, iyb, zb;
      project2(make_float2(d.x, d.y), g, ixa, iya, za);
      project2(make_float2(d.z, d.w), g, ixb, iyb, zb);
      // anything left of -1 / right of W (above / below likewise) has all four taps out of the image: clamp so that
      // cell coordinates stay small and NaN (fmaxf drops it) maps to "out of bounds"
      float cx[4], cy[4];
      cx[0] = floorf(fminf(fmaxf(ixa.x, -2.0f), xmax)); cy[0] = floorf(fminf(fmaxf(iya.x, -2.0f), ymax));
      cx[1] = floorf(fminf(fmaxf(ixa.y, -2.0f), xmax)); cy[1] = floorf(fminf(fmaxf(iya.y, -2.0f), ymax));
      cx[2] = floorf(fminf(fmaxf(ixb.x, -2.0f), xmax)); cy[2] = floorf(fminf(fmaxf(iyb.x, -2.0f), ymax));
      cx[3] = floorf(fminf(fmaxf(ixb.y, -2.0f), xmax)); cy[3] = floorf(fminf(fmaxf(iyb.y, -2.0f), ymax));
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int mm = m + e;
        const float qx = e ? cx[e - 1] : pcx, qy = e ? cy[e - 1] : pcy;
        const bool f = (mm >= mlo) && ((cx[e] != qx) || (cy[e] != qy) || mm == mlo);
        if (f) {
          if (k < KL) mystg[k * SK] = make_float2(cx[e], cy[e]);
          ++k;
          mask |= 1u << mm;
        }
      }
      pcx = cx[3];
      pcy = cy[3];
    }
    if (__any_sync(FULL, k > KL)) {                       // more cells than staging slots: cover up to the first unsaved
      if (k > KL) {
        lane_stop = (int)__fns(mask, 0, KL + 1);
        mask &= (1u << lane_stop) - 1u;
        k = KL;
      }
    }
  }
  // ---- splice the four lists of the pixel --------------------------------------------------------------------
  const bool has = mlo < TJL;
  const float plx = __shfl_up_sync(FULL, pcx, 8), ply = __shfl_up_sync(FULL, pcy, 8);   // last cell of lane h-1
  const float2 first = (has && k > 0) ? mystg[0] : make_float2(-1e9f, -1e9f);
  // my first pending hypothesis continues the cell of the previous lane's last hypothesis (which is pending, too)
  const bool cont = has && h > 0 && mlo == 0 && jb > jlo && first.x == plx && first.y == ply;
  const int skip = cont ? 1 : 0;
  if (cont) mask &= ~1u;
  int n = __popc(mask);
  auto scan4 = [&](int v, int& incl) {                    // inclusive scan over the 4 lanes of the pixel (stride 8)
    int s = v;
    int t = __shfl_up_sync(FULL, s, 8);
    if (h >= 1) s += t;
    t = __shfl_up_sync(FULL, s, 16);
    if (h >= 2) s += t;
    incl = s;
  };
  int incl;
  scan4(n, incl);
  int base = incl - n;
  const int kept_g = max(0, min(n, NORG - base));
  int jstop = Dc;
  if (__any_sync(FULL, kept_g < n || lane_stop < nj)) {   // some lane of the warp has to drop cells: rare
    int js = Dc;
    if (kept_g < n) js = jb + (int)__fns(mask, 0, kept_g + 1);   // my first dropped start
    else if (lane_stop < nj) js = jb + lane_stop;
    js = min(js, __shfl_xor_sync(FULL, js, 8));
    js = min(js, __shfl_xor_sync(FULL, js, 16));
    jstop = js;
    const int lim = jstop - jb;
    if (lim <= 0) mask = 0u;
    else if (lim < TJL) mask &= (1u << lim) - 1u;
    n = __popc(mask);
    scan4(n, incl);
    base = incl - n;
  }
  const int ncell = __shfl_sync(FULL, incl, 24 + (lane & 7));
  // ---- compaction: staging -> cell origins in hypothesis order, bounding box of the kept cells --------------
  float bx_lo = 1e9f, bx_hi = -1e9f, by_lo = 1e9f, by_hi = -1e9f;
#pragma unroll
  for (int kk = 0; kk < KL; ++kk) {
    const int gi = kk - skip;
    if (gi >= 0 && gi < n) {
      const float2 o = mystg[kk * SK];
      org[(base + gi) * TPX + pxl] = o;
      bx_lo = fminf(bx_lo, o.x); bx_hi = fmaxf(bx_hi, o.x);
      by_lo = fminf(by_lo, o.y); by_hi = fmaxf(by_hi, o.y);
    }
  }
  box[0] = __reduce_min_sync(FULL, (int)bx_lo);
  box[1] = __reduce_max_sync(FULL, (int)bx_hi);
  box[2] = __reduce_min_sync(FULL, (int)by_lo);
  box[3] = __reduce_max_sync(FULL, (int)by_hi);
  __syncwarp();                                           // origins visible to the other lanes of the pixel
  LaneCells lc;
  lc.mask = mask;
  lc.base = base;
  lc.ncell = ncell;
  lc.jstop = jstop;
  lc.mlo = mlo;
  return lc;
}

// ---------------------------------------------------------------------------------------------------------------
// Phase B: polynomial records of the pixel's cells [i0, i1).  STAGED: taps from the shared-memory window (no bounds
// checks: the copy engine zero-filled what lies outside the image); otherwise from the PIXC image in global memory.
// ---------------------------------------------------------------------------------------------------------------
struct CornerState {                    // previous cell of the pixel and the corner values of MY quantity there
  int px0, py0;
  float c00, c01, c10, c11;
};

template <int C, bool CW, bool STAGED>
__device__ __forceinline__ void phase_b(const float2 (&ref2)[C / 8], const int ncell, const int i0, const int i1,
                                        CornerState& cs, const int lane, const int pxl,
                                        const float2* __restrict__ org, float4* __restrict__ rec,
                                        const unsigned char* __restrict__ sm, const int cbase,
                                        const unsigned char* __restrict__ img, const int row_bytes, const int sx,
                                        const int sy, const int W, const int H) {
  constexpr int QL = C / 16;              // float4 per lane per tap
  constexpr int PS = pix_floats(C) * 4;   // bytes per pixel
  const unsigned FULL = 0xffffffffu;
  const int h = lane >> 3;
  // STAGED: a tap lives at sm[cbase + y*row_bytes + x*PS], cbase = window offset + my channel offset -
  // (wy0*row_bytes + wx0*PS) (kept as an offset into the shared array so that the loads stay LDS); (sx, sy) = window
  // origin (safe tap for idle lanes).  Global: img = image + my channel offset, row_bytes = W*PS.
  struct TapV { float f, m, s; };
  auto tap = [&](int x, int y) -> TapV {
    bool inb = true;
    if (!STAGED) {
      inb = x >= 0 && x < W && y >= 0 && y < H;
      x = min(max(x, 0), W - 1);
      y = min(max(y, 0), H - 1);
    }
    const unsigned char* pp = STAGED ? sm + (cbase + y * row_bytes + x * PS) : img + ((size_t)y * row_bytes + (size_t)x * PS);
    const float4* s = reinterpret_cast<const float4*>(pp);
    float2 s0 = make_float2(0.f, 0.f), s1 = make_float2(0.f, 0.f);
#pragma unroll
    for (int q = 0; q < QL; ++q) {
      const float4 t = STAGED ? s[q] : __ldg(s + q);
      s0 = ffma2_rn(ref2[2 * q + 0], make_float2(t.x, t.y), s0);
      s1 = ffma2_rn(ref2[2 * q + 1], make_float2(t.z, t.w), s1);
    }
    TapV r;
    r.f = (s0.x + s0.y) + (s1.x + s1.y);
    r.m = r.s = 0.0f;
    if (CW) {
      const float2* g2 = reinterpret_cast<const float2*>(pp + (C * 4 - h * QL * 16));
      const float2 ms = STAGED ? *g2 : __ldg(g2);
      r.m = ms.x;
      r.s = ms.y;
    }
    if (!STAGED && !inb) r.f = r.m = r.s = 0.0f;
    return r;
  };
  auto reduce4 = [&](float v) {                           // sum over the 4 lanes of the pixel (all get the result)
    v += __shfl_xor_sync(FULL, v, 8);
    v += __shfl_xor_sync(FULL, v, 16);
    return v;
  };
  // the quantity this lane keeps corner values / builds the polynomial of: 0 cost, 1 mu, 2 sigma (3: idle)
  auto mine = [&](const TapV& t, float f) { return h == 0 ? f : (h == 1 ? t.m : t.s); };

  for (int i = i0; i < i1; ++i) {
    const bool act = i < ncell;
    int x0 = sx, y0 = sy;
    if (act) {
      const float2 o = org[i * TPX + pxl];
      x0 = (int)o.x;
      y0 = (int)o.y;
    }
    const int dx = x0 - cs.px0, dy = y0 - cs.py0;
    const bool mvx = act && dy == 0 && (dx == 1 || dx == -1);
    const bool mvy = act && dx == 0 && (dy == 1 || dy == -1);
    const bool all4 = act && !(mvx || mvy);                // first cell of the view / diagonal move / jump
    // two taps every lane computes: the new column (x move), the new row (y move), or the top row
    int ax = x0, ay = y0, bx = x0 + 1, by = y0;
    if (mvx) { ax = bx = (dx == 1) ? x0 + 1 : x0; by = y0 + 1; }
    if (mvy) { ay = by = (dy == 1) ? y0 + 1 : y0; }
    if (!act) { bx = x0; }
    const TapV tA = tap(ax, ay), tB = tap(bx, by);
    const float fA = reduce4(tA.f), fB = reduce4(tB.f);
    const float vA = mine(tA, fA), vB = mine(tB, fB);
    float vC = 0.f, vD = 0.f;
    if (__any_sync(FULL, all4)) {
      const int cy = all4 ? y0 + 1 : y0, ex = all4 ? x0 + 1 : x0;
      const TapV tC = tap(x0, cy), tD = tap(ex, cy);
      const float fC = reduce4(tC.f), fD = reduce4(tD.f);
      vC = mine(tC, fC);
      vD = mine(tD, fD);
    }
    if (act) {
      float n00, n01, n10, n11;
      if (mvx) {
        if (dx == 1) { n00 = cs.c01; n10 = cs.c11; n01 = vA; n11 = vB; }
        else         { n01 = cs.c00; n11 = cs.c10; n00 = vA; n10 = vB; }
      } else if (mvy) {
        if (dy == 1) { n00 = cs.c10; n01 = cs.c11; n10 = vA; n11 = vB; }
        else         { n10 = cs.c00; n11 = cs.c01; n00 = vA; n01 = vB; }
      } else {
        n00 = vA; n01 = vB; n10 = vC; n11 = vD;
      }
      cs.c00 = n00; cs.c01 = n01; cs.c10 = n10; cs.c11 = n11;
      cs.px0 = x0; cs.py0 = y0;
      if (h < (CW ? 3 : 1)) rec[(h * NCP + (i - i0)) * TPX + pxl] = bilinear_poly4(n00, n01, n10, n11);
    }
  }
  __syncwarp();                                           // records visible to the other lanes of the pixel
}

// ---------------------------------------------------------------------------------------------------------------
// Phase C: every lane evaluates its pending hypotheses whose cell index lies in [i0, i0 + NCP) from the records and
// adds them to its accumulators (scratch columns 8q + 4 .. 8q + 7).
// ---------------------------------------------------------------------------------------------------------------
template <bool CW>
__device__ __forceinline__ void phase_c(const ViewGeom& g, float4* __restrict__ scr, const int mend, const LaneCells& lc,
                                        const int jb, const int i0, const float kappa, const int pxl,
                                        const float2* __restrict__ org, const float4* __restrict__ rec) {
  const int mhi = min(max(lc.jstop - jb, 0), TJL);
  float ox = 0.f, oy = 0.f;
  float4 rd = make_float4(0.f, 0.f, 0.f, 0.f), rm = rd, rs = rd;
  const uint32_t org_a = smem_u32(org + pxl), rec_a = smem_u32(rec + pxl);
  int cnt = lc.base - 1;                                  // index of the cell my current hypothesis lies in: starts
  int cur = -1000;                                        // at the cell lane h-1 ended in; cur = the one loaded
  unsigned msk = lc.mask;
#pragma unroll 1
  for (int m = 0; m < mend; m += 4) {                     // 4 hypotheses per trip (instruction-level parallelism)
    const float4 dv = scr_at(scr, 2 * m), av = scr_at(scr, 2 * m + 4);
    float v[8] = {dv.x, dv.y, dv.z, dv.w, av.x, av.y, av.z, av.w};   // my depths m..m+3 and their accumulators
    float2 ix2[2], iy2[2], z2[2];
    project2(make_float2(v[0], v[1]), g, ix2[0], iy2[0], z2[0]);
    project2(make_float2(v[2], v[3]), g, ix2[1], iy2[1], z2[1]);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int mm = m + e;
      cnt += (int)(msk & 1u);
      msk >>= 1;
      const int slot = cnt - i0;
      const bool inr = mm >= lc.mlo && mm < mhi && (unsigned)slot < (unsigned)NCP;
      const bool st = inr && cnt != cur;                  // entering another cell: reload its record (predicated)
      cur = st ? cnt : cur;
      const uint32_t ro = (uint32_t)(max(slot, 0) * TPX) * 16u;
      lds64_if(st, org_a + (uint32_t)(max(cnt, 0) * TPX) * 8u, ox, oy);
      lds128_if(st, rec_a + ro, rd);
      if (CW) {
        lds128_if(st, rec_a + ro + (uint32_t)(NCP * TPX * 16), rm);
        lds128_if(st, rec_a + ro + (uint32_t)(2 * NCP * TPX * 16), rs);
      }
      const float pxi = (e & 1) ? ix2[e >> 1].y : ix2[e >> 1].x, pyi = (e & 1) ? iy2[e >> 1].y : iy2[e >> 1].x;
      const float pz = (e & 1) ? z2[e >> 1].y : z2[e >> 1].x;
      const float fx = pxi - ox, fy = pyi - oy;
      const float cost = __fmaf_rn(fy, __fmaf_rn(fx, rd.w, rd.z), __fmaf_rn(fx, rd.y, rd.x));
      bool ok;
      if (CW) {
        const float mu = __fmaf_rn(fy, __fmaf_rn(fx, rm.w, rm.z), __fmaf_rn(fx, rm.y, rm.x));
        const float sg = __fmaf_rn(fy, __fmaf_rn(fx, rs.w, rs.z), __fmaf_rn(fx, rs.y, rs.x));
        // homography.py:157-158: |z - mu~| < sigma~ * kappa, strict.  A non-finite position makes mu~ NaN (0 * inf),
        // the comparison false and the contribution 0 — what the reference's +-10 clamp + zero padding produce.
        ok = fabsf(__fsub_rn(pz, mu)) < __fmul_rn(sg, kappa);
      } else {
        ok = fabsf(cost) < 3.0e38f;                       // all-zero record x non-finite position
      }
      v[4 + e] += (ok && inr) ? cost : 0.0f;
    }
    scr_at(scr, 2 * m + 4) = make_float4(v[4], v[5], v[6], v[7]);
  }
}

template <int C, int MODE, bool CW, bool IDX>
__global__ void __launch_bounds__(TNT, 2)
cost_tma_kernel(const __grid_constant__ CostParams p, const __grid_constant__ CUtensorMap tmap, const int win_cap,
                const int nchunks, const int32_t* __restrict__ src_index) {
  constexpr int QL = C / 16;
  constexpr int PS = pix_floats(C) * 4;
  constexpr int BOX = tma_box_bytes(C);
  extern __shared__ __align__(128) unsigned char smem[];
  int* bbox = reinterpret_cast<int*>(smem + OFF_BBOX);
  float* ks = reinterpret_cast<float*>(smem + OFF_KS);
  const magnet_camera* cams_s = reinterpret_cast<const magnet_camera*>(smem + OFF_CAM);
  float2* org = reinterpret_cast<float2*>(smem + OFF_ORG);
  float4* rec = reinterpret_cast<float4*>(smem + OFF_REC);
  float2* stg = reinterpret_cast<float2*>(smem + OFF_REC);
  unsigned char* win = smem + OFF_WIN;
  const uint32_t bar = smem_u32(smem + OFF_BAR);
  const unsigned FULL = 0xffffffffu;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, h = lane >> 3;
  const int b = blockIdx.y;
  const int H = p.H, W = p.W, HW = p.HW, D = p.D, V = p.V;
  const int tiles_x = (W + TTW - 1) / TTW;
  const int tile = blockIdx.x / nchunks;                   // the chunks of a tile are adjacent CTAs (window reuse in L2)
  const int jc = (blockIdx.x % nchunks) * TCH;
  const int Dc = min(TCH, D - jc);
  const int JLc = (Dc + 3) >> 2;                           // hypotheses per lane in this chunk
  const int mend = (JLc + 3) & ~3;                         // ... rounded up to whole quads (CTA-uniform loop bound)
  const int jb = h * JLc;                                  // my first (chunk-local) hypothesis
  const int nj = min(max(Dc - jb, 0), JLc);                // how many I own
  const int trow = warp >> 1, tcol = (warp & 1) * 8 + (lane & 7);
  const int pxl = trow * TTW + tcol;
  const int px = (tile % tiles_x) * TTW + tcol, py = (tile / tiles_x) * TTH + trow;
  const bool live = px < W && py < H;
  const int n = min(py, H - 1) * W + min(px, W - 1);       // dead lanes shadow the nearest pixel of the image, never store

  if (tid == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
    bbox[0] = bbox[2] = bbox[4] = bbox[6] = 1 << 30;
    bbox[1] = bbox[3] = bbox[5] = bbox[7] = -(1 << 30);
    prefetch_tmap(&tmap);
  }
  if (tid < TCH) ks[tid] = (MODE != MAGNET_DEPTH_VOLUME && jc + tid < D) ? p.k[jc + tid] : 0.0f;
  __syncthreads();
  if (tid == 0) {                                          // camera constants of this batch element: one bulk copy
    mbar_arrive_expect_tx(bar, (uint32_t)V * 64u);
    bulk_load(smem_u32(smem + OFF_CAM), p.cams + (size_t)b * V, (uint32_t)V * 64u, bar);
  }
  // my scratch: columns 8q+{0..3} depths, 8q+{4..7} accumulators
  float4* scr = reinterpret_cast<float4*>(smem + OFF_SCR) + tid;

  // ---- per-lane constants: 16 reference channels, the ray, my depth hypotheses -------------------------------
  float2 ref2[C / 8];
  {
    const float* rp = p.ref_feat + ((size_t)b * C + (size_t)h * (C / 4)) * HW + n;
#pragma unroll
    for (int c = 0; c < C / 8; ++c) ref2[c] = make_float2(ldg_f(rp + (size_t)(2 * c) * HW), ldg_f(rp + (size_t)(2 * c + 1) * HW));
  }
  const float r0 = ldg_f(p.rays + ((size_t)b * 3 + 0) * HW + n);
  const float r1 = ldg_f(p.rays + ((size_t)b * 3 + 1) * HW + n);
  const float r2 = ldg_f(p.rays + ((size_t)b * 3 + 2) * HW + n);
  {
    float mu = 0.f, sg = 0.f;
    if (MODE == MAGNET_DEPTH_GAUSS) {
      mu = ldg_f(p.ref_gmm + ((size_t)b * 2 + 0) * HW + n);
      sg = ldg_f(p.ref_gmm + ((size_t)b * 2 + 1) * HW + n);
    }
#pragma unroll 1
    for (int m = 0; m < mend; m += 4) {
      float d[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int j = jb + min(m + e, max(nj - 1, 0));     // tail replicates my last hypothesis (never starts a cell)
        float v = 0.0f;
        if (nj > 0) {
          if (MODE == MAGNET_DEPTH_VOLUME) v = ldg_f(p.d_volume + ((size_t)b * D + jc + j) * HW + n);
          else if (MODE == MAGNET_DEPTH_GAUSS) v = __fadd_rn(mu, __fmul_rn(sg, ks[j]));   // MAGNET.py:155: mul, then add
          else v = ks[j];
        }
        d[e] = v;
      }
      scr_at(scr, 2 * m) = make_float4(d[0], d[1], d[2], d[3]);
      scr_at(scr, 2 * m + 4) = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
  }
  mbar_wait(bar, 0);                                       // camera table landed
  uint32_t phase = 1;
  int it = 0;                                              // valid views processed so far (bbox slot = it & 1)

  for (int v = 0; v < V; ++v) {
    const magnet_camera* cam = cams_s + v;                 // V <= TMAXV is checked on the host
    if (cam->valid != 1.0f) continue;                      // CTA-uniform
    ViewGeom g;
    g.a0 = cam->a[0]; g.a1 = cam->a[1]; g.a2 = cam->a[2];
    g.q0 = __fmaf_rn(cam->A[2], r2, __fmaf_rn(cam->A[1], r1, __fmul_rn(cam->A[0], r0)));
    g.q1 = __fmaf_rn(cam->A[5], r2, __fmaf_rn(cam->A[4], r1, __fmul_rn(cam->A[3], r0)));
    g.q2 = __fmaf_rn(cam->A[8], r2, __fmaf_rn(cam->A[7], r1, __fmul_rn(cam->A[6], r0)));
    const int vb = src_image<IDX>(src_index, b, v, p.B, V);
    const unsigned char* img = reinterpret_cast<const unsigned char*>(p.src_feat) + (size_t)vb * HW * PS + h * QL * 16;

    // ---------------- phase A + bounding box of the CTA's cells ---------------------------------------------
    int box[4];
    LaneCells lc = phase_a(g, scr, mend, nj, jb, 0, Dc, W, H, lane, pxl, stg, org, box);
    int* bb = bbox + (it & 1) * 4;
    if (lane == 0) {
      atomicMin(bb + 0, box[0]); atomicMax(bb + 1, box[1]); atomicMin(bb + 2, box[2]); atomicMax(bb + 3, box[3]);
    }
    __syncthreads();                                       // box complete; every warp is done with the previous window
    const int wx0 = bb[0], wy0 = bb[2];
    const int ww = bb[1] - wx0 + 2, wh = bb[3] - wy0 + 2;   // +1: right / lower taps of the last cells
    const int nxb = (ww + 7) >> 3;
    const bool staged = nxb * wh <= win_cap;
    if (tid == 0) {                                        // re-arm the other slot for the next view
      int* nb = bbox + ((it + 1) & 1) * 4;
      nb[0] = nb[2] = 1 << 30;
      nb[1] = nb[3] = -(1 << 30);
    }
    ++it;
    const int row_bytes = nxb * BOX;
    const int cbase = OFF_WIN + h * QL * 16 - (wy0 * row_bytes + wx0 * PS);
    if (staged) {
      // one elected lane per warp issues its share of the 8-pixel boxes (uniform-datapath instructions: a per-lane
      // loop would be serialised by the compiler anyway); thread 0 arms the barrier with the byte count — the
      // transaction count may run negative until then, the phase cannot complete before the arrival
      const int nops = nxb * wh;
      if (tid == 0) mbar_arrive_expect_tx(bar, (uint32_t)nops * BOX);
      if (lane == 0) {
        int r = warp / nxb, xb = warp - r * nxb;
        for (int op = warp; op < nops; op += TNT / 32) {
          tma_load_4d(smem_u32(win) + (uint32_t)op * BOX, &tmap, bar, 0, wx0 + 8 * xb, wy0 + r, vb);
          xb += TNT / 32;
          while (xb >= nxb) { xb -= nxb; ++r; }
        }
      }
      __syncwarp();
      mbar_wait(bar, phase);
      phase ^= 1u;
    }
    int jlo = 0;
    while (true) {                                         // one trip unless a pixel has > NORG cells (warp-uniform)
      const int nmax = __reduce_max_sync(FULL, lc.ncell);
      CornerState cs;
      cs.px0 = cs.py0 = -1000000;
      cs.c00 = cs.c01 = cs.c10 = cs.c11 = 0.0f;
      for (int i0 = 0; i0 < nmax; i0 += NCP) {             // NCP cells at a time (one pass for most warps)
        const int i1 = min(i0 + NCP, nmax);
        if (staged && jlo == 0)
          phase_b<C, CW, true>(ref2, lc.ncell, i0, i1, cs, lane, pxl, org, rec, smem, cbase, img, row_bytes, wx0, wy0, W, H);
        else
          phase_b<C, CW, false>(ref2, lc.ncell, i0, i1, cs, lane, pxl, org, rec, smem, 0, img, W * PS, 0, 0, W, H);
        phase_c<CW>(g, scr, mend, lc, jb, i0, p.kappa, pxl, org, rec);
      }
      if (!__any_sync(FULL, lc.jstop < Dc)) break;
      jlo = lc.jstop;                                      // restart the walk behind the last covered hypothesis;
      lc = phase_a(g, scr, mend, nj, jb, jlo, Dc, W, H, lane, pxl, stg, org, box);   // (the window only covers the
                                                                                      //  first walk's cells: global taps)
    }
  }

  // -------- epilogue: 1/V mean over ALL views (homography.py:120) ---------------------------------------------
  {
    float* outp = p.out + ((size_t)b * D + jc + jb) * HW + n;
    const bool exact = p.inv_v_exact != 0.0f;              // V a power of two: the division is an exact scaling
#pragma unroll 1
    for (int m = 0; m < mend; m += 4) {
      const float4 av = scr_at(scr, 2 * m + 4);
      const float a[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (live && m + e < nj) outp[(size_t)(m + e) * HW] = exact ? a[e] * p.inv_v_exact : __fdiv_rn(a[e], p.vf);
    }
  }
}

// (N, C, H, W) [+ (N, 2, H, W) Gaussians] -> MAGNET_SRC_PIXC (N, H, W, C+4).  One CTA per 32 pixels of one image:
// coalesced 128-byte reads per channel plane, transposed through shared memory, one contiguous 32*(C+4)*4-byte write.
template <int C>
__global__ void __launch_bounds__(256) repack_pixc_kernel(const float* __restrict__ src, const float* __restrict__ gmm,
                                                           float* __restrict__ dst, int HW) {
  constexpr int PF = pix_floats(C);
  __shared__ float t[32 * (PF + 1)];
  const int xi = threadIdx.x & 31, cy = threadIdx.x >> 5;
  const size_t img = blockIdx.y;
  const int p0 = blockIdx.x * 32;
  const int pix = p0 + xi;
  for (int c = cy; c < PF; c += 8) {
    float v = 0.0f;
    if (pix < HW) {
      if (c < C) v = src[(img * C + c) * HW + pix];
      else if (c < C + 2 && gmm != nullptr) v = gmm[(img * 2 + (c - C)) * HW + pix];
    }
    t[xi * (PF + 1) + c] = v;
  }
  __syncthreads();
  const int npx = min(32, HW - p0);
  float* o = dst + (img * HW + p0) * PF;
  for (int f = threadIdx.x; f < npx * PF; f += 256) o[f] = t[(f / PF) * (PF + 1) + f % PF];
}

cudaError_t launch_repack_pixc(const float* src, const float* gmm, float* dst, int N, int C, int H, int W,
                               cudaStream_t st) {
  const int HW = H * W;
  dim3 grid((HW + 31) / 32, N), block(256);
  switch (C) {
    case 16: repack_pixc_kernel<16><<<grid, block, 0, st>>>(src, gmm, dst, HW); break;
    case 32: repack_pixc_kernel<32><<<grid, block, 0, st>>>(src, gmm, dst, HW); break;
    case 64: repack_pixc_kernel<64><<<grid, block, 0, st>>>(src, gmm, dst, HW); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
// rank-4 map over the PIXC buffer: (C+4 floats, W, H, N), box = one row of 8 pixels, zero fill outside
static cudaError_t make_pixc_map(CUtensorMap* tm, const float* src, int N, int C, int H, int W) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) return cudaErrorNotSupported;
  const cuuint64_t ps = (cuuint64_t)pix_floats(C) * 4;
  const cuuint64_t dims[4] = {(cuuint64_t)pix_floats(C), (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t strides[3] = {ps, ps * W, ps * W * H};
  const cuuint32_t box[4] = {(cuuint32_t)pix_floats(C), 8u, 1u, 1u};
  const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(src), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

template <int C, int MODE, bool CW, bool IDX>
static cudaError_t launch_tma(const CostParams& p, const int32_t* src_index, int n_src, cudaStream_t st) {
  static std::once_flag flags[64];
  auto kern = cost_tma_kernel<C, MODE, CW, IDX>;
  cudaError_t e = set_smem_once(kern, flags, TMA_SMEM_TOTAL, true);
  if (e != cudaSuccess) return e;
  CUtensorMap tm;
  e = make_pixc_map(&tm, p.src_feat, IDX ? n_src : p.B * p.V, C, p.H, p.W);
  if (e != cudaSuccess) return e;
  const int nchunks = (p.D + TCH - 1) / TCH;
  const int tiles = ((p.W + TTW - 1) / TTW) * ((p.H + TTH - 1) / TTH);
  dim3 grid(tiles * nchunks, p.B), block(TNT);
#ifdef MAGNET_TMA_FORCE_GLOBAL   // debug build: never stage a window (all taps through the global-memory path)
  const int cap = 0;
#else
  const int cap = tma_win_cap(C);
#endif
  kern<<<grid, block, TMA_SMEM_TOTAL, st>>>(p, tm, cap, nchunks, src_index);
  return cudaGetLastError();
}

bool tma_supports(int C, int D, int V, int layout) {
  return (C == 16 || C == 32 || C == 64) && layout == MAGNET_SRC_PIXC && D >= 1 && V <= TMAXV;
}

void tma_launch_info(int B, int H, int W, int D, int* grid, int* block, int* smem) {
  *grid = ((W + TTW - 1) / TTW) * ((H + TTH - 1) / TTH) * ((D + TCH - 1) / TCH) * B;
  *block = TNT;
  *smem = TMA_SMEM_TOTAL;
}

// src_index: NULL (view-major source images, V*B of them) or the (B, V) frame table over n_src images
cudaError_t launch_cost_tma(const CostParams& p, int mode, int C, bool cw, const int32_t* src_index, int n_src,
                            cudaStream_t st, int* launches) {
  *launches = 1;
  return dispatch([&](auto c, auto m, auto w, auto idx) { return launch_tma<c, m, w, idx>(p, src_index, n_src, st); },
                  Choice<int, 16, 32, 64>{C}, DepthMode{mode}, Flag{cw}, Flag{src_index != nullptr});
}

}  // namespace magnet
