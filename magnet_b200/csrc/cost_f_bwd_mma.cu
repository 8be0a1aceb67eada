// Tensor-core backward of the fronto-parallel plane-sweep volume (homography.est_costvolume_F, homography.py:10-75)
// w.r.t. both feature maps, on the MAGNET_SRC_SPLIT16 operands of the forward (cost_mma.cu) — F-Net training
// (train_FNet.py:95-114).  The same kernel, instantiated with per-pixel depths and the consistency mask, gives the feature
// gradients of the CW volume (est_costvolume_CW) after a tensor-core forward (DESIGN §3.5).
//
// With g = dL/dscore (the workspace of score_grad_kernel, already divided by V) and w_t(p, j) the bilinear weights of
// plane j at reference pixel p in source view v, the gradients are the transpose of the forward's all-pairs product
// G[p][cell] = <ref_p, src_cell> (DESIGN §3.1):
//     Gc_v[p][cell] = sum_j sum_t g[p,j] w_t(p,j) [tap_t(p,j) == cell]     coefficient matrix, 64 pixels x window cells
//     g_ref[p][:]   += sum_v Gc_v[p][:] S_v[window][:]                       GEMM 1: M = 64 pixels, N = 64 channels, K = cells
//     g_src_v[cell][:] += sum_p Gc_v[p][cell] R[p][:]                         GEMM 2: M = cells, N = 64 channels, K = 64 pixels
//
//   * work item = (batch element, 8x8 tile) on persistent CTAs (two per SM) with a graph-replay-safe work counter (the
//     scheme of cost_mma.cu, own slots).  The item loops over the valid views and all D planes, so g_ref of the tile has
//     one owner and is written once, without atomics.
//   * window: positions are clamped to [-2, W+1] x [-2, H+1] as in the forward; only (pixel, plane) pairs whose cell
//     touches the image and whose g is nonzero can contribute, so the bounding box (warp reduction) is taken over those.
//     A box wider than 128 cells is cut into sub-windows of <= 16 eight-cell segments that overlap by one cell column /
//     row; a (pixel, plane) contributes in the sub-window that holds its cell origin, so its four taps lie inside.
//     Sub-windows that hold no cell origin (SID planes from min_depth = 1e-3 spread a tile along an epipolar line) are
//     skipped through an occupancy bitmap.
//   * Gc is accumulated in fp32 shared memory (red.shared.add.f32), then split once into fp16 hi / lo with ONE power-of-
//     two scale per work item, from max_p sum_j |g[p,j]|: that bounds every entry because the bilinear weights sum to one,
//     so GEMM 1 accumulates across all views and sub-windows in one register accumulator.  The fp16 Gc is stored as
//     rows of one cell x 64 pixels (128 bytes, 128-byte swizzle): GEMM 1 reads it as the MN-major (transposed) A operand,
//     GEMM 2 as the K-major A operand — one copy serves both.
//   * operands by TMA, same tensor maps and boxes as the forward: the source window (8-cell segments, hi atom | lo atom,
//     2048 bytes apart) and the reference tile (8 pixel rows of 1024 bytes per plane).  In both GEMMs they are the B
//     operand with the 64 channels as the contiguous N dimension: the MN-major form of the 128-byte-swizzle atom, whose
//     descriptor stride byte offset is the distance of consecutive 8-row K groups (2048 and 1024 bytes).
//   * three products hi*hi + hi*lo + lo*hi per GEMM (no lo*lo), fp32 accumulation; epilogues multiply by the exact
//     1 / (s_G s_src) and 1 / (s_G s_ref).  GEMM 1's K steps are split between the two warpgroups (summed in shared
//     memory at the end of the item); GEMM 2's two 64-cell M tiles go one to each warpgroup.
//   * g_src epilogue: cells outside the image are dropped, the others are added into the caller-zeroed NCHW grad_src
//     with red.global.add.f32 — results are NOT bit-deterministic from run to run (the order of the additions varies),
//     exactly like cost_f_bwd.cu and torch's grid_sample backward.
//
// Shared memory: reference tile 16 KB + one 32 KB region that holds fp32 Gc, then (Gc dead) the source window, then the
// g_ref partial sums + fp16 Gc 32 KB + tables: ~83 KB, two CTAs per SM (DESIGN §3.4).
#include <cuda_fp16.h>

#include <algorithm>
#include <atomic>
#include <mutex>

#include "cells_common.cuh"
#include "cw_mask.cuh"
#include "tma_common.cuh"

namespace magnet {

constexpr int BNT = 256;                 // threads: thread t handles pixel t % 64 of the tile, planes j = t / 64 (mod 4)
constexpr int BTW = 8, BTH = 8;          // tile in reference pixels
constexpr int BSEG = 16;                 // 8-cell segments per sub-window: <= 128 cells = two m64 tiles of GEMM 2
constexpr int BSEG_BYTES = 2048;         // hi atom (8 cells x 128 B) + lo atom
constexpr int BMAP_WORDS = 128;          // occupancy bitmap: up to 4096 sub-windows per view (else all are visited)

// shared-memory map (bytes from the 1024-aligned base)
constexpr int BOFF_REF = 0;                        // reference tile: hi 8 KB | lo 8 KB
constexpr int BOFF_WIN = 16384;                    // fp32 Gc [128 cells][64 px] -> source window -> g_ref [64 c][65]
constexpr int BOFF_G16 = BOFF_WIN + 32768;         // fp16 Gc hi [128 cells][64 px] | lo, 128-byte swizzle
constexpr int BOFF_PART = BOFF_G16 + 32768;        // float[4][64]: row sums of |g|
constexpr int BOFF_MAP = BOFF_PART + 1024;         // unsigned[BMAP_WORDS]
constexpr int BOFF_MISC = BOFF_MAP + BMAP_WORDS * 4;   // int[2 slots][4] box, [8] bound bits, [9] next item; 2 mbarriers
constexpr int B_SMEM_USED = BOFF_MISC + 64;
constexpr int B_SMEM_TOTAL = B_SMEM_USED + 1024;   // slack for the 1024-byte alignment of the base
static_assert(BSEG * BSEG_BYTES == 32768 && 128 * 64 * 4 == 32768 && 64 * 65 * 4 <= 32768, "region WIN");
static_assert(2 * (B_SMEM_TOTAL + 1024) <= 227 * 1024, "two CTAs per SM");

constexpr int FB_SLOTS = 1024;
__device__ unsigned g_fbwd_next[FB_SLOTS];
__device__ unsigned g_fbwd_done[FB_SLOTS];

// debug dump (MAGNET_MMA_DEBUG builds): header, fp32 Gc, GEMM 2 and both warpgroups' GEMM 1 accumulators of the first
// processed sub-window of work item 0, handed in through magnet_f_bwd_mma_debug_buffer
#ifdef MAGNET_MMA_DEBUG
constexpr int FDBG_GC = 16, FDBG_G2 = FDBG_GC + 128 * 64, FDBG_G1 = FDBG_G2 + 128 * 64;   // FDBG_G1 + 2 * 64 * 64 floats in all
#endif

// The forward's consistency test (cost_mma.cu) of a sample at (ix, iy) with source depth z, cell (x0, y0) touching the
// image: (mu, sigma) taps from the split buffer's paired table of the view (entry x0 + 1 <-> cell x0, zeros outside),
// the helpers of cw_mask.cuh.  Not inlined: the call keeps the mask's temporaries out of the GEMM loop's registers.
__device__ __noinline__ bool table_keep(const float4* __restrict__ meta, float ix, float iy, float z, int x0, int y0,
                                        int W, int H, float kappa) {
  float xf, yf, fx, fy;
  cell_split(ix, xf, fx);
  cell_split(iy, yf, fy);
  const float4* row = meta + (size_t)y0 * (W + 1) + (x0 + 1);
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  const float4 top = y0 >= 0 ? __ldg(row) : zero, bot = y0 + 1 < H ? __ldg(row + (W + 1)) : zero;
  return cw_keep(z, lerp2d_x2(top, bot, fx, fy), kappa);
}

// P = BwdParams, MODE = PLANES, CW = false: the F volume.  P = CwBwdParams (MODE VOLUME or GAUSS, CW = true): the CW
// volume, whose depths are per pixel and whose (pixel, hypothesis) pairs count only where the forward's consistency
// mask kept them (p.cw == 1): the mask is evaluated with the helpers of cw_mask.cuh on the (mu, sigma) table of the
// source SPLIT16 buffer, exactly as cost_mma.cu evaluates it.
template <class P, int MODE, bool CW>
__global__ void __launch_bounds__(BNT, 2)
cost_f_bwd_mma_kernel(const __grid_constant__ P p, const __grid_constant__ CUtensorMap tm_ref,
                      const __grid_constant__ CUtensorMap tm_src, const int n_items, const int slot,
                      float* __restrict__ dbg) {
  extern __shared__ unsigned char smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t padb = (1024u - (raw & 1023u)) & 1023u;
  unsigned char* smem = smem_raw + padb;
  const uint32_t sbase = raw + padb;
  float* gc = reinterpret_cast<float*>(smem + BOFF_WIN);
  float* part = reinterpret_cast<float*>(smem + BOFF_PART);
  unsigned* occ = reinterpret_cast<unsigned*>(smem + BOFF_MAP);
  int* misc = reinterpret_cast<int*>(smem + BOFF_MISC);
  const uint32_t bar_ref = sbase + BOFF_MISC + 48, bar_win = sbase + BOFF_MISC + 56;
  const unsigned FULL = 0xffffffffu;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2;
  const int H = p.H, W = p.W, HW = p.HW, D = p.D, V = p.V;
  const int tiles_x = (W + BTW - 1) / BTW, tiles = tiles_x * ((H + BTH - 1) / BTH);
  const Split16Header* hdr_ref = reinterpret_cast<const Split16Header*>(p.ref_feat);
  const Split16Header* hdr_src = reinterpret_cast<const Split16Header*>(p.src_feat);

  if (tid == 0) {
    mbar_init(bar_ref, 1);
    mbar_init(bar_win, 1);
    fence_mbar_init();
    prefetch_tmap(&tm_ref);
    prefetch_tmap(&tm_src);
  }
  if (tid < 8) misc[tid] = (tid & 1) ? -(1 << 28) : (1 << 28);     // [slot][x_lo, x_hi, y_lo, y_hi]
  __syncthreads();
  uint32_t ph_ref = 0, ph_win = 0;
  int it = 0;
#ifdef MAGNET_MMA_DEBUG
  bool dumped = false;
#endif
  const float xmax = (float)W + 1.0f, ymax = (float)H + 1.0f;
  const int pp = tid & 63, jg = tid >> 6;

  int item = blockIdx.x;
  while (item < n_items) {
  const int b = item / tiles, tile = item - b * tiles;
  const int tx0 = (tile % tiles_x) * BTW, ty0 = (tile / tiles_x) * BTH;
  if (tid == 0) {
    // every reader of the tile region and of misc[8..9] passed the barrier that ended the previous item
    mbar_arrive_expect_tx(bar_ref, 16384u);
    tma_load_5d(sbase + BOFF_REF, &tm_ref, bar_ref, 0, tx0, ty0, 0, b);
    misc[8] = 0;
    misc[9] = (int)gridDim.x + (int)atomicAdd(&g_fbwd_next[slot], 1u);
  }
  const int px = tx0 + (pp & 7), py = ty0 + (pp >> 3);
  const bool live = px < W && py < H;
  const int n = min(py, H - 1) * W + min(px, W - 1);
  const float r0 = ldg_f(p.rays + ((size_t)b * 3 + 0) * HW + n);
  const float r1 = ldg_f(p.rays + ((size_t)b * 3 + 1) * HW + n);
  const float r2 = ldg_f(p.rays + ((size_t)b * 3 + 2) * HW + n);
  const float* gs = p.g_score + (size_t)b * D * HW + n;

  // ---- per-item scale of Gc: every entry of row p is bounded by sum_j |g[p,j]| (the bilinear weights sum to one) ----
  {
    float s = 0.0f;
    if (live)
      for (int j = jg; j < D; j += 4) s += fabsf(ldg_f(gs + (size_t)j * HW));
    part[jg * 64 + pp] = s;
  }
  __syncthreads();
  if (tid < 64) {
    const float s = (part[tid] + part[64 + tid]) + (part[128 + tid] + part[192 + tid]);
    const unsigned u = __reduce_max_sync(FULL, __float_as_uint(s));     // non-negative floats order as integers
    if (lane == 0) atomicMax(reinterpret_cast<unsigned*>(misc + 8), u);
  }
  __syncthreads();
  const unsigned bound = (unsigned)misc[8];
  const int eb = (int)(bound >> 23) & 0xff;
  const int shg = (eb == 0 || eb == 255) ? 0 : max(-100, min(100, 14 - (eb - 127)));   // bound * s_G in [2^14, 2^15)
  const float s_g = __uint_as_float((unsigned)(127 + shg) << 23), inv_sg = __uint_as_float((unsigned)(127 - shg) << 23);

  float acc1[32];
#pragma unroll
  for (int e = 0; e < 32; ++e) acc1[e] = 0.0f;
  bool ref_ready = false;

  for (int v = 0; v < V && bound != 0u; ++v) {             // an all-zero g contributes nothing
    const magnet_camera* cam = p.cams + (b * V + v);
    if (cam->valid != 1.0f) continue;                      // CTA-uniform
    const float a0 = cam->a[0], a1 = cam->a[1], a2 = cam->a[2];
    const float q0 = __fmaf_rn(cam->A[2], r2, __fmaf_rn(cam->A[1], r1, __fmul_rn(cam->A[0], r0)));
    const float q1 = __fmaf_rn(cam->A[5], r2, __fmaf_rn(cam->A[4], r1, __fmul_rn(cam->A[3], r0)));
    const float q2 = __fmaf_rn(cam->A[8], r2, __fmaf_rn(cam->A[7], r1, __fmul_rn(cam->A[6], r0)));
    const int vb = v * p.B + b;
    const float4* meta = nullptr;                          // (mu, sigma) table of the source split buffer (CW)
    if constexpr (CW)
      meta = reinterpret_cast<const float4*>(reinterpret_cast<const unsigned char*>(p.src_feat) + SPLIT16_HEADER +
                                             (size_t)p.B * V * HW * 256);
    // cell origin of plane j at my pixel, and whether it can contribute (a tap in the image, g != 0)
    auto cell = [&](const int j, float& g, float& ix, float& iy, int& x0, int& y0) -> bool {
      g = ldg_f(gs + (size_t)j * HW);
      float z, d;
      if constexpr (MODE == MAGNET_DEPTH_VOLUME) d = ldg_f(p.d_volume + ((size_t)b * D + j) * HW + n);
      else if constexpr (MODE == MAGNET_DEPTH_GAUSS)     // MAGNET.py:155 (the pixel's Gaussian is re-read: registers)
        d = __fadd_rn(ldg_f(p.ref_gmm + ((size_t)b * 2 + 0) * HW + n),
                      __fmul_rn(ldg_f(p.ref_gmm + ((size_t)b * 2 + 1) * HW + n), p.k[j]));
      else d = p.k[j];
      project(d, a0, a1, a2, q0, q1, q2, ix, iy, z);
      clamp_pos(ix, iy, xmax, ymax);
      x0 = (int)floorf(ix);
      y0 = (int)floorf(iy);
      bool ok = live && g != 0.0f && x0 >= -1 && x0 < W && y0 >= -1 && y0 < H;
      if constexpr (CW) {
        if (ok && p.cw) ok = table_keep(meta + (size_t)vb * H * (W + 1), ix, iy, z, x0, y0, W, H, p.kappa);
      }
      return ok;
    };

    // ---------------- pass 1: bounding box of the contributing cell origins ----------------------------------------
    int* bb = misc + (it & 1) * 4;
    {
      int xl = 1 << 28, xh = -(1 << 28), yl = 1 << 28, yh = -(1 << 28);
      for (int j = jg; j < D; j += 4) {
        float g, ix, iy;
        int x0, y0;
        if (cell(j, g, ix, iy, x0, y0)) { xl = min(xl, x0); xh = max(xh, x0); yl = min(yl, y0); yh = max(yh, y0); }
      }
      xl = __reduce_min_sync(FULL, xl); xh = __reduce_max_sync(FULL, xh);
      yl = __reduce_min_sync(FULL, yl); yh = __reduce_max_sync(FULL, yh);
      if (lane == 0) { atomicMin(bb + 0, xl); atomicMax(bb + 1, xh); atomicMin(bb + 2, yl); atomicMax(bb + 3, yh); }
    }
    for (int i = tid; i < BMAP_WORDS; i += BNT) occ[i] = 0u;
    __syncthreads();
    const int wx0 = bb[0], wx1 = bb[1], wy0 = bb[2], wy1 = bb[3];
    if (tid < 4) misc[((it + 1) & 1) * 4 + tid] = (tid & 1) ? -(1 << 28) : (1 << 28);   // re-arm the other slot
    ++it;
    if (wx0 > wx1) continue;                               // nothing of this view reaches the image (CTA-uniform)
    // sub-windows as in the forward, with <= BSEG segments (at least two rows: <= 8 segments wide)
    const int nseg_all = (wx1 - wx0 + 2 + 7) >> 3, rows_all = wy1 - wy0 + 2;
    const int nsw = min(nseg_all, BSEG / 2);
    const int rmax = nseg_all * rows_all <= BSEG ? rows_all : max(2, BSEG / nsw);
    const int stepx = 8 * nsw - 1, stepy = rmax - 1;
    const int nsx = (wx1 - wx0) / stepx + 1, nsy = (wy1 - wy0) / stepy + 1, nsub = nsx * nsy;
    const bool map = nsub > 1 && nsub <= BMAP_WORDS * 32;

    // ---------------- pass 2: which sub-windows hold a contributing cell origin ------------------------------------
    if (map) {
      for (int j = jg; j < D; j += 4) {
        float g, ix, iy;
        int x0, y0;
        if (cell(j, g, ix, iy, x0, y0)) {
          const int si = ((y0 - wy0) / stepy) * nsx + (x0 - wx0) / stepx;
          atomicOr(occ + (si >> 5), 1u << (si & 31));
        }
      }
      __syncthreads();
    }

    for (int si = 0; si < nsub; ++si) {
      if (map && !((occ[si >> 5] >> (si & 31)) & 1u)) continue;   // CTA-uniform
      const int syi = si / nsx, sxi = si - syi * nsx;
      const int sx = wx0 + sxi * stepx, sy = wy0 + syi * stepy;
      const int rows = min(stepy, wy1 - sy + 1) + 1;
      const int nseg = (min(stepx, wx1 - sx + 1) + 1 + 7) >> 3;
      const int nsegs = nseg * rows, ncells = nsegs * 8, pitch = nseg * 8;
      const int nrow = (ncells + 63) & ~63;                // rows of Gc the GEMMs read (M tiles of 64)

      // ---------------- Gc in fp32: zero, then red.shared.add of g * w_t at the four taps ---------------------------
      float4* gc4 = reinterpret_cast<float4*>(gc);
      for (int i = tid; i < nrow * 16; i += BNT) gc4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      __syncthreads();
      for (int j = jg; j < D; j += 4) {
        float g, ix, iy;
        int x0, y0;
        if (cell(j, g, ix, iy, x0, y0) && (x0 - wx0) / stepx == sxi && (y0 - wy0) / stepy == syi) {
          const float fx = ix - floorf(ix), fy = iy - floorf(iy);
          const float wx0f = 1.0f - fx, wy0f = 1.0f - fy;
          float* c00 = gc + ((y0 - sy) * pitch + (x0 - sx)) * 64 + pp;
          atomicAdd(c00, g * (wx0f * wy0f));
          atomicAdd(c00 + 64, g * (fx * wy0f));
          atomicAdd(c00 + pitch * 64, g * (wx0f * fy));
          atomicAdd(c00 + pitch * 64 + 64, g * (fx * fy));
        }
      }
      __syncthreads();
#ifdef MAGNET_MMA_DEBUG
      const bool dump = dbg != nullptr && item == 0 && !dumped;
      if (dump) {
        if (tid == 0) {
          dbg[0] = (float)sx; dbg[1] = (float)sy; dbg[2] = (float)nseg; dbg[3] = (float)rows; dbg[4] = (float)ncells;
          dbg[5] = (float)v; dbg[6] = s_g; dbg[7] = hdr_ref->inv_scale; dbg[8] = hdr_src->inv_scale; dbg[9] = (float)tx0;
          dbg[10] = (float)ty0; dbg[11] = (float)b;
        }
        for (int i = tid; i < ncells * 64; i += BNT) dbg[FDBG_GC + i] = gc[i];
      }
#endif
      // ---------------- split: fp16 hi / lo of Gc * s_G, rows of one cell x 64 pixels, 128-byte swizzle -------------
      for (int i = tid; i < nrow * 8; i += BNT) {
        const int row = i >> 3, ch = i & 7;                // cell, 8-pixel chunk
        const float4 u = gc4[row * 16 + ch * 2], w = gc4[row * 16 + ch * 2 + 1];
        const float x[8] = {u.x, u.y, u.z, u.w, w.x, w.y, w.z, w.w};
        __align__(16) __half hi[8], lo[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float s = x[e] * s_g;                      // exact: power of two
          hi[e] = __float2half_rn(s);
          lo[e] = __float2half_rn(s - __half2float(hi[e]));
        }
        const int off = row * 128 + ((ch ^ (row & 7)) << 4);
        *reinterpret_cast<uint4*>(smem + BOFF_G16 + off) = *reinterpret_cast<const uint4*>(hi);
        *reinterpret_cast<uint4*>(smem + BOFF_G16 + 16384 + off) = *reinterpret_cast<const uint4*>(lo);
      }
      fence_proxy_async();
      __syncthreads();                                     // fp16 Gc complete, fp32 Gc dead: the window may land on it
      // ---------------- source window by TMA (an odd segment count is padded with a box wholly outside the image,
      // which the copy engine fills with zeros: the last K step of GEMM 1 spans two segments) -------------------------
      const int nload = nsegs + (nsegs & 1);
      if (tid == 0) mbar_arrive_expect_tx(bar_win, (uint32_t)nload * BSEG_BYTES);
      if (lane == 0) {
        for (int s = warp; s < nload; s += BNT / 32) {
          const int r = s / nseg, xb = s - r * nseg;
          const int cx = s < nsegs ? sx + 8 * xb : -64, cy = s < nsegs ? sy + r : -64;
          tma_load_5d(sbase + BOFF_WIN + (uint32_t)s * BSEG_BYTES, &tm_src, bar_win, 0, cx, cy, 0, vb);
        }
      }
      __syncwarp();
      mbar_wait_or_trap(bar_win, ph_win);
      ph_win ^= 1u;
      if (!ref_ready) {                                    // CTA-uniform
        mbar_wait_or_trap(bar_ref, ph_ref);
        ph_ref ^= 1u;
        ref_ready = true;
      }
      // ---------------- GEMM 1 (K steps split between the warpgroups) and GEMM 2 (M tile = warpgroup) ----------------
      {
        const uint32_t g_hi = sbase + BOFF_G16, g_lo = g_hi + 16384;
        const uint32_t w_hi = sbase + BOFF_WIN, w_lo = w_hi + 1024;
        const uint32_t r_hi = sbase + BOFF_REF, r_lo = r_hi + 8192;
        const int nk = (ncells + 15) >> 4, nk0 = (nk + 1) >> 1;
        const int k_lo = wg == 0 ? 0 : nk0, k_hi = wg == 0 ? nk0 : nk;
        const bool m_on = wg * 64 < ncells;
        float acc2[32];
#pragma unroll
        for (int e = 0; e < 32; ++e) acc2[e] = 0.0f;
        __syncwarp();
        wgmma_fence();
        // g_ref[p][c] += sum_cell Gc[p][cell] S[cell][c]: A = Gc (M = pixels contiguous), B = window (N = channels
        // contiguous), both MN-major; a K step of 16 cells = two atoms
        for (int kk = k_lo; kk < k_hi; ++kk) {
          const uint64_t ah = gmma_desc_sw128(g_hi + kk * 2048, 1024), al = gmma_desc_sw128(g_lo + kk * 2048, 1024);
          const uint64_t bh = gmma_desc_sw128(w_hi + kk * 4096, BSEG_BYTES), bl = gmma_desc_sw128(w_lo + kk * 4096, BSEG_BYTES);
          wgmma_m64n64k16_f16<1, 1>(acc1, al, bh);
          wgmma_m64n64k16_f16<1, 1>(acc1, ah, bl);
          wgmma_m64n64k16_f16<1, 1>(acc1, ah, bh);
        }
        // g_src[cell][c] = sum_p Gc[p][cell] R[p][c]: A = Gc K-major (the K step of 16 pixels is +32 bytes inside the
        // swizzle row), B = reference tile MN-major (a K step = two pixel rows)
        if (m_on) {
          const uint64_t ah = gmma_desc_sw128(g_hi + wg * 8192, 1024), al = gmma_desc_sw128(g_lo + wg * 8192, 1024);
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const uint64_t bh = gmma_desc_sw128(r_hi + kk * 2048, 1024), bl = gmma_desc_sw128(r_lo + kk * 2048, 1024);
            wgmma_m64n64k16_f16<0, 1>(acc2, al + 2u * kk, bh);
            wgmma_m64n64k16_f16<0, 1>(acc2, ah + 2u * kk, bl);
            wgmma_m64n64k16_f16<0, 1>(acc2, ah + 2u * kk, bh);
          }
        }
        wgmma_commit();
        wgmma_wait_all();
#ifdef MAGNET_MMA_DEBUG
        if (dump) {
          const int rr = 16 * (warp & 3) + (lane >> 2);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int c = 8 * j + 2 * (lane & 3);
            for (int h = 0; h < 2; ++h) {
              const int li = wg * 64 + rr + 8 * h;
              if (li < ncells) {
                dbg[FDBG_G2 + li * 64 + c] = acc2[4 * j + 2 * h];
                dbg[FDBG_G2 + li * 64 + c + 1] = acc2[4 * j + 2 * h + 1];
              }
              dbg[FDBG_G1 + wg * 4096 + (rr + 8 * h) * 64 + c] = acc1[4 * j + 2 * h];
              dbg[FDBG_G1 + wg * 4096 + (rr + 8 * h) * 64 + c + 1] = acc1[4 * j + 2 * h + 1];
            }
          }
        }
        dumped = dumped || dump;
#endif
        // ---------------- g_src epilogue: cells inside the image, red.global.add, 1 / (s_G s_ref) -------------------
        if (m_on && (!CW || p.grad_src != nullptr)) {
          const float sc = hdr_ref->inv_scale * inv_sg;
          float* gsrc = p.grad_src + (size_t)vb * 64 * HW;
          const int rr = wg * 64 + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int li = rr + 8 * h;
            const int sg = li >> 3, r = sg / nseg;
            const int x = sx + 8 * (sg - r * nseg) + (li & 7), y = sy + r;
            if (li < ncells && x >= 0 && x < W && y >= 0 && y < H) {
              float* gp = gsrc + (size_t)y * W + x;
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const int c = 8 * j + 2 * (lane & 3);
                const float e0 = acc2[4 * j + 2 * h], e1 = acc2[4 * j + 2 * h + 1];
                if (e0 != 0.0f) atomicAdd(gp + (size_t)c * HW, e0 * sc);
                if (e1 != 0.0f) atomicAdd(gp + (size_t)(c + 1) * HW, e1 * sc);
              }
            }
          }
        }
      }
      __syncthreads();                                     // window and fp16 Gc are read: the next sub-window may write
    }
  }

  if (!ref_ready) {                                        // no GEMM ran: the reference-tile copy is still in flight
    mbar_wait_or_trap(bar_ref, ph_ref);
    ph_ref ^= 1u;
  }
  // -------- g_ref: the warpgroups' K halves summed in shared memory (region WIN is free), 1 / (s_G s_src), stored --------
  {
    float* st = gc;                                        // [64 channels][65]
    const int rr = 16 * (warp & 3) + (lane >> 2);
    for (int pass = 1; pass >= 0; --pass) {
      if (wg == pass) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = 8 * j + 2 * (lane & 3);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float* s0 = st + c * 65 + rr + 8 * h;
            float* s1 = s0 + 65;
            if (pass == 1) { *s0 = acc1[4 * j + 2 * h]; *s1 = acc1[4 * j + 2 * h + 1]; }
            else { *s0 += acc1[4 * j + 2 * h]; *s1 += acc1[4 * j + 2 * h + 1]; }
          }
        }
      }
      __syncthreads();
    }
    const float sc = hdr_src->inv_scale * inv_sg;
    for (int idx = tid; idx < 64 * 64 && (!CW || p.grad_ref != nullptr); idx += BNT) {
      const int c = idx >> 6, q = idx & 63;
      const int x = tx0 + (q & 7), y = ty0 + (q >> 3);
      if (x < W && y < H) p.grad_ref[((size_t)b * 64 + c) * HW + (size_t)y * W + x] = st[c * 65 + q] * sc;
    }
  }
  const int nxt = misc[9];                                 // written by thread 0 when this item began
  __syncthreads();                                         // staging and tables are free; misc may be rewritten
  item = nxt;
  }  // work items

  if (tid == 0) {                                          // the last CTA to finish re-arms the work counter
    __threadfence();
    if (atomicAdd(&g_fbwd_done[slot], 1u) == gridDim.x - 1) {
      g_fbwd_next[slot] = 0u;
      g_fbwd_done[slot] = 0u;
      __threadfence();
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
cudaError_t make_planes_map(CUtensorMap* tm, const void* planes, int N, int H, int W, int box_rows);   // cost_mma.cu
int sm_count(int dev);                                                                                 // cost_mma.cu
cudaError_t launch_score_grad(const BwdParams& p, cudaStream_t st);                                    // cost_f_bwd.cu

#ifdef MAGNET_MMA_DEBUG
static float* g_fbwd_dbg = nullptr;
void f_bwd_mma_set_debug_buffer(float* p) { g_fbwd_dbg = p; }
#endif

bool f_bwd_mma_supports(int C, int V) { return C == 64 && V >= 1 && V <= 16; }

void f_bwd_mma_launch_info(int B, int H, int W, int* grid, int* block, int* smem) {
  int dev = 0;
  cudaGetDevice(&dev);
  *grid = std::min(((W + BTW - 1) / BTW) * ((H + BTH - 1) / BTH) * B, 2 * sm_count(dev));
  *block = BNT;
  *smem = B_SMEM_TOTAL;
}

// work-counter tickets shared by every instantiation (they share the slots of g_fbwd_next / g_fbwd_done)
static std::atomic<unsigned> ticket{0}, graph_ticket{0};

// p.ref_feat / p.src_feat point to the SPLIT16 buffers of the forward (B and V*B images); p.g_score is written
template <class P, int MODE, bool CW>
static cudaError_t launch_bwd_mma(const P& p, cudaStream_t st) {
  static std::once_flag flags[64];
  auto kern = cost_f_bwd_mma_kernel<P, MODE, CW>;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  cudaError_t res = cudaSuccess;
  std::call_once(flags[dev & 63], [&] {
    res = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, B_SMEM_TOTAL);
    if (res == cudaSuccess)
      res = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  });
  if (res != cudaSuccess) return res;
  const unsigned char* refbuf = reinterpret_cast<const unsigned char*>(p.ref_feat);
  const unsigned char* srcbuf = reinterpret_cast<const unsigned char*>(p.src_feat);
  CUtensorMap tm_ref, tm_src;
  if ((e = make_planes_map(&tm_ref, refbuf + SPLIT16_HEADER, p.B, p.H, p.W, 8)) != cudaSuccess) return e;
  if ((e = make_planes_map(&tm_src, srcbuf + SPLIT16_HEADER, p.B * p.V, p.H, p.W, 1)) != cudaSuccess) return e;
  const int n_items = ((p.W + BTW - 1) / BTW) * ((p.H + BTH - 1) / BTH) * p.B;
  // work-counter slot: eager launches cycle through the lower half, captured launches own one of the upper half for
  // the life of their graph (cost_mma.cu)
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &cap) != cudaSuccess) cap = cudaStreamCaptureStatusNone;
  const int slot = cap == cudaStreamCaptureStatusActive ? FB_SLOTS / 2 + (int)(graph_ticket.fetch_add(1) % (FB_SLOTS / 2))
                                                        : (int)(ticket.fetch_add(1) % (FB_SLOTS / 2));
  float* dbg = nullptr;
#ifdef MAGNET_MMA_DEBUG
  dbg = g_fbwd_dbg;
#endif
  kern<<<std::min(n_items, 2 * sm_count(dev)), BNT, B_SMEM_TOTAL, st>>>(p, tm_ref, tm_src, n_items, slot, dbg);
  return cudaGetLastError();
}

cudaError_t launch_cost_f_bwd_mma(const BwdParams& p, cudaStream_t st, int* launches) {
  cudaError_t e = launch_score_grad(p, st);
  if (e != cudaSuccess) return e;
  *launches = 2;
  return launch_bwd_mma<BwdParams, MAGNET_DEPTH_PLANES, false>(p, st);
}

// CW volume, feature gradients on the tensor cores: p.ref_feat / p.src_feat are the forward's split buffers, p.g_score
// already holds grad_out / V (cost_cw_bwd.cu)
cudaError_t launch_cost_cw_bwd_mma(const CwBwdParams& p, int mode, cudaStream_t st) {
  if (mode == MAGNET_DEPTH_VOLUME) return launch_bwd_mma<CwBwdParams, MAGNET_DEPTH_VOLUME, true>(p, st);
  return launch_bwd_mma<CwBwdParams, MAGNET_DEPTH_GAUSS, true>(p, st);
}

}  // namespace magnet
