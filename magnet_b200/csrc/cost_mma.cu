// MAGNET_VARIANT_MMA — tensor-core kernel: fused warp + sample + consistency + view fusion with the channel dot
// products of a whole (tile, view) computed by wgmma (fp32 accumulators in registers).
//
// Replaces homography.py:79-161 (and :10-75 with CW == false); absorbs the sampler of MAGNET.py:154-156.
//
// Identity: sum_c ref_c (sum_t w_t src_tc) = sum_t w_t <ref, src_t>.  cost_cells.cu / cost_tma.cu find, per pixel, the
// ~6 bilinear cells its hypotheses visit and compute <ref, src_t> for exactly those taps on the CUDA cores — the
// bookkeeping (cell walk, records, lockstep over cells) costs 3x the instructions of the arithmetic.  Here the dot
// products of ALL (reference pixel, window cell) pairs of an 8x8 tile are one small GEMM,
//        G[p][c] = <ref_p, src_c>,  64 pixels x (<= 256 window cells) x 64 channels,
// ~12x more products than needed but on the tensor pipe, which is otherwise idle; what remains per hypothesis is the
// projection, four G[p][c] and two paired (mu, sigma) shared-memory reads and three bilinear interpolations.
//
//   * fp32 accuracy on fp16 tensor cores: every feature map is split once per forward into x*s = hi + lo (two fp16
//     planes, s a power of two that maps the largest finite |x| into [2^14, 2^15)); hi*hi + hi*lo + lo*hi carries 22
//     significant bits per factor, products are exact in the fp32 accumulator (MAGNET_SRC_SPLIT16,
//     magnet_repack_split16_f32).
//   * the planes are (image, plane, y, x, 64 channels) fp16 = 128-byte rows: an 8-pixel x 2-plane TMA box with
//     CU_TENSOR_MAP_SWIZZLE_128B lands as one canonical K-major wgmma atom per plane; the window of a (tile, view) is the
//     bounding box of the tile's sample positions cut into such 8-cell segments (zero fill outside the image =
//     grid_sample's padding_mode='zeros'), cell index = B-operand row = accumulator column.  The reference tile is the
//     A operand (M = 64); warpgroup g computes accumulator columns [128 g, 128 g + 128).
//   * one warp per tile row (8 pixels in turn), one LANE per hypothesis (lane j: hypotheses j and j + 32 of the
//     64-hypothesis chunk, evaluated side by side as float2 pairs): the pixel's constants are warp-uniform (per-warp table
//     in shared memory), the 32 lanes read a handful of neighbouring cells of ONE accumulator row (broadcast /
//     conflict-free); lanes beyond the last hypothesis replicate it, so there are no activity predicates.
//   * per view: project all hypotheses (exact bounding box) -> TMA window + paired (mu, sigma) table -> 12 x wgmma
//     m64n128k16 per warpgroup (3 products x 4 K steps) -> the 64 accumulator rows into shared memory (over the window,
//     which is dead by then) -> per-hypothesis phase, which projects again from the per-warp pixel table (the 32
//     positions do not fit the registers next to the 64 accumulators).  The view
//     accumulators live in shared memory (hypothesis-major: the layout the coalesced epilogue reads).
//   * a window that does not fit 256 cells is cut into sub-windows of <= 32 segments that overlap by one cell column /
//     row; a hypothesis is evaluated in the sub-window that holds its cell origin.  Same code for any depth distribution.
//   * persistent CTAs (two per SM): work items (batch element, tile, 64-hypothesis chunk) come from a global counter in a
//     per-launch slot that the last CTA re-arms (graph-replay safe); barriers are set up once per CTA.
//
// Numerics: the per-view channel sum is the tensor core's fp32 accumulation of exact products of the split factors
// (relative error ~2^-21 of sum |ref||src|, the same order as an fp32 FMA chain); everything else — projection, weights,
// consistency test, view accumulation, 1/V — is the fp32 arithmetic of the other kernels (common.cuh project2).
#include <cuda_fp16.h>

#include <algorithm>
#include <atomic>
#include <cstddef>
#include <mutex>
#include <type_traits>

#include "common.cuh"
#include "tma_common.cuh"
#include "cw_mask.cuh"

namespace magnet {

constexpr int MNT = 256;               // threads per CTA: warp w owns tile row w, pixel i of the row in turn
constexpr int MTW = 8, MTH = 8;        // CTA tile in reference pixels
constexpr int MPX = MTW * MTH;         // 64 = rows of the accumulator that are used
constexpr int MCH = 64;                // hypotheses per CTA (two per lane)
constexpr int MSEG = 32;               // 8-cell segments per window: N <= 256 accumulator columns
constexpr int MMAXV = 16;              // views whose camera constants are staged in shared memory
constexpr int SEG_BYTES = 2048;        // hi atom (8 cells x 128 B) + lo atom
constexpr int META_SEG_BYTES = 128;    // 8 cells x (mu, sigma of the cell and of its right neighbour)

// shared-memory map (bytes from the 1024-aligned base)
constexpr int MOFF_A = 0;                                   // reference tile: hi 8 KB | lo 8 KB
constexpr int MOFF_R = 16384;                               // window segments, later the accumulator rows G[64][GP]
constexpr int MR_BYTES = 67584;                             //   >= 32 * 2048 and >= 64 * 264 * 4
constexpr int MOFF_META = MOFF_R + MR_BYTES;                // float4[256] (mu, sigma)[c], (mu, sigma)[c + 1] per window cell
constexpr int MOFF_CAM = MOFF_META + MSEG * META_SEG_BYTES; // magnet_camera[MMAXV]
constexpr int MOFF_KS = MOFF_CAM + MMAXV * 64;              // float[MCH]
constexpr int MOFF_BBOX = MOFF_KS + MCH * 4;                // int[2 slots][4]
constexpr int MOFF_BAR = MOFF_BBOX + 64;                    // 2 mbarriers, next work item
constexpr int MOFF_ACC = MOFF_BAR + 64;                     // float[MCH][65]: view accumulators, hypothesis-major
constexpr int MOFF_PIX = MOFF_ACC + MCH * 65 * 4;           // float4[8 warps][8 pixels][2]: (q0,q1,q2,-) (q2,mu,sigma,-)
constexpr int M_SMEM_USED = MOFF_PIX + 8 * 8 * 32;
constexpr int M_SMEM_TOTAL = M_SMEM_USED + 1024;            // slack for the 1024-byte alignment of the base
static_assert(MR_BYTES >= MSEG * SEG_BYTES && MR_BYTES >= MPX * 264 * 4 && MR_BYTES >= MCH * 65 * 4, "region R");
static_assert(2 * (M_SMEM_TOTAL + 1024) <= 227 * 1024, "two CTAs per SM");

// header | fp16 planes (N, 2, H, W, 64) | table (N, H, W + 1, 4): entry x + 1 of a row = (mu, sigma)[x], (mu, sigma)[x + 1]
// with zeros outside the row — both horizontal taps of a bilinear cell in ONE 16-byte read
__host__ __device__ inline size_t split16_bytes(size_t N, size_t H, size_t W) {
  return SPLIT16_HEADER + N * H * W * 256 + N * H * (W + 1) * 16;
}

// work counters of the persistent kernel: one slot per launch in flight (host ticket), re-armed by the last CTA of the
// launch, so a captured launch can be replayed.  Launches that share a slot must not run concurrently: 512 eager
// launches or 512 captured ones would have to be in flight / alive at once.
constexpr int MMA_SLOTS = 1024;
__device__ unsigned g_mma_next[MMA_SLOTS];
__device__ unsigned g_mma_done[MMA_SLOTS];

// shared-memory loads by 32-bit shared address (the window / table offsets are computed as integers)
__device__ __forceinline__ float lds_f32(uint32_t a) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ float4 lds_f32x4(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
  return v;
}
template <int MODE, bool CW>
__global__ void __launch_bounds__(MNT, 2)
cost_mma_kernel(const __grid_constant__ CostParams p, const __grid_constant__ CUtensorMap tm_ref,
                const __grid_constant__ CUtensorMap tm_src, const __grid_constant__ CUtensorMap tm_meta, const int nchunks,
                const int n_items, const int slot, float* __restrict__ dbg) {
  extern __shared__ unsigned char smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t padb = (1024u - (raw & 1023u)) & 1023u;
  unsigned char* smem = smem_raw + padb;
  const uint32_t sbase = raw + padb;
  const magnet_camera* cams_s = reinterpret_cast<const magnet_camera*>(smem + MOFF_CAM);
  float* ks = reinterpret_cast<float*>(smem + MOFF_KS);
  int* bbox = reinterpret_cast<int*>(smem + MOFF_BBOX);
  float* regR = reinterpret_cast<float*>(smem + MOFF_R);
  const uint32_t bar_tma = sbase + MOFF_BAR, bar_cam = sbase + MOFF_BAR + 24;
  float* acc_s = reinterpret_cast<float*>(smem + MOFF_ACC);
  const unsigned FULL = 0xffffffffu;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int H = p.H, W = p.W, HW = p.HW, D = p.D, V = p.V;
  const int tiles_x = (W + MTW - 1) / MTW;
  const int items_per_b = tiles_x * ((H + MTH - 1) / MTH) * nchunks;

  const unsigned char* refbuf = reinterpret_cast<const unsigned char*>(p.ref_feat);
  const unsigned char* srcbuf = reinterpret_cast<const unsigned char*>(p.src_feat);
  const Split16Header* hdr_ref = reinterpret_cast<const Split16Header*>(refbuf);
  const Split16Header* hdr_src = reinterpret_cast<const Split16Header*>(srcbuf);
  volatile int* next_item = reinterpret_cast<volatile int*>(smem + MOFF_BAR + 40);

  // ---- once per CTA: barriers ---------------------------------------------------------------------------------
  if (tid == 0) {
    mbar_init(bar_tma, 1);
    mbar_init(bar_cam, 1);
    fence_mbar_init();
    prefetch_tmap(&tm_ref);
    prefetch_tmap(&tm_src);
    prefetch_tmap(&tm_meta);
  }
  if (tid < 8) bbox[tid] = (tid & 1) ? -(1 << 28) : (1 << 28);       // [slot][x_lo, x_hi, y_lo, y_hi]
  __syncthreads();
  uint32_t ph_tma = 0, ph_cam = 0;
  int it = 0;
  int cur_b = -1;
  const float xmax = (float)W + 1.0f, ymax = (float)H + 1.0f;
  const float kappa = p.kappa;
  const uint32_t g_row0 = sbase + MOFF_R, m_base = sbase + MOFF_META;

  // ---- persistent CTA: work items (batch element, tile, hypothesis chunk) are handed out dynamically -----------
  // (the first one is the block index, the others come from a global counter: no tail of a partial last wave, barriers
  // set up once per SM slot)
  int item = blockIdx.x;
  while (item < n_items) {
  const int b = item / items_per_b;
  const int rem = item - b * items_per_b;
  const int tile = rem / nchunks;
  const int jc = (rem - tile * nchunks) * MCH;
  const int Dc = min(MCH, D - jc);
  const int tx0 = (tile % tiles_x) * MTW, ty0 = (tile / tiles_x) * MTH;

  if (tid == 0) {
    // first of all: the camera table when the batch element changes (own barrier, needed first) and the reference
    // tile, whose 16 KB complete on the window barrier, armed together with the first window (the transaction count
    // may run negative until then).  Every reader of these regions passed the barrier that ended the previous item.
    if (b != cur_b) {
      mbar_arrive_expect_tx(bar_cam, (uint32_t)V * 64u);
      bulk_load(sbase + MOFF_CAM, p.cams + (size_t)b * V, (uint32_t)V * 64u, bar_cam);
    }
    tma_load_5d(sbase + MOFF_A, &tm_ref, bar_tma, 0, tx0, ty0, 0, b);
    *next_item = (int)gridDim.x + (int)atomicAdd(&g_mma_next[slot], 1u);   // read after the barrier that ends the item
  }
  // lanes beyond the last hypothesis of the chunk replicate it (same sample position: inside every window, no
  // predicates); their accumulator rows are never stored
  if (tid < MCH) ks[tid] = MODE != MAGNET_DEPTH_VOLUME ? p.k[min(jc + tid, D - 1)] : 0.0f;
  for (int idx = tid; idx < MCH * 65; idx += MNT) acc_s[idx] = 0.0f;
  __syncthreads();

  // ---- per-warp constants: lane i (mod 8) holds the ray / Gaussian of pixel i of my tile row ----------------
  const int py = ty0 + warp;
  float R0, R1, R2, MU = 0.f, SG = 0.f;
  unsigned livemask;
  {
    const int px = tx0 + (lane & 7);
    const bool live = px < W && py < H;
    const int n = min(py, H - 1) * W + min(px, W - 1);     // dead pixels shadow the nearest pixel, never store
    R0 = ldg_f(p.rays + ((size_t)b * 3 + 0) * HW + n);
    R1 = ldg_f(p.rays + ((size_t)b * 3 + 1) * HW + n);
    R2 = ldg_f(p.rays + ((size_t)b * 3 + 2) * HW + n);
    if (MODE == MAGNET_DEPTH_GAUSS) {
      MU = ldg_f(p.ref_gmm + ((size_t)b * 2 + 0) * HW + n);
      SG = ldg_f(p.ref_gmm + ((size_t)b * 2 + 1) * HW + n);
    }
    livemask = __ballot_sync(FULL, live) & 0xffu;
  }
  // my two hypotheses of every pixel of the row: (hypothesis jc + lane, hypothesis jc + 32 + lane).  Read from the
  // depth volume they stay in registers; sampled (MAGNET.py:155: multiply, then add) or plane depths are recomputed
  // from the pixel's Gaussian where needed (a few instructions instead of 16 registers).
  float2 dvol[MODE == MAGNET_DEPTH_VOLUME ? MTW : 1];
  float2 k2 = make_float2(0.f, 0.f);
  if (MODE == MAGNET_DEPTH_VOLUME) {                       // coalesced read, transposed through shared memory
    for (int idx = tid; idx < MCH * MPX; idx += MNT) {
      const int j = idx >> 6, pp = idx & 63;
      const int y = ty0 + (pp >> 3), x = tx0 + (pp & 7);
      const size_t n = (size_t)min(y, H - 1) * W + min(x, W - 1);
      regR[j * 65 + pp] = ldg_f(p.d_volume + ((size_t)b * D + jc + min(j, Dc - 1)) * HW + n);
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < MTW; ++i) dvol[i] = make_float2(regR[lane * 65 + warp * 8 + i], regR[(lane + 32) * 65 + warp * 8 + i]);
    fence_proxy_async();
    __syncthreads();
  } else {
    k2 = make_float2(ks[lane], ks[lane + 32]);
  }
  // (mu, sigma) come from the warp's pixel table; the product is rounded by __fmul_rn so that it is never contracted
  // into an FMA with the add (the reference rounds twice)
  auto depth2 = [&](const int i, const float mu, const float sg) -> float2 {
    if (MODE == MAGNET_DEPTH_VOLUME) return dvol[i];
    if (MODE == MAGNET_DEPTH_PLANES) return k2;
    return fadd2_rn(make_float2(mu, mu), make_float2(__fmul_rn(sg, k2.x), __fmul_rn(sg, k2.y)));
  };
  float4* pixt = reinterpret_cast<float4*>(smem + MOFF_PIX) + warp * 16;

  if (b != cur_b) {                                        // CTA-uniform: camera table landed
    mbar_wait_or_trap(bar_cam, ph_cam);
    ph_cam ^= 1u;
    cur_b = b;
  }
  bool first = true;                                       // the first window also waits for the reference tile

  for (int v = 0; v < V; ++v) {
    const magnet_camera* cam = cams_s + v;                 // V <= MMAXV is checked on the host
    if (cam->valid != 1.0f) continue;                      // CTA-uniform
    const float a0 = cam->a[0], a1 = cam->a[1], a2 = cam->a[2];
    // (K R) ray of the pixel this lane holds (lane & 7); the pixel loop below broadcasts it
    const float Q0 = __fmaf_rn(cam->A[2], R2, __fmaf_rn(cam->A[1], R1, __fmul_rn(cam->A[0], R0)));
    const float Q1 = __fmaf_rn(cam->A[5], R2, __fmaf_rn(cam->A[4], R1, __fmul_rn(cam->A[3], R0)));
    const float Q2 = __fmaf_rn(cam->A[8], R2, __fmaf_rn(cam->A[7], R1, __fmul_rn(cam->A[6], R0)));
    __syncwarp();                                          // the previous view's readers are done
    if (lane < 8) {
      pixt[2 * lane] = make_float4(Q0, Q1, Q2, 0.0f);
      pixt[2 * lane + 1] = make_float4(Q2, MU, SG, 0.0f);
    }
    __syncwarp();
    const int vb = v * p.B + b;
    // sample position of my two hypotheses of pixel i of the row, clamped: anything left of -1 / right of W (above /
    // below likewise) has all four taps out of the image, so cells stay near the image and NaN (fmaxf drops it) maps to
    // "out of bounds"; z = depth in the source camera
    auto project_px = [&](const int i, float2& ix, float2& iy, float2& z) {
      const float4 t1 = pixt[2 * i], t2 = pixt[2 * i + 1];   // same address on every lane: broadcast
      project2(depth2(i, t2.y, t2.z), a0, a1, a2, t1.x, t1.y, t1.z, ix, iy, z);
      ix.x = clamp_coord(ix.x, xmax); ix.y = clamp_coord(ix.y, xmax);
      iy.x = clamp_coord(iy.x, ymax); iy.y = clamp_coord(iy.y, ymax);
    };

    // ---------------- projection of every hypothesis, bounding box of the tile's sample positions -------------
    // (phase C projects again from the pixel table: holding the 32 positions across the MMA would not fit the registers)
    float xl = 1e9f, xh = -1e9f, yl = 1e9f, yh = -1e9f;
#pragma unroll
    for (int i = 0; i < MTW; ++i) {
      float2 ix, iy, z;
      project_px(i, ix, iy, z);
      if ((livemask >> i) & 1u) {                          // warp-uniform
        xl = fminf(xl, fminf(ix.x, ix.y)); xh = fmaxf(xh, fmaxf(ix.x, ix.y));
        yl = fminf(yl, fminf(iy.x, iy.y)); yh = fmaxf(yh, fmaxf(iy.x, iy.y));
      }
    }
    int* bb = bbox + (it & 1) * 4;
    {
      const int r0 = __reduce_min_sync(FULL, (int)floorf(xl)), r1 = __reduce_max_sync(FULL, (int)floorf(xh));
      const int r2 = __reduce_min_sync(FULL, (int)floorf(yl)), r3 = __reduce_max_sync(FULL, (int)floorf(yh));
      if (lane == 0) { atomicMin(bb + 0, r0); atomicMax(bb + 1, r1); atomicMin(bb + 2, r2); atomicMax(bb + 3, r3); }
    }
    fence_proxy_async();
    __syncthreads();                                       // box complete; region R is free (phase C of the last pass)
    const int wx0 = bb[0], wx1 = bb[1], wy0 = bb[2], wy1 = bb[3];
    if (tid < 4) bbox[((it + 1) & 1) * 4 + tid] = (tid & 1) ? -(1 << 28) : (1 << 28);   // re-arm the other slot
    ++it;
    // The cell origins span [wx0, wx1] x [wy0, wy1].  One pass when the window (origins + right / lower taps, cut into
    // 8-cell segments) fits MSEG segments, else sub-windows of <= MSEG segments that overlap by one cell column / row;
    // a hypothesis is evaluated in the sub-window that holds its cell origin.
    const int nseg_all = (wx1 - wx0 + 2 + 7) >> 3, rows_all = wy1 - wy0 + 2;
    const int nsw = min(nseg_all, 16);
    const int rmax = nseg_all * rows_all <= MSEG ? rows_all : max(2, MSEG / nsw);
    const int stepx = 8 * nsw - 1, stepy = rmax - 1;

    for (int sy = wy0; sy <= wy1; sy += stepy) {
      const int rows = min(stepy, wy1 - sy + 1) + 1;
      for (int sx = wx0; sx <= wx1; sx += stepx) {
        const int nseg = (min(stepx, wx1 - sx + 1) + 1 + 7) >> 3;
        const int nsegs = nseg * rows;                     // <= MSEG
        // ---------------- window + (mu, sigma) table by TMA ---------------------------------------------------
        if (tid == 0)
          mbar_arrive_expect_tx(bar_tma, (uint32_t)nsegs * (SEG_BYTES + (CW ? META_SEG_BYTES : 0)) + (first ? 16384u : 0u));
        first = false;
        if (lane == 0) {
          for (int s = warp; s < nsegs; s += MNT / 32) {
            const int r = s / nseg, xb = s - r * nseg;
            tma_load_5d(sbase + MOFF_R + (uint32_t)s * SEG_BYTES, &tm_src, bar_tma, 0, sx + 8 * xb, sy + r, 0, vb);
            if (CW) tma_load_4d(m_base + (uint32_t)s * META_SEG_BYTES, &tm_meta, bar_tma, 0, sx + 8 * xb + 1, sy + r, vb);   // entry x + 1 <-> cell x
          }
        }
        __syncwarp();
        const int npad = (nsegs * 8 + 15) & ~15;           // accumulator columns (N % 16 == 0)
        const int gp = ((npad + 23) & ~31) + 8;            // row pitch of G in floats: >= npad, % 32 == 8
        mbar_wait_or_trap(bar_tma, ph_tma);                // every thread observes the copies (it reads the table)
        ph_tma ^= 1u;
        // ---------------- G = ref x window^T: warpgroup g computes columns [128 g, 128 g + 128) -----------------
        // (3 products x 4 K steps of m64n128k16; the whole fence .. wait sequence sits inside the warpgroup-uniform
        // branch, so ptxas keeps the wgmma pipelined)
        {
          const int wg = warp >> 2;
          float acc[64];
#pragma unroll
          for (int e = 0; e < 64; ++e) acc[e] = 0.0f;
          const uint32_t bseg = sbase + MOFF_R + (uint32_t)(wg * 16 * SEG_BYTES);
          const uint64_t a_hi = gmma_desc_sw128(sbase + MOFF_A, 1024), a_lo = gmma_desc_sw128(sbase + MOFF_A + 8192, 1024);
          const uint64_t b_hi = gmma_desc_sw128(bseg, SEG_BYTES), b_lo = gmma_desc_sw128(bseg + 1024, SEG_BYTES);
          __syncwarp();                                      // wgmma is warp-synchronous (.aligned)
          if (wg == 0 || npad > 128) {                       // CTA-uniform: warpgroup 1 idles on a narrow window
            wgmma_fence();
#pragma unroll
            for (int pr = 0; pr < 3; ++pr) {                // small cross terms first
              const uint64_t ad = pr == 0 ? a_lo : a_hi, bd = pr == 1 ? b_lo : b_hi;
#pragma unroll
              for (int kk = 0; kk < 4; ++kk) wgmma_m64n128k16_f16(acc, ad + 2u * kk, bd + 2u * kk, (pr | kk) != 0);
            }
            wgmma_commit();
            wgmma_wait_all();
          }
          __syncthreads();                                   // both warpgroups have read the window: G may overwrite it
          // accumulator fragment -> G rows (pixels) x columns (cells); gp % 32 == 8 keeps the 8-byte stores conflict-free
          const int r0 = ((warp & 3) << 4) + (lane >> 2);
          float* g0 = regR + (size_t)r0 * gp + wg * 128 + 2 * (lane & 3);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            if (wg * 128 + 8 * j < npad) {                   // warp-uniform
              *reinterpret_cast<float2*>(g0 + 8 * j) = make_float2(acc[4 * j], acc[4 * j + 1]);
              *reinterpret_cast<float2*>(g0 + 8 * gp + 8 * j) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
            }
          }
          __syncthreads();
        }
#ifdef MAGNET_MMA_DEBUG
        if (dbg != nullptr && item == 0 && v == 0 && sy == wy0 && sx == wx0) {
          if (tid == 0) {
            dbg[0] = (float)sx; dbg[1] = (float)sy; dbg[2] = (float)nseg; dbg[3] = (float)rows; dbg[4] = (float)npad;
            dbg[5] = (float)gp; dbg[6] = (float)v; dbg[7] = 3.0f; dbg[8] = hdr_ref->scale; dbg[9] = hdr_src->scale;
          }
          for (int idx = tid; idx < MPX * npad; idx += MNT) dbg[16 + (idx / npad) * 256 + idx % npad] = regR[(idx / npad) * gp + idx % npad];
        }
#endif
        // ---------------- per hypothesis: 4 G reads, 4 table reads, 3 bilinear interpolations -------------------
        // byte offset of cell (x0, y0) in a G row = 4 * ((y0 - sy) * pitch + (x0 - sx)), evaluated in fp32 (small
        // integers, exact) on top of 1.5 * 2^23 so that the integer sits in the mantissa
        const bool single = nseg_all * rows_all <= MSEG;    // every cell origin lies in this (only) window
        auto phase_c = [&](auto single_tag) {
          constexpr bool SINGLE = decltype(single_tag)::value;
          const float MAGIC = 12582912.0f;
          const float sxf = (float)sx, syf = (float)sy;
          const float xend = sx + stepx > wx1 ? 1e9f : (float)(sx + stepx), yend = sy + stepy > wy1 ? 1e9f : (float)(sy + stepy);
          const float pitch4f = (float)(nseg * 32);
          const float c0f = MAGIC - 4.0f * sxf - pitch4f * syf;   // exact: integers below 2^24
          const uint32_t pitch4 = (uint32_t)nseg * 32u;
          uint32_t rowaddr = g_row0 + (uint32_t)(warp * 8 * gp) * 4u;
          float* accp = acc_s + lane * 65 + warp * 8;
#pragma unroll
          for (int i = 0; i < MTW; ++i, rowaddr += (uint32_t)gp * 4u) {
            if (!((livemask >> i) & 1u)) continue;         // warp-uniform
            float2 x, y, z;
            project_px(i, x, y, z);
            float2 x0, y0, fx, fy;                         // cell origins and fractions (cw_mask.cuh)
            cell_split(x.x, x0.x, fx.x); cell_split(x.y, x0.y, fx.y);
            cell_split(y.x, y0.x, fy.x); cell_split(y.y, y0.y, fy.y);
            const float2 m1 = make_float2(-1.0f, -1.0f);
            // byte offset of the cell in a G row = 4 * ((y0 - sy) * pitch + (x0 - sx)), in fp32 (small integers, exact)
            // on top of 1.5 * 2^23 so that the integer sits in the mantissa
            const float2 o = ffma2_rn(y0, make_float2(pitch4f, pitch4f), ffma2_rn(x0, make_float2(4.0f, 4.0f), make_float2(c0f, c0f)));
            uint32_t ca = __float_as_uint(o.x) & 0x3fffffu, cb = __float_as_uint(o.y) & 0x3fffffu;
            bool pa = true, pb = true;
            if (!SINGLE) {                                 // evaluated in the sub-window that holds the cell origin
              pa = x0.x >= sxf && x0.x < xend && y0.x >= syf && y0.x < yend;
              pb = x0.y >= sxf && x0.y < xend && y0.y >= syf && y0.y < yend;
              ca = pa ? ca : 0u;                           // the others read cell 0
              cb = pb ? cb : 0u;
            }
            const uint32_t ga = rowaddr + ca, gb = rowaddr + cb;
            const float2 g00 = make_float2(lds_f32(ga), lds_f32(gb)), g01 = make_float2(lds_f32(ga + 4), lds_f32(gb + 4));
            const float2 g10 = make_float2(lds_f32(ga + pitch4), lds_f32(gb + pitch4));
            const float2 g11 = make_float2(lds_f32(ga + pitch4 + 4), lds_f32(gb + pitch4 + 4));
            const float2 ct = ffma2_rn(fx, ffma2_rn(g00, m1, g01), g00), cu = ffma2_rn(fx, ffma2_rn(g10, m1, g11), g10);
            const float2 cost = ffma2_rn(fy, ffma2_rn(ct, m1, cu), ct);            // both hypotheses at once
            const float costa = cost.x, costb = cost.y;
            bool oka, okb;
            if (CW) {
              const uint32_t ma = m_base + ca * 4u, mb = m_base + cb * 4u;
              // table entry of a cell = (mu, sigma) of the cell and of its right neighbour: two 16-byte reads per hypothesis
              const float2 msa = lerp2d_x2(lds_f32x4(ma), lds_f32x4(ma + pitch4 * 4u), fx.x, fy.x);
              const float2 msb = lerp2d_x2(lds_f32x4(mb), lds_f32x4(mb + pitch4 * 4u), fx.y, fy.y);
              oka = cw_keep(z.x, msa, kappa);               // homography.py:157-158 (cw_mask.cuh)
              okb = cw_keep(z.y, msb, kappa);
            } else {
              oka = fabsf(costa) < 3.0e38f;
              okb = fabsf(costb) < 3.0e38f;
            }
            // the accumulator of (hypothesis, pixel) is touched by this lane only
            if (pa && oka) accp[i] += costa;
            if (pb && okb) accp[32 * 65 + i] += costb;
          }
        };
        if (single) phase_c(std::true_type{});
        else phase_c(std::false_type{});
        fence_proxy_async();
        __syncthreads();                                   // G / table dead: the next copies and MMAs may overwrite
      }
    }
  }

  if (first) {                                             // no valid view: the reference-tile copy is still in flight
    if (tid == 0) mbar_arrive_expect_tx(bar_tma, 16384u);
    mbar_wait_or_trap(bar_tma, ph_tma);
    ph_tma ^= 1u;
  }

  // -------- epilogue: undo the split scales, 1/V mean over ALL views (homography.py:120), coalesced store --------
  {
    const float inv = hdr_ref->inv_scale * hdr_src->inv_scale;   // powers of two: exact
    const bool exact = p.inv_v_exact != 0.0f;              // V a power of two: the division is an exact scaling
    auto fin = [&](float a) { a *= inv; return exact ? a * p.inv_v_exact : __fdiv_rn(a, p.vf); };
    if ((W & 3) == 0 && (reinterpret_cast<uintptr_t>(p.out) & 15) == 0) {
      for (int idx = tid; idx < MCH * 16; idx += MNT) {    // (hypothesis, tile row, half row): one 16-byte store
        const int j = idx >> 4, r = (idx >> 1) & 7, hx = (idx & 1) * 4;
        const int y = ty0 + r, x = tx0 + hx;
        if (j < Dc && x < W && y < H) {
          const float* a = acc_s + j * 65 + r * 8 + hx;
          *reinterpret_cast<float4*>(p.out + ((size_t)b * D + jc + j) * HW + (size_t)y * W + x) =
              make_float4(fin(a[0]), fin(a[1]), fin(a[2]), fin(a[3]));
        }
      }
    } else {
      for (int idx = tid; idx < MCH * MPX; idx += MNT) {
        const int j = idx >> 6, pp = idx & 63;
        const int y = ty0 + (pp >> 3), x = tx0 + (pp & 7);
        if (j < Dc && x < W && y < H) p.out[((size_t)b * D + jc + j) * HW + (size_t)y * W + x] = fin(acc_s[j * 65 + pp]);
      }
    }
  }
  const int nxt = *next_item;                              // written by thread 0 when this item began
  __syncthreads();                                         // accumulators and tables are free; next_item may be rewritten
  item = nxt;
  }  // work items

  if (tid == 0) {                                          // the last CTA to finish re-arms the work counter
    __threadfence();
    if (atomicAdd(&g_mma_done[slot], 1u) == gridDim.x - 1) {
      g_mma_next[slot] = 0u;
      g_mma_done[slot] = 0u;
      __threadfence();
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// MAGNET_SRC_SPLIT16 producer: (N, 64, H, W) fp32 [+ (N, 2, H, W) Gaussians] ->
//   header | fp16 planes (N, 2, H, W, 64): hi = fp16(x*s), lo = fp16(x*s - hi) | table (N, H, W + 1, 4), entry x + 1 =
//   (mu[x], sigma[x], mu[x+1], sigma[x+1]), zeros outside the row
// ---------------------------------------------------------------------------------------------------------------
// bits of |x|, 0 for inf / NaN: the scale is chosen from the finite values, non-finite elements poison only their own
// products
__device__ __forceinline__ unsigned finite_abs_bits(float x) {
  const unsigned u = __float_as_uint(x) & 0x7fffffffu;
  return u >= 0x7f800000u ? 0u : u;
}

__global__ void __launch_bounds__(256) absmax_kernel(const float4* __restrict__ x, size_t n4, const float* __restrict__ tail,
                                                     int ntail, unsigned* __restrict__ out) {
  unsigned m = 0u;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    const float4 v = __ldg(x + i);
    m = max(max(m, finite_abs_bits(v.x)), finite_abs_bits(v.y));
    m = max(max(m, finite_abs_bits(v.z)), finite_abs_bits(v.w));
  }
  if (blockIdx.x == 0 && (int)threadIdx.x < ntail) m = max(m, finite_abs_bits(tail[threadIdx.x]));
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0 && m != 0u) atomicMax(out, m);
}

// power-of-two scale that maps absmax into [2^14, 2^15); 1 for an all-zero or non-finite tensor
__device__ __forceinline__ int split16_shift(unsigned absmax_bits) {
  const int e = (int)(absmax_bits >> 23) & 0xff;
  if (e == 0 || e == 255) return 0;
  return max(-100, min(100, 14 - (e - 127)));
}

// One CTA per SPX pixels of one image: channel planes are read coalesced along the pixels (16-byte loads when the image
// size allows, all of a thread's loads in flight together), transposed through shared memory, and the two fp16 planes
// are written as contiguous 128-byte pixel rows.
template <int SPX, bool VEC>
__global__ void __launch_bounds__(256) split16_repack_kernel(const float* __restrict__ src, const float* __restrict__ gmm,
                                                             unsigned char* __restrict__ dst, int N, int HW, int W) {
  constexpr int C = 64;
  __shared__ float t[SPX * (C + 1)];
  Split16Header* hdr = reinterpret_cast<Split16Header*>(dst);
  const int sh = split16_shift(hdr->absmax);
  const float s = __uint_as_float((unsigned)(127 + sh) << 23);
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
    hdr->scale = s;
    hdr->inv_scale = __uint_as_float((unsigned)(127 - sh) << 23);
  }
  const size_t img = blockIdx.y;
  const int p0 = blockIdx.x * SPX;
  if constexpr (VEC) {                                     // HW % 4 == 0, src 16-byte aligned
    static_assert(SPX == 128, "thread mapping below");
    constexpr int CPI = 8;                                 // channels per iteration
    // a warp reads 4 channel rows x 8 float4 (4 x 128 contiguous bytes); this way its transposed stores hit 32 banks
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int q4 = (warp & 3) * 8 + (lane & 7), c0 = (warp >> 2) * 4 + (lane >> 3);
    float4 v[C / CPI];
#pragma unroll
    for (int e = 0; e < C / CPI; ++e) {
      const int c = c0 + e * CPI, pix = p0 + 4 * q4;
      v[e] = pix < HW ? __ldg(reinterpret_cast<const float4*>(src + (img * C + c) * HW + pix)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int e = 0; e < C / CPI; ++e) {
      const int c = c0 + e * CPI;
      t[(4 * q4 + 0) * (C + 1) + c] = v[e].x;
      t[(4 * q4 + 1) * (C + 1) + c] = v[e].y;
      t[(4 * q4 + 2) * (C + 1) + c] = v[e].z;
      t[(4 * q4 + 3) * (C + 1) + c] = v[e].w;
    }
  } else {
    const int xi = threadIdx.x % SPX, cy = threadIdx.x / SPX;
    for (int c = cy; c < C; c += 256 / SPX) t[xi * (C + 1) + c] = p0 + xi < HW ? src[(img * C + c) * HW + p0 + xi] : 0.0f;
  }
  __syncthreads();
  __half* planes = reinterpret_cast<__half*>(dst + SPLIT16_HEADER);
  float4* meta = reinterpret_cast<float4*>(dst + SPLIT16_HEADER + (size_t)N * HW * 256);
#pragma unroll
  for (int itw = 0; itw < SPX * 8 / 256; ++itw) {
    const int item = itw * 256 + threadIdx.x;
    const int pl = item >> 3, q = item & 7;                // pixel of the group, 8-channel chunk
    if (p0 + pl < HW) {
      __align__(16) __half hi[8], lo[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float v = t[pl * (C + 1) + q * 8 + e] * s;
        hi[e] = __float2half_rn(v);
        lo[e] = __float2half_rn(v - __half2float(hi[e]));
      }
      const size_t o = (size_t)(p0 + pl) * 64 + q * 8;
      *reinterpret_cast<uint4*>(planes + (img * 2 + 0) * (size_t)HW * 64 + o) = *reinterpret_cast<const uint4*>(hi);
      *reinterpret_cast<uint4*>(planes + (img * 2 + 1) * (size_t)HW * 64 + o) = *reinterpret_cast<const uint4*>(lo);
    }
  }
  if (threadIdx.x < SPX && p0 + threadIdx.x < HW) {       // my (mu, sigma): first half of entry x + 1, second half of entry x
    const int pix = p0 + threadIdx.x;
    const int y = pix / W, x = pix - y * W;
    float2 ms = make_float2(0.0f, 0.0f);
    if (gmm != nullptr) ms = make_float2(gmm[(img * 2 + 0) * HW + pix], gmm[(img * 2 + 1) * HW + pix]);
    float2* row = reinterpret_cast<float2*>(meta + (img * (HW / W) + y) * (size_t)(W + 1));
    row[2 * (x + 1)] = ms;
    row[2 * x + 1] = ms;
    if (x == 0) row[0] = make_float2(0.0f, 0.0f);          // entry 0 = (outside, pixel 0)
    if (x == W - 1) row[2 * W + 1] = make_float2(0.0f, 0.0f);   // entry W = (pixel W-1, outside)
  }
}

int sm_count(int dev) {
  static int cached[64] = {0};
  int& c = cached[dev & 63];
  if (c == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    c = n;
  }
  return c;
}

cudaError_t launch_repack_split16(const float* src, const float* gmm, void* dst, int N, int C, int H, int W,
                                  cudaStream_t st, int* launches) {
  if (C != 64) return cudaErrorInvalidValue;
  const int HW = H * W;
  const size_t n = (size_t)N * C * HW;
  cudaError_t e = cudaMemsetAsync(dst, 0, SPLIT16_HEADER, st);
  if (e != cudaSuccess) return e;
  const size_t n4 = n / 4;
  int dev = 0;
  if ((e = cudaGetDevice(&dev)) != cudaSuccess) return e;
  const int blocks = (int)std::min<size_t>((size_t)sm_count(dev) * 8, (n4 + 255) / 256 + 1);
  absmax_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<const float4*>(src), n4, src + n4 * 4, (int)(n - n4 * 4),
                                        reinterpret_cast<unsigned*>(static_cast<unsigned char*>(dst) + offsetof(Split16Header, absmax)));
  dim3 block(256);
  if (HW % 4 == 0 && reinterpret_cast<uintptr_t>(src) % 16 == 0) {
    dim3 grid((HW + 127) / 128, N);
    split16_repack_kernel<128, true><<<grid, block, 0, st>>>(src, gmm, static_cast<unsigned char*>(dst), N, HW, W);
  } else {
    dim3 grid((HW + 31) / 32, N);
    split16_repack_kernel<32, false><<<grid, block, 0, st>>>(src, gmm, static_cast<unsigned char*>(dst), N, HW, W);
  }
  *launches = 2;
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled_fn();   // cost_tma.cu

// rank-5 map over the fp16 planes: (64 channels, W, H, 2 planes, N); box = 8 pixels of one row (window segment) or an
// 8x8 tile (reference), both planes; 128-byte swizzle = the canonical K-major wgmma layout (cost_f_bwd_mma.cu reads
// the same boxes as MN-major operands)
cudaError_t make_planes_map(CUtensorMap* tm, const void* planes, int N, int H, int W, int box_rows) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) return cudaErrorNotSupported;
  const cuuint64_t dims[5] = {64, (cuuint64_t)W, (cuuint64_t)H, 2, (cuuint64_t)N};
  const cuuint64_t strides[4] = {128, (cuuint64_t)W * 128, (cuuint64_t)H * W * 128, (cuuint64_t)H * W * 256};
  const cuuint32_t box[5] = {64u, 8u, (cuuint32_t)box_rows, 2u, 1u};
  const cuuint32_t estr[5] = {1u, 1u, 1u, 1u, 1u};
  const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(planes), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

// rank-4 map over the paired (mu, sigma) table: (4 floats, W + 1, H, N), box = 8 entries of one row
static cudaError_t make_meta_map(CUtensorMap* tm, const void* meta, int N, int H, int W) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) return cudaErrorNotSupported;
  const cuuint64_t dims[4] = {4, (cuuint64_t)W + 1, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t strides[3] = {16, ((cuuint64_t)W + 1) * 16, (cuuint64_t)H * (W + 1) * 16};
  const cuuint32_t box[4] = {4u, 8u, 1u, 1u};
  const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<void*>(meta), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

#ifdef MAGNET_MMA_DEBUG
static float* g_mma_dbg = nullptr;
void mma_set_debug_buffer(float* p) { g_mma_dbg = p; }
#endif

template <int MODE, bool CW>
static cudaError_t launch_mma_mw(const CostParams& p, cudaStream_t st) {
  static std::once_flag flags[64];
  auto kern = cost_mma_kernel<MODE, CW>;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  cudaError_t res = cudaSuccess;
  std::call_once(flags[dev & 63], [&] {
    res = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, M_SMEM_TOTAL);
    if (res == cudaSuccess)
      res = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  });
  if (res != cudaSuccess) return res;
  const int N = p.B * p.V;
  const unsigned char* refbuf = reinterpret_cast<const unsigned char*>(p.ref_feat);
  const unsigned char* srcbuf = reinterpret_cast<const unsigned char*>(p.src_feat);
  CUtensorMap tm_ref, tm_src, tm_meta;
  if ((e = make_planes_map(&tm_ref, refbuf + SPLIT16_HEADER, p.B, p.H, p.W, 8)) != cudaSuccess) return e;
  if ((e = make_planes_map(&tm_src, srcbuf + SPLIT16_HEADER, N, p.H, p.W, 1)) != cudaSuccess) return e;
  if ((e = make_meta_map(&tm_meta, srcbuf + SPLIT16_HEADER + (size_t)N * p.HW * 256, N, p.H, p.W)) != cudaSuccess) return e;
  const int nchunks = (p.D + MCH - 1) / MCH;
  const int tiles = ((p.W + MTW - 1) / MTW) * ((p.H + MTH - 1) / MTH);
  const int n_items = tiles * nchunks * p.B;
  // work-counter slot of this launch: eager launches cycle through the lower half, launches recorded into a CUDA graph
  // take theirs from the upper half (a replay reuses its slot for the life of the graph, so it must never meet an eager
  // launch on another stream)
  static std::atomic<unsigned> ticket{0}, graph_ticket{0};
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &cap) != cudaSuccess) cap = cudaStreamCaptureStatusNone;
  const int slot = cap == cudaStreamCaptureStatusActive ? MMA_SLOTS / 2 + (int)(graph_ticket.fetch_add(1) % (MMA_SLOTS / 2))
                                                        : (int)(ticket.fetch_add(1) % (MMA_SLOTS / 2));
  dim3 grid(std::min(n_items, 2 * sm_count(dev))), block(MNT);   // persistent: two CTAs per SM
  float* dbg = nullptr;
#ifdef MAGNET_MMA_DEBUG
  dbg = g_mma_dbg;
#endif
  kern<<<grid, block, M_SMEM_TOTAL, st>>>(p, tm_ref, tm_src, tm_meta, nchunks, n_items, slot, dbg);
  return cudaGetLastError();
}

bool mma_supports(int C, int D, int V, int layout) {
  return C == 64 && layout == MAGNET_SRC_SPLIT16 && D >= 1 && V <= MMAXV;
}

void mma_launch_info(int B, int H, int W, int D, int* grid, int* block, int* smem) {
  int dev = 0;
  cudaGetDevice(&dev);
  *grid = std::min(((W + MTW - 1) / MTW) * ((H + MTH - 1) / MTH) * ((D + MCH - 1) / MCH) * B, 2 * sm_count(dev));
  *block = MNT;
  *smem = M_SMEM_TOTAL;
}

size_t split16_buffer_bytes(int N, int H, int W) { return split16_bytes((size_t)N, (size_t)H, (size_t)W); }

cudaError_t launch_cost_mma(const CostParams& p, int mode, bool cw, cudaStream_t st) {
  if (cw) {
    if (mode == MAGNET_DEPTH_VOLUME) return launch_mma_mw<MAGNET_DEPTH_VOLUME, true>(p, st);
    if (mode == MAGNET_DEPTH_GAUSS) return launch_mma_mw<MAGNET_DEPTH_GAUSS, true>(p, st);
    return launch_mma_mw<MAGNET_DEPTH_PLANES, true>(p, st);
  }
  if (mode == MAGNET_DEPTH_VOLUME) return launch_mma_mw<MAGNET_DEPTH_VOLUME, false>(p, st);
  if (mode == MAGNET_DEPTH_GAUSS) return launch_mma_mw<MAGNET_DEPTH_GAUSS, false>(p, st);
  return launch_mma_mw<MAGNET_DEPTH_PLANES, false>(p, st);
}

}  // namespace magnet
