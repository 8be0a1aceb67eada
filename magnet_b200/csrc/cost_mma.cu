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
//     magnet_repack_split16_f32).  An fp16 / bf16 map needs no lo plane: x*s is itself an fp16 number (MAGNET_SRC_HALF16,
//     magnet_repack_half16, DESIGN §3.7), so PLANES = 1 loads one plane per box and issues the hi*hi product only (4
//     wgmma per warpgroup); shared-memory map, descriptors (the lo atom slot is left unwritten) and everything after
//     the MMA are those of PLANES = 2.
//   * the planes are (image, plane, y, x, 64 channels) fp16 = 128-byte rows: an 8-pixel x 2-plane TMA box with
//     CU_TENSOR_MAP_SWIZZLE_128B lands as one canonical K-major wgmma atom per plane; the window of a (tile, view) is the
//     bounding box of the tile's sample positions cut into such 8-cell segments (zero fill outside the image =
//     grid_sample's padding_mode='zeros'), cell index = B-operand row = accumulator column.  The reference tile is the
//     A operand (M = 64); warpgroup g computes accumulator columns [128 g, 128 g + 128).
//   * one warp per tile row (8 pixels in turn), one LANE per hypothesis (lane j: hypotheses j and j + 32 of the
//     64-hypothesis chunk, evaluated side by side as float2 pairs): the pixel's constants are warp-uniform (per-warp table
//     in shared memory), the 32 lanes read a handful of neighbouring cells of ONE accumulator row (broadcast /
//     conflict-free); lanes beyond the last hypothesis replicate it, so there are no activity predicates.
//   * per view: TMA window + paired (mu, sigma) table, and while the copies land the NEXT view's window box
//     (projections of each pixel's smallest and largest depth, window_box) -> 12 wgmma per warpgroup (3 products x 4 K
//     steps; m64n128k16, or m64n64k16 for warpgroup 1 when the window ends below column 192) -> the 64 accumulator rows
//     into shared memory (over the window, which is dead by then) -> per-hypothesis phase, which projects from the
//     per-warp pixel table.  The box is complete at the barrier that ends the phase, so the next view's copies are issued
//     right after it.  The 16 view accumulators of a lane stay in registers; the epilogue transposes them through
//     region R into the hypothesis-major layout of the coalesced stores.
//   * a window that does not fit 256 cells is cut into sub-windows of <= 32 segments that overlap by one cell column /
//     row; a hypothesis is evaluated in the sub-window that holds its cell origin.  Same code for any depth distribution.
//   * persistent CTAs (two per SM): work items (batch element, tile, 64-hypothesis chunk) come from a global counter in a
//     per-launch slot that the last CTA re-arms (graph-replay safe); barriers are set up once per CTA.
//
// Numerics: the per-view channel sum is the tensor core's fp32 accumulation of exact products of the split factors
// (relative error ~2^-21 of sum |ref||src|, the same order as an fp32 FMA chain); everything else — projection, weights,
// consistency test, view accumulation, 1/V — is the fp32 arithmetic of the other kernels (common.cuh project2).
#include <algorithm>
#include <cstddef>
#include <mutex>

#include "common.cuh"
#include "cw_mask.cuh"
#include "launchers.h"
#include "packed_layout.cuh"
#include "tma_common.cuh"

namespace magnet {

constexpr int MNT = 256;               // threads per CTA: warp w owns tile row w, pixel i of the row in turn
constexpr int MTW = 8, MTH = 8;        // CTA tile in reference pixels
constexpr int MPX = MTW * MTH;         // 64 = rows of the accumulator that are used
constexpr int MCH = 64;                // hypotheses per CTA (two per lane)
constexpr int MSEG = 32;               // 8-cell segments per window: N <= 256 accumulator columns
constexpr int MBATCH = 4;              // pixels of a tile row evaluated together in phase C (see there)
constexpr int MMAXV = 16;              // views whose camera constants are staged in shared memory
constexpr int SEG_BYTES = 2048;        // hi atom (8 cells x 128 B) + lo atom
constexpr int META_SEG_BYTES = 128;    // 8 cells x (mu, sigma of the cell and of its right neighbour)
constexpr uint32_t SEG_TX = 1024;      // bytes per plane of a window segment's box (PLANES planes land, 1 or 2)
constexpr uint32_t REF_TX = 8192;      // bytes per plane of the reference tile's box

// shared-memory map (bytes from the 1024-aligned base)
constexpr int MOFF_A = 0;                                   // reference tile: hi 8 KB | lo 8 KB
constexpr int MOFF_R = 16384;                               // window segments, later the accumulator rows G[64][GP]
constexpr int MR_BYTES = 67584;                             //   >= 32 * 2048 and >= 64 * 264 * 4
constexpr int MOFF_META = MOFF_R + MR_BYTES;                // float4[256] (mu, sigma)[c], (mu, sigma)[c + 1] per window cell
constexpr int MOFF_CAM = MOFF_META + MSEG * META_SEG_BYTES; // magnet_camera[MMAXV]
constexpr int MOFF_KS = MOFF_CAM + MMAXV * 64;              // float[MCH]
constexpr int MOFF_BBOX = MOFF_KS + MCH * 4;                // int[2 slots][4]
constexpr int MOFF_BAR = MOFF_BBOX + 64;                    // 2 mbarriers, next work item
constexpr int MOFF_DV = MOFF_BAR + 64;                      // float[MPX][65]: depths of the item, pixel-major (VOLUME)
constexpr int MOFF_DEND = MOFF_DV + MPX * 65 * 4;           // float2[MPX]: depth range of each pixel (VOLUME)
constexpr int MOFF_PIXR = MOFF_DEND + MPX * 8;              // float4[MPX][2]: (ray, -) (mu, sigma, -, -) of each pixel
constexpr int MOFF_PIX = MOFF_PIXR + MPX * 32;              // float4[8 warps][8 pixels][2]: (q0,q1,q2,a0) (a1,mu,sigma,a2)
constexpr int M_SMEM_USED = MOFF_PIX + 8 * 8 * 32;
constexpr int M_SMEM_TOTAL = M_SMEM_USED + 1024;            // slack for the 1024-byte alignment of the base
static_assert(MR_BYTES >= MSEG * SEG_BYTES && MR_BYTES >= MPX * 264 * 4 && MR_BYTES >= MCH * 65 * 4, "region R");
// MAGNET_MMA_DEBUG builds: the debug buffer holds a G dump (16 + 64 * 256 floats), then two uint32 counters: hypotheses
// whose cell origin fell outside their window box (must stay 0) and tile rows whose box took the exact per-hypothesis pass
constexpr int MMA_DBG_OUTSIDE = 16 + MPX * 256;
static_assert(2 * (M_SMEM_TOTAL + 1024) <= 227 * 1024, "two CTAs per SM");

// work counters of the persistent kernel (work slots, common.cuh)
__device__ unsigned g_mma_next[WORK_SLOTS];
__device__ unsigned g_mma_done[WORK_SLOTS];

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
// MAGNET_MMA_PROFILE builds: thread 0 reads clock64() at the CTA barriers that separate the stages of a work item and
// adds each interval to its stage; at exit the CTA's totals go to the debug buffer (uint64[8], scripts/mma_profile.py)
enum { PROF_SETUP, PROF_BOX, PROF_TMA, PROF_MMA, PROF_PHASEC, PROF_EPI, PROF_NSTAGES };
#ifdef MAGNET_MMA_PROFILE
#define MMA_STAGE(s)                                                                                                   \
  do {                                                                                                                 \
    if (tid == 0) {                                                                                                    \
      const long long t_ = clock64();                                                                                  \
      prof_s[s] += t_ - prof_s[7];                                                                                     \
      prof_s[7] = t_;                                                                                                  \
    }                                                                                                                  \
  } while (0)
#else
#define MMA_STAGE(s) do { } while (0)
#endif

// PLANES = 2: MAGNET_SRC_SPLIT16 (hi / lo), 1: MAGNET_SRC_HALF16 (one plane, the hi*hi product only)
template <int MODE, bool CW, int PLANES, bool IDX>
__global__ void __launch_bounds__(MNT, 2)
cost_mma_kernel(const __grid_constant__ CostParams p, const __grid_constant__ CUtensorMap tm_ref,
                const __grid_constant__ CUtensorMap tm_src, const __grid_constant__ CUtensorMap tm_meta, const int nchunks,
                const int n_items, const int slot, float* __restrict__ dbg, const int32_t* __restrict__ src_index) {
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
  const unsigned FULL = 0xffffffffu;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#ifdef MAGNET_MMA_PROFILE
  __shared__ long long prof_s[8];
  if (tid < 8) prof_s[tid] = tid == 7 ? clock64() : 0ll;
#endif
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
  // window boxes from the depth-range endpoints: margin and the largest error amplification it covers (DESIGN.md §3.1)
  constexpr float BOX_EPS = 0.015625f;
  const float amp_max = 65536.0f / (float)(max(W, H) + 3) - 8.0f;
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
    *next_item = (int)gridDim.x + (int)slot_claim(g_mma_next, slot);   // read after the barrier that ends the item
  }
  // lanes beyond the last hypothesis of the chunk replicate it (same sample position: inside every window, no
  // predicates); their accumulators are never stored
  if (tid < MCH) ks[tid] = MODE != MAGNET_DEPTH_VOLUME ? p.k[min(jc + tid, D - 1)] : 0.0f;
  __syncthreads();

  // ---- per-warp constants: lane i (mod 8) holds the ray / Gaussian of pixel i of my tile row ----------------
  // (kept in shared memory, pixr: registers are short next to the accumulators of the MMA)
  const int py = ty0 + warp;
  float4* pixr = reinterpret_cast<float4*>(smem + MOFF_PIXR) + warp * 16;
  unsigned livemask;
  {
    float R0, R1, R2, MU = 0.f, SG = 0.f;
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
    if (lane < 8) {
      pixr[2 * lane] = make_float4(R0, R1, R2, 0.0f);
      pixr[2 * lane + 1] = make_float4(MU, SG, 0.0f, 0.0f);
    }
    __syncwarp();
  }
  // my two hypotheses of every pixel of the row: (hypothesis jc + lane, hypothesis jc + 32 + lane).  Read from the
  // depth volume they stay in shared memory (pixel-major, conflict-free per pixel); sampled (MAGNET.py:155: multiply,
  // then add) or plane depths are recomputed from the pixel's Gaussian where needed.
  // (by 32-bit shared address: registers are short next to the accumulators of the MMA)
  const uint32_t dvw = sbase + MOFF_DV + (uint32_t)(warp * 8 * 65 + lane) * 4u;
  if (MODE == MAGNET_DEPTH_VOLUME) {
    float* dv_s = reinterpret_cast<float*>(smem + MOFF_DV);                       // coalesced read, transposed through shared memory
    // thread: pixel tid % 64, hypotheses tid / 64 + 4 r (loads in flight together, then the conflict-free stores)
    const int pp = tid & 63, y = ty0 + (pp >> 3), x = tx0 + (pp & 7);
    const float* dsrc = p.d_volume + ((size_t)b * D + jc) * HW + (size_t)min(y, H - 1) * W + min(x, W - 1);
#pragma unroll 1
    for (int j0 = tid >> 6; j0 < MCH; j0 += 32) {         // two batches of 8 loads (registers)
      float dl[8];
#pragma unroll
      for (int r = 0; r < 8; ++r) dl[r] = ldg_f(dsrc + (size_t)min(j0 + 4 * r, Dc - 1) * HW);
#pragma unroll
      for (int r = 0; r < 8; ++r) dv_s[pp * 65 + j0 + 4 * r] = dl[r];
    }
    __syncthreads();
    // depth range of every pixel of my row over the chunk (NaN when a depth is not finite): the window boxes
#pragma unroll
    for (int i = 0; i < MTW; ++i) {
      const float da = lds_f32(dvw + i * 260), db = lds_f32(dvw + i * 260 + 128);
      float lo = fminf(da, db), hi = fmaxf(da, db);
      const bool fin = __all_sync(FULL, isfinite(da) && isfinite(db));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        lo = fminf(lo, __shfl_xor_sync(FULL, lo, o));
        hi = fmaxf(hi, __shfl_xor_sync(FULL, hi, o));
      }
      if (lane == i) reinterpret_cast<float2*>(smem + MOFF_DEND)[warp * 8 + i] = fin ? make_float2(lo, hi) : make_float2(NAN, NAN);
    }
    __syncwarp();
  }
  // (mu, sigma) come from the warp's pixel table; the product is rounded by __fmul_rn so that it is never contracted
  // into an FMA with the add (the reference rounds twice)
  auto depth2 = [&](const int i, const float mu, const float sg) -> float2 {
    if (MODE == MAGNET_DEPTH_VOLUME) return make_float2(lds_f32(dvw + i * 260), lds_f32(dvw + i * 260 + 128));
    const float2 k2 = make_float2(ks[lane], ks[lane + 32]);
    if (MODE == MAGNET_DEPTH_PLANES) return k2;
    return fadd2_rn(make_float2(mu, mu), make_float2(__fmul_rn(sg, k2.x), __fmul_rn(sg, k2.y)));
  };
  float4* pixt = reinterpret_cast<float4*>(smem + MOFF_PIX) + warp * 16;

  // ---- window box of view v: the bounding box of the cell origins of the tile's hypotheses, added into the bbox
  // slot bb by shared atomics (complete after the next CTA barrier).  The sample position is a Moebius map of the depth,
  // monotone on a depth interval where z keeps its sign, so the positions of a pixel's depths lie between those of its
  // smallest and largest depth: 2 projections per pixel instead of 64, widened by BOX_EPS for the rounding of the
  // evaluation (DESIGN.md §3.1).  A row with a pixel outside the conditions of that bound (non-finite depth range,
  // unsorted k, z <= 0 or a large error amplification at an endpoint) projects every hypothesis instead, exactly as
  // phase C does.
  auto window_box = [&](const int v, int* bb) {
    const magnet_camera* cam = cams_s + v;
    const float a0 = cam->a[0], a1 = cam->a[1], a2 = cam->a[2];
    const float4 ray = pixr[2 * (lane & 7)];
    const float MU = pixr[2 * (lane & 7) + 1].x, SG = pixr[2 * (lane & 7) + 1].y;
    const float Q0 = __fmaf_rn(cam->A[2], ray.z, __fmaf_rn(cam->A[1], ray.y, __fmul_rn(cam->A[0], ray.x)));
    const float Q1 = __fmaf_rn(cam->A[5], ray.z, __fmaf_rn(cam->A[4], ray.y, __fmul_rn(cam->A[3], ray.x)));
    const float Q2 = __fmaf_rn(cam->A[8], ray.z, __fmaf_rn(cam->A[7], ray.y, __fmul_rn(cam->A[6], ray.x)));
    float2 dr;                                             // depth range of my pixel (lane & 7) over the chunk
    if (MODE == MAGNET_DEPTH_VOLUME) {
      const uint32_t a = sbase + MOFF_DEND + (uint32_t)(warp * 8 + (lane & 7)) * 8u;
      dr = make_float2(lds_f32(a), lds_f32(a + 4));
    }
    else if (MODE == MAGNET_DEPTH_PLANES) dr = make_float2(ks[0], ks[MCH - 1]);
    else dr = fadd2_rn(make_float2(MU, MU), make_float2(__fmul_rn(SG, ks[0]), __fmul_rn(SG, ks[MCH - 1])));
    float2 ix, iy, z;
    project2(dr, a0, a1, a2, Q0, Q1, Q2, ix, iy, z);
    const float amp = fmaxf(fabsf(__fmul_rn(Q2, dr.x)) / z.x, fabsf(__fmul_rn(Q2, dr.y)) / z.y) + 2.0e-3f / fminf(z.x, z.y);
    const bool ok = (MODE == MAGNET_DEPTH_VOLUME || p.k_sorted) && isfinite(dr.x) && isfinite(dr.y) && z.x > 0.0f &&
                    z.y > 0.0f && amp <= amp_max && isfinite(ix.x) && isfinite(ix.y) && isfinite(iy.x) && isfinite(iy.y);
    const bool live = (livemask >> (lane & 7)) & 1u;
    float xl = 1e9f, xh = -1e9f, yl = 1e9f, yh = -1e9f;
    if (__all_sync(FULL, ok || !live)) {                   // warp-uniform
      if (live) {
        xl = clamp_coord(__fsub_rn(fminf(ix.x, ix.y), BOX_EPS), xmax); xh = clamp_coord(__fadd_rn(fmaxf(ix.x, ix.y), BOX_EPS), xmax);
        yl = clamp_coord(__fsub_rn(fminf(iy.x, iy.y), BOX_EPS), ymax); yh = clamp_coord(__fadd_rn(fmaxf(iy.x, iy.y), BOX_EPS), ymax);
      }
    } else {
#ifdef MAGNET_MMA_DEBUG
      if (dbg != nullptr && lane == 0) atomicAdd(reinterpret_cast<unsigned*>(dbg + MMA_DBG_OUTSIDE + 1), 1u);   // exact rows
#endif
#pragma unroll
      for (int i = 0; i < MTW; ++i) {
        const float q0 = __shfl_sync(FULL, Q0, i), q1 = __shfl_sync(FULL, Q1, i), q2 = __shfl_sync(FULL, Q2, i);
        const float mu = __shfl_sync(FULL, MU, i), sg = __shfl_sync(FULL, SG, i);
        project2(depth2(i, mu, sg), a0, a1, a2, q0, q1, q2, ix, iy, z);
        ix.x = clamp_coord(ix.x, xmax); ix.y = clamp_coord(ix.y, xmax);
        iy.x = clamp_coord(iy.x, ymax); iy.y = clamp_coord(iy.y, ymax);
        if ((livemask >> i) & 1u) {                        // warp-uniform
          xl = fminf(xl, fminf(ix.x, ix.y)); xh = fmaxf(xh, fmaxf(ix.x, ix.y));
          yl = fminf(yl, fminf(iy.x, iy.y)); yh = fmaxf(yh, fmaxf(iy.x, iy.y));
        }
      }
    }
    const int r0 = __reduce_min_sync(FULL, (int)floorf(xl)), r1 = __reduce_max_sync(FULL, (int)floorf(xh));
    const int r2 = __reduce_min_sync(FULL, (int)floorf(yl)), r3 = __reduce_max_sync(FULL, (int)floorf(yh));
    if (lane == 0) { atomicMin(bb + 0, r0); atomicMax(bb + 1, r1); atomicMin(bb + 2, r2); atomicMax(bb + 3, r3); }
  };
  auto next_valid = [&](int v) {                           // CTA-uniform
    while (v < V && cams_s[v].valid != 1.0f) ++v;          // V <= MMAXV is checked on the host
    return v;
  };

  if (b != cur_b) {                                        // CTA-uniform: camera table landed
    mbar_wait_or_trap(bar_cam, ph_cam);
    ph_cam ^= 1u;
    cur_b = b;
  }
  bool first = true;                                       // the first window also waits for the reference tile
  float2 accr[MTW];                                        // view accumulators of (hypotheses lane, lane + 32) x pixel
#pragma unroll
  for (int i = 0; i < MTW; ++i) accr[i] = make_float2(0.0f, 0.0f);
  MMA_STAGE(PROF_SETUP);
  int v = next_valid(0);
  if (v < V) window_box(v, bbox + (it & 1) * 4);
  __syncthreads();                                         // box of the first view complete
  MMA_STAGE(PROF_BOX);

  while (v < V) {
    const int vn = next_valid(v + 1);
    __syncwarp();                                          // the previous view's readers are done
    if (lane < 8) {                                        // (K R) ray of pixel `lane` of the row and the view's a
      const magnet_camera* cam = cams_s + v;
      const float4 ray = pixr[2 * lane], ms = pixr[2 * lane + 1];
      const float Q0 = __fmaf_rn(cam->A[2], ray.z, __fmaf_rn(cam->A[1], ray.y, __fmul_rn(cam->A[0], ray.x)));
      const float Q1 = __fmaf_rn(cam->A[5], ray.z, __fmaf_rn(cam->A[4], ray.y, __fmul_rn(cam->A[3], ray.x)));
      const float Q2 = __fmaf_rn(cam->A[8], ray.z, __fmaf_rn(cam->A[7], ray.y, __fmul_rn(cam->A[6], ray.x)));
      pixt[2 * lane] = make_float4(Q0, Q1, Q2, cam->a[0]);
      pixt[2 * lane + 1] = make_float4(cam->a[1], ms.x, ms.y, cam->a[2]);
    }
    __syncwarp();
    const int vb = src_image<IDX>(src_index, b, v, p.B, V);

    // the box of this view was completed by the barrier that ended the previous pass (or the item set-up)
    const int* bb = bbox + (it & 1) * 4;
    const int wx0 = bb[0], wx1 = bb[1], wy0 = bb[2], wy1 = bb[3];
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
          mbar_arrive_expect_tx(bar_tma, (uint32_t)nsegs * (SEG_TX * PLANES + (CW ? META_SEG_BYTES : 0)) + (first ? REF_TX * PLANES : 0u));
        first = false;
        if (lane == 0) {
          for (int s = warp; s < nsegs; s += MNT / 32) {
            const int r = s / nseg, xb = s - r * nseg;
            tma_load_5d(sbase + MOFF_R + (uint32_t)s * SEG_BYTES, &tm_src, bar_tma, 0, sx + 8 * xb, sy + r, 0, vb);
            if (CW) tma_load_4d(m_base + (uint32_t)s * META_SEG_BYTES, &tm_meta, bar_tma, 0, sx + 8 * xb + 1, sy + r, vb);   // entry x + 1 <-> cell x
          }
        }
        __syncwarp();
        // the next view's box while the copies land: it reads only the camera and pixel tables, and it is complete at
        // the barrier that ends this view's last phase C, right before the next view's copies are issued
        const bool first_pass = sy == wy0 && sx == wx0;    // CTA-uniform
        if (first_pass && vn < V) window_box(vn, bbox + (it & 1) * 4);
        const int npad = (nsegs * 8 + 15) & ~15;           // accumulator columns (N % 16 == 0)
        const int gp = ((npad + 23) & ~31) + 8;            // row pitch of G in floats: >= npad, % 32 == 8
        mbar_wait_or_trap(bar_tma, ph_tma);                // every thread observes the copies (it reads the table)
        ph_tma ^= 1u;
        MMA_STAGE(PROF_TMA);
        // ---------------- G = ref x window^T: warpgroup g computes columns [128 g, 128 g + 128) -----------------
        // (3 products x 4 K steps; warpgroup 0 issues m64n128k16, warpgroup 1 the narrowest of n128 / n64 / nothing
        // that covers npad - 128.  Each shape's whole fence .. wait sequence sits inside its own warpgroup-uniform
        // branch, so ptxas keeps the wgmma pipelined.)
        {
          const int wg = warp >> 2;
          float acc[64];
#pragma unroll
          for (int e = 0; e < 64; ++e) acc[e] = 0.0f;
          const uint32_t bseg = sbase + MOFF_R + (uint32_t)(wg * 16 * SEG_BYTES);
          const uint64_t a_hi = gmma_desc_sw128(sbase + MOFF_A, 1024), a_lo = gmma_desc_sw128(sbase + MOFF_A + 8192, 1024);
          const uint64_t b_hi = gmma_desc_sw128(bseg, SEG_BYTES), b_lo = gmma_desc_sw128(bseg + 1024, SEG_BYTES);
          __syncwarp();                                      // wgmma is warp-synchronous (.aligned)
          // ptxas (CUDA 12.9) serialises the wgmma of <GAUSS, false> when it holds the second shape (C7511, out of
          // registers), so that instantiation keeps n128 for warpgroup 1; so does <VOLUME, false, 1> (HALF16), where the
          // same happens with the second shape (DESIGN §3.7)
          constexpr bool WG1_N64 = (CW || MODE != MAGNET_DEPTH_GAUSS) && (PLANES == 2 || CW || MODE != MAGNET_DEPTH_VOLUME);
          // (PLANES = 1: the hi*hi product alone, scale-d 0 on its first K step)
          if (wg == 0 || npad > (WG1_N64 ? 192 : 128)) {     // warpgroup-uniform: N = 128
            wgmma_fence();
#pragma unroll
            for (int pr = PLANES == 2 ? 0 : 2; pr < 3; ++pr) {   // small cross terms first
              const uint64_t ad = pr == 0 ? a_lo : a_hi, bd = pr == 1 ? b_lo : b_hi;
#pragma unroll
              for (int kk = 0; kk < 4; ++kk) wgmma_m64n128k16_f16(acc, ad + 2u * kk, bd + 2u * kk, ((PLANES == 2 ? pr : 0) | kk) != 0);
            }
            wgmma_commit();
            wgmma_wait_all();
          } else if (WG1_N64 && npad > 128) {                // warpgroup 1, columns [128, 192): N = 64
            float (&acc64)[32] = *reinterpret_cast<float (*)[32]>(acc);
            wgmma_fence();
#pragma unroll
            for (int pr = PLANES == 2 ? 0 : 2; pr < 3; ++pr) {
              const uint64_t ad = pr == 0 ? a_lo : a_hi, bd = pr == 1 ? b_lo : b_hi;
#pragma unroll
              for (int kk = 0; kk < 4; ++kk) wgmma_m64n64k16_f16(acc64, ad + 2u * kk, bd + 2u * kk, ((PLANES == 2 ? pr : 0) | kk) != 0);
            }
            wgmma_commit();
            wgmma_wait_all();
          }                                                  // (else warpgroup 1 idles on a narrow window)
          __syncthreads();                                   // both warpgroups have read the window: G may overwrite it;
                                                             // every thread has read this view's box
          // re-arm the box slot this view was read from: the view after next adds its box into it
          if (tid == 0 && first_pass) *reinterpret_cast<int4*>(bbox + ((it + 1) & 1) * 4) = make_int4(1 << 28, -(1 << 28), 1 << 28, -(1 << 28));
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
        MMA_STAGE(PROF_MMA);
#ifdef MAGNET_MMA_DEBUG
        if (dbg != nullptr && item == 0 && v == 0 && sy == wy0 && sx == wx0) {
          if (tid == 0) {
            dbg[0] = (float)sx; dbg[1] = (float)sy; dbg[2] = (float)nseg; dbg[3] = (float)rows; dbg[4] = (float)npad;
            dbg[5] = (float)gp; dbg[6] = (float)v; dbg[7] = 2.0f * PLANES - 1.0f; dbg[8] = hdr_ref->scale; dbg[9] = hdr_src->scale;
          }
          for (int idx = tid; idx < MPX * npad; idx += MNT) dbg[16 + (idx / npad) * 256 + idx % npad] = regR[(idx / npad) * gp + idx % npad];
        }
#endif
        // ---------------- per hypothesis: 4 G reads, 4 table reads, 3 bilinear interpolations -------------------
        // The pixels of the row go in batches of MBATCH, stage by stage: the batch's pixel constants and depths, then
        // its projections and cell offsets, then all its G and table reads, then the interpolations and adds, so the
        // chains of the batch's pixels overlap.  Inside a batch there is no branch: a dead pixel reads cells inside
        // the window like any other (the min / select below) and liveness only predicates its adds.  A warp-uniform
        // branch skips a batch
        // without a live pixel; it also bounds the block ptxas schedules as one.  With the whole row in one block,
        // ptxas (CUDA 12.9) needs more than 128 registers and serialises the wgmma of <GAUSS, true> (C7511); with
        // blocks of 4 pixels no instantiation has more spills or C7511 / C7520 warnings than with one pixel per
        // block.  Each hypothesis sees the same operations in the same order as with one pixel at a time, so the
        // accumulators are the same bit for bit.
        const bool single = nseg_all * rows_all <= MSEG;    // every cell origin lies in this (only) window
        auto phase_c = [&](auto single_tag) {
          constexpr bool SINGLE = decltype(single_tag)::value;
          const float MAGIC = 12582912.0f;
          const float sxf = (float)sx, syf = (float)sy;
          const float xend = sx + stepx > wx1 ? 1e9f : (float)(sx + stepx), yend = sy + stepy > wy1 ? 1e9f : (float)(sy + stepy);
          const float pitch4f = (float)(nseg * 32);
          const float c0f = MAGIC - 4.0f * sxf - pitch4f * syf;   // exact: integers below 2^24
          const uint32_t pitch4 = (uint32_t)nseg * 32u;
          uint32_t rowaddr = g_row0 + (uint32_t)(warp * 8 * gp) * 4u;   // G row of pixel i0 (one running address)
          const uint32_t cmax = pitch4 * (uint32_t)(rows - 1) - 8u;   // last cell origin of the window (bytes)
          const float2 m1 = make_float2(-1.0f, -1.0f);
#pragma unroll
          for (int i0 = 0; i0 < MTW; i0 += MBATCH, rowaddr += (uint32_t)(MBATCH * gp) * 4u) {
            if (!((livemask >> i0) & ((1u << MBATCH) - 1u))) continue;   // warp-uniform
            float4 t1[MBATCH], t2[MBATCH];                 // pixel table: same address on every lane, broadcast
            float2 d[MBATCH];
#pragma unroll
            for (int u = 0; u < MBATCH; ++u) {
              t1[u] = pixt[2 * (i0 + u)];
              t2[u] = pixt[2 * (i0 + u) + 1];
            }
#pragma unroll
            for (int u = 0; u < MBATCH; ++u) d[u] = depth2(i0 + u, t2[u].y, t2[u].z);
            float2 z[MBATCH], fx[MBATCH], fy[MBATCH];
            uint32_t ca[MBATCH], cb[MBATCH];
            bool pa[MBATCH], pb[MBATCH];
#pragma unroll
            for (int u = 0; u < MBATCH; ++u) {
              // sample position of my two hypotheses, clamped: anything left of -1 / right of W (above / below
              // likewise) has all four taps out of the image, so cells stay near the image and NaN (fmaxf drops it)
              // maps to "out of bounds"; z = depth in the source camera
              float2 x, y;
              project2(d[u], t1[u].w, t2[u].x, t2[u].w, t1[u].x, t1[u].y, t1[u].z, x, y, z[u]);
              x.x = clamp_coord(x.x, xmax); x.y = clamp_coord(x.y, xmax);
              y.x = clamp_coord(y.x, ymax); y.y = clamp_coord(y.y, ymax);
              float2 x0, y0;                               // cell origins and fractions (cw_mask.cuh)
              cell_split(x.x, x0.x, fx[u].x); cell_split(x.y, x0.y, fx[u].y);
              cell_split(y.x, y0.x, fy[u].x); cell_split(y.y, y0.y, fy[u].y);
              // byte offset of the cell in a G row = 4 * ((y0 - sy) * pitch + (x0 - sx)), in fp32 (small integers,
              // exact) on top of 1.5 * 2^23 so that the integer sits in the mantissa
              const float2 o = ffma2_rn(y0, make_float2(pitch4f, pitch4f), ffma2_rn(x0, make_float2(4.0f, 4.0f), make_float2(c0f, c0f)));
              ca[u] = __float_as_uint(o.x) & 0x3fffffu;
              cb[u] = __float_as_uint(o.y) & 0x3fffffu;
              const bool live = (livemask >> (i0 + u)) & 1u;
              pa[u] = live;
              pb[u] = live;
              if (!SINGLE) {                               // evaluated in the sub-window that holds the cell origin
                pa[u] = live && x0.x >= sxf && x0.x < xend && y0.x >= syf && y0.x < yend;
                pb[u] = live && x0.y >= sxf && x0.y < xend && y0.y >= syf && y0.y < yend;
                ca[u] = pa[u] ? ca[u] : 0u;                // the others (dead pixels too) read cell 0
                cb[u] = pb[u] ? cb[u] : 0u;
              } else {                                     // a wrong box can never address outside the window
                ca[u] = min(ca[u], cmax);
                cb[u] = min(cb[u], cmax);
              }
#ifdef MAGNET_MMA_DEBUG
              if (dbg != nullptr && sy == wy0 && sx == wx0) {   // hypotheses whose cell origin fell outside the box
                const bool outa = live && lane < Dc && (x0.x < (float)wx0 || x0.x > (float)wx1 || y0.x < (float)wy0 || y0.x > (float)wy1);
                const bool outb = live && lane + 32 < Dc && (x0.y < (float)wx0 || x0.y > (float)wx1 || y0.y < (float)wy0 || y0.y > (float)wy1);
                const unsigned nout = __popc(__ballot_sync(FULL, outa)) + __popc(__ballot_sync(FULL, outb));
                if (lane == 0 && nout != 0u) atomicAdd(reinterpret_cast<unsigned*>(dbg + MMA_DBG_OUTSIDE), nout);
              }
#endif
            }
            float2 g00[MBATCH], g01[MBATCH], g10[MBATCH], g11[MBATCH];
            float4 mta[MBATCH], mba[MBATCH], mtb[MBATCH], mbb[MBATCH];   // (CW) table: top / bottom row x hypothesis a / b
            uint32_t ra = rowaddr;
#pragma unroll
            for (int u = 0; u < MBATCH; ++u, ra += (uint32_t)gp * 4u) {
              const uint32_t ga = ra + ca[u], gb = ra + cb[u];
              g00[u] = make_float2(lds_f32(ga), lds_f32(gb));
              g01[u] = make_float2(lds_f32(ga + 4), lds_f32(gb + 4));
              g10[u] = make_float2(lds_f32(ga + pitch4), lds_f32(gb + pitch4));
              g11[u] = make_float2(lds_f32(ga + pitch4 + 4), lds_f32(gb + pitch4 + 4));
              if (CW) {
                // table entry of a cell = (mu, sigma) of the cell and of its right neighbour: two 16-byte reads per
                // hypothesis
                const uint32_t ma = m_base + ca[u] * 4u, mb = m_base + cb[u] * 4u;
                mta[u] = lds_f32x4(ma);
                mba[u] = lds_f32x4(ma + pitch4 * 4u);
                mtb[u] = lds_f32x4(mb);
                mbb[u] = lds_f32x4(mb + pitch4 * 4u);
              }
            }
#pragma unroll
            for (int u = 0; u < MBATCH; ++u) {
              const float2 ct = ffma2_rn(fx[u], ffma2_rn(g00[u], m1, g01[u]), g00[u]);
              const float2 cu = ffma2_rn(fx[u], ffma2_rn(g10[u], m1, g11[u]), g10[u]);
              const float2 cost = ffma2_rn(fy[u], ffma2_rn(ct, m1, cu), ct);        // both hypotheses at once
              const float costa = cost.x, costb = cost.y;
              bool oka, okb;
              if (CW) {
                const float2 msa = lerp2d_x2(mta[u], mba[u], fx[u].x, fy[u].x);
                const float2 msb = lerp2d_x2(mtb[u], mbb[u], fx[u].y, fy[u].y);
                oka = cw_keep(z[u].x, msa, kappa);          // homography.py:157-158 (cw_mask.cuh)
                okb = cw_keep(z[u].y, msb, kappa);
              } else {
                oka = fabsf(costa) < 3.0e38f;
                okb = fabsf(costb) < 3.0e38f;
              }
              if (pa[u] && oka) accr[i0 + u].x += costa;
              if (pb[u] && okb) accr[i0 + u].y += costb;
            }
          }
        };
        if (single) phase_c(std::true_type{});
        else phase_c(std::false_type{});
        fence_proxy_async();
        __syncthreads();                                   // G / table dead: the next copies and MMAs may overwrite
        MMA_STAGE(PROF_PHASEC);
      }
    }
    v = vn;
  }

  if (first) {                                             // no valid view: the reference-tile copy is still in flight
    if (tid == 0) mbar_arrive_expect_tx(bar_tma, REF_TX * PLANES);
    mbar_wait_or_trap(bar_tma, ph_tma);
    ph_tma ^= 1u;
  }

  // -------- epilogue: undo the split scales, 1/V mean over ALL views (homography.py:120), coalesced store --------
  {
    // the accumulators go through region R (free: the last pass ended with a CTA barrier), hypothesis-major
    float* acc_s = regR;
    // the item's coordinates, decoded again: not kept in registers across the views
    const int b = item / items_per_b;
    const int rem = item - b * items_per_b;
    const int tile = rem / nchunks;
    const int jc = (rem - tile * nchunks) * MCH;
    const int Dc = min(MCH, D - jc);
    const int tx0 = (tile % tiles_x) * MTW, ty0 = (tile / tiles_x) * MTH;
#pragma unroll
    for (int i = 0; i < MTW; ++i) {
      acc_s[lane * 65 + warp * 8 + i] = accr[i].x;
      acc_s[(lane + 32) * 65 + warp * 8 + i] = accr[i].y;
    }
    __syncthreads();
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
  fence_proxy_async();                                     // region R is overwritten by the next item's copies
  __syncthreads();                                         // accumulators and tables are free; next_item may be rewritten
  MMA_STAGE(PROF_EPI);
  item = nxt;
  }  // work items

#ifdef MAGNET_MMA_PROFILE
  if (tid == 0 && dbg != nullptr) {
    unsigned long long* tot = reinterpret_cast<unsigned long long*>(dbg);
    for (int s = 0; s < PROF_NSTAGES; ++s) atomicAdd(tot + s, (unsigned long long)prof_s[s]);
    atomicAdd(tot + 7, 1ull);                              // CTAs
  }
#endif
  if (tid == 0) slot_finish(g_mma_next, g_mma_done, slot);
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
#if defined(MAGNET_MMA_DEBUG) || defined(MAGNET_MMA_PROFILE)
static float* g_mma_dbg = nullptr;
void mma_set_debug_buffer(float* p) { g_mma_dbg = p; }
#endif

static SlotTickets mma_tickets;

template <int MODE, bool CW, int PLANES, bool IDX>
static cudaError_t launch_mma(const CostParams& p, const int32_t* src_index, int n_src, cudaStream_t st) {
  static std::once_flag flags[64];
  auto kern = cost_mma_kernel<MODE, CW, PLANES, IDX>;
  int dev = 0;
  cudaError_t e = set_smem_once(kern, flags, M_SMEM_TOTAL, true, &dev);
  if (e != cudaSuccess) return e;
  const int N = IDX ? n_src : p.B * p.V;               // source images in the buffer
  CUtensorMap tm_ref, tm_src, tm_meta;
  if ((e = make_planes_map(&tm_ref, p.ref_feat, p.B, p.H, p.W, 8, PLANES)) != cudaSuccess) return e;
  if ((e = make_planes_map(&tm_src, p.src_feat, N, p.H, p.W, 1, PLANES)) != cudaSuccess) return e;
  if ((e = make_meta_map(&tm_meta, p.src_feat, N, p.H, p.W, PLANES)) != cudaSuccess) return e;
  const int nchunks = (p.D + MCH - 1) / MCH;
  const int tiles = ((p.W + MTW - 1) / MTW) * ((p.H + MTH - 1) / MTH);
  const int n_items = tiles * nchunks * p.B;
  dim3 grid(std::min(n_items, 2 * sm_count(dev))), block(MNT);   // persistent: two CTAs per SM
  float* dbg = nullptr;
#if defined(MAGNET_MMA_DEBUG) || defined(MAGNET_MMA_PROFILE)
  dbg = g_mma_dbg;
#endif
  kern<<<grid, block, M_SMEM_TOTAL, st>>>(p, tm_ref, tm_src, tm_meta, nchunks, n_items, work_slot(mma_tickets, st), dbg,
                                          src_index);
  return cudaGetLastError();
}

bool mma_supports(int C, int D, int V, int layout) {
  return C == 64 && (layout == MAGNET_SRC_SPLIT16 || layout == MAGNET_SRC_HALF16) && D >= 1 && V <= MMAXV;
}

void mma_launch_info(int B, int H, int W, int D, int* grid, int* block, int* smem) {
  int dev = 0;
  cudaGetDevice(&dev);
  *grid = std::min(((W + MTW - 1) / MTW) * ((H + MTH - 1) / MTH) * ((D + MCH - 1) / MCH) * B, 2 * sm_count(dev));
  *block = MNT;
  *smem = M_SMEM_TOTAL;
}

// layout: MAGNET_SRC_SPLIT16 (hi / lo planes) or MAGNET_SRC_HALF16 (one plane); src_index: NULL (view-major source
// images, V*B of them) or the (B, V) frame table over n_src images
cudaError_t launch_cost_mma(const CostParams& p, int mode, bool cw, int layout, const int32_t* src_index, int n_src,
                            cudaStream_t st, int* launches) {
  *launches = 1;
  return dispatch([&](auto m, auto w, auto planes, auto idx) { return launch_mma<m, w, planes, idx>(p, src_index, n_src, st); },
                  DepthMode{mode}, Flag{cw}, Choice<int, 1, 2>{layout == MAGNET_SRC_HALF16 ? 1 : 2},
                  Flag{src_index != nullptr});
}

}  // namespace magnet
