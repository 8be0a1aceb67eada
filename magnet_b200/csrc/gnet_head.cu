// G-Net head of inference in one kernel (DESIGN §3.8): per 8x16 pixel tile, the 3x3 conv of the cost volume, the
// hoisted x_d3 part, three ReLU layers, the 128 -> 2 layer and the Gaussian update.  No 128-channel map leaves the SM.
//
// GEMMs run on the fp16 tensor cores (mma.sync m16n8k16, fp32 accumulation) in the SPLIT16 scheme: x*s = hi + lo with
// a power-of-two s, three products hi*hi + hi*lo + lo*hi, exact descale.  Scales: one per call for the cost volume
// (largest finite |cost|), one per layer for the weights (chosen by the pack), one per pixel row for the hidden
// activations (taken from the fp32 accumulator row after ReLU).
#include <cuda_fp16.h>

#include <algorithm>
#include <mutex>

#include "gaussian_common.cuh"
#include "head_common.cuh"

namespace magnet {

int sm_count(int dev);                                                                   // cost_mma.cu
cudaError_t launch_absmax_f32(const float* x, size_t n, unsigned* out, cudaStream_t st);  // cost_mma.cu

namespace {
constexpr int TY = 8, TX = 16;                 // pixel tile of a CTA: warp w owns row w (16 pixels = the MMA's M)
constexpr int HX = TX + 2, HP = (TY + 2) * HX; // the tile's 3x3 halo, 180 pixels
constexpr int NT = 32 * TY;
constexpr int CCH = 16;                        // cost channels staged per chunk (one K step)

// Packed weight buffer (magnet_gnet_pack_weights_f32).  B fragments are stored in the order the MMA consumes them:
// per (K step, n8 tile) 32 lanes x 16 bytes {hi(b0), hi(b1), lo(b0), lo(b1)}, so each lane loads its fragment with
// one 16-byte load.
constexpr size_t G_HDR = 0;                    // int32 shift of W0, W1, W2
constexpr size_t G_VEC = 256;                  // fp32 b1[128], b2[128], W3[2][128], b3[2]
constexpr int G_NVEC = 4 * HID + 2;
constexpr size_t G_W1 = 4096;
constexpr size_t G_LAYER = (size_t)(HID / 16) * NTILE * 32 * 16;   // 64 KiB per 128x128 layer
constexpr size_t G_W2 = G_W1 + G_LAYER;
constexpr size_t G_W0 = G_W2 + G_LAYER;
constexpr size_t G_W0_CHUNK = (size_t)9 * NTILE * 32 * 16;           // one 16-channel chunk of the 3x3 weights

constexpr size_t S_W12 = 2 * G_LAYER;
constexpr size_t S_HALO = (size_t)2 * HP * CCH * 2;                   // hi and lo planes, 32 bytes per pixel
constexpr size_t S_VEC = ((G_NVEC * 4 + 15) / 16) * 16;
constexpr size_t S_RAW = (size_t)CCH * HP * 4;                       // fp32 staging of the next chunk
constexpr size_t S_TOTAL = S_W12 + S_HALO + S_VEC + S_RAW;
static_assert(G_NVEC == 514, "b1, b2, W3, b3");
static_assert(G_VEC + G_NVEC * 4 <= G_W1, "vectors fit before W1");
}  // namespace

size_t gnet_weights_bytes(int D) { return G_W0 + (size_t)((D + CCH - 1) / CCH) * G_W0_CHUNK; }

namespace {
struct GnetParams {
  int B, D, H, W, ncs, tiles_x, tiles_y, ntiles;
  const float* __restrict__ cost;
  const float* __restrict__ inv;
  const unsigned char* __restrict__ weights;
  const float* __restrict__ prev;
  const unsigned* __restrict__ absmax;
  float* __restrict__ out;
  float* __restrict__ save;   // SAVE: h0, h1, h2 as (B,128,H,W) each, then raw (mu1, sigma1) as (B,2,H,W)
};

// SAVE (training forward, DESIGN §3.10): the same arithmetic, plus stores of the three ReLU'd hidden maps and the raw
// output for the backward.
template <bool SAVE>
__global__ void __launch_bounds__(NT, 1) gnet_head_kernel(const GnetParams p) {
  extern __shared__ __align__(16) unsigned char smem[];
  uint4* w12 = reinterpret_cast<uint4*>(smem);                          // W1 then W2, resident
  uint4* halo = reinterpret_cast<uint4*>(smem + S_W12);                 // [hi, lo][HP pixels][2 x 8 channels]
  float* vec = reinterpret_cast<float*>(smem + S_W12 + S_HALO);
  float* raw = reinterpret_cast<float*>(smem + S_W12 + S_HALO + S_VEC);  // [CCH channels][HP pixels] fp32
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, q = lane & 3;
  const int HW = p.H * p.W;
  {
    const uint4* src = reinterpret_cast<const uint4*>(p.weights + G_W1);
    for (int i = tid; i < (int)(S_W12 / 16); i += NT) w12[i] = __ldg(src + i);
    const float* vs = reinterpret_cast<const float*>(p.weights + G_VEC);
    for (int i = tid; i < G_NVEC; i += NT) vec[i] = __ldg(vs + i);
  }
  const int* shw = reinterpret_cast<const int*>(p.weights + G_HDR);
  const int sh_w0 = __ldg(shw + 0), sh_w1 = __ldg(shw + 1), sh_w2 = __ldg(shw + 2);
  const int sh_c = split16_shift(*p.absmax);
  const float sc = pow2(sh_c), dc = pow2(-sh_c), dw0 = pow2(-sh_w0);
  const uint4* w0 = reinterpret_cast<const uint4*>(p.weights + G_W0);
  const int per_img = p.tiles_x * p.tiles_y;

  // one 16-channel chunk of a tile's halo: thread t < HP owns halo pixel t and copies its 16 values (zeros outside the
  // image and past D) into the fp32 staging buffer by cp.async, one chunk ahead of the MMAs
  const uint32_t raw_s = (uint32_t)__cvta_generic_to_shared(raw);
  auto load_chunk = [&](int tile, int cs) {
    if (tid < HP) {
      const int b = tile / per_img, t = tile - b * per_img, ty = t / p.tiles_x;
      const int y = ty * TY - 1 + tid / HX, x = (t - ty * p.tiles_x) * TX - 1 + tid % HX;
      const bool in = y >= 0 && y < p.H && x >= 0 && x < p.W;
      const float* src = p.cost + ((size_t)b * p.D + (size_t)cs * CCH) * HW + (in ? y * p.W + x : 0);
#pragma unroll
      for (int j = 0; j < CCH; ++j) {
        const bool ok = in && cs * CCH + j < p.D;
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;"
                     :: "r"(raw_s + (uint32_t)(j * HP + tid) * 4), "l"(ok ? src + (size_t)j * HW : p.cost), "r"(ok ? 4 : 0)
                     : "memory");
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  // scaled, split, stored pixel-major; the two 16-byte halves of a pixel swap places every 4 pixels, so the 8 rows of
  // an ldmatrix phase (8 consecutive halo pixels) hit 8 distinct 16-byte bank groups
  auto store_chunk = [&]() {
    if (tid >= HP) return;
    uint32_t hi[8], lo[8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
      split2(__fmul_rn(raw[2 * j * HP + tid], sc), __fmul_rn(raw[(2 * j + 1) * HP + tid], sc), hi[j], lo[j]);
    const int sw = (tid >> 2) & 1;
    halo[tid * 2 + sw] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    halo[tid * 2 + (sw ^ 1)] = make_uint4(hi[4], hi[5], hi[6], hi[7]);
    halo[HP * 2 + tid * 2 + sw] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    halo[HP * 2 + tid * 2 + (sw ^ 1)] = make_uint4(lo[4], lo[5], lo[6], lo[7]);
  };

  const uint32_t halo_s = (uint32_t)__cvta_generic_to_shared(halo);
  const int a_row = (lane & 7) + ((lane >> 3) & 1) * 8, a_half = lane >> 4;   // ldmatrix.x4 row address of this lane
  int tile = blockIdx.x;
  if (tile < p.ntiles) load_chunk(tile, 0);
  for (; tile < p.ntiles; tile += gridDim.x) {
    const int b = tile / per_img, t = tile - b * per_img, ty = t / p.tiles_x;
    const int y = ty * TY + warp, x0 = (t - ty * p.tiles_x) * TX;
    float acc[NTILE][4];
#pragma unroll
    for (int nt = 0; nt < NTILE; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.0f;

    // ---- 3x3 conv of the cost volume: per chunk, nine shifted views of the halo against W0's tap slices ----
    for (int cs = 0; cs < p.ncs; ++cs) {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      __syncthreads();                                  // chunk landed; every warp is done with the previous halo
      store_chunk();
      __syncthreads();                                  // halo written; the staging buffer is free again
      if (cs + 1 < p.ncs) load_chunk(tile, cs + 1);
      else if (tile + (int)gridDim.x < p.ntiles) load_chunk(tile + gridDim.x, 0);
#pragma unroll 1
      for (int tap = 0; tap < 9; ++tap) {
        const int hp = (warp + tap / 3) * HX + a_row + tap % 3;
        const uint32_t off = (uint32_t)(hp * 32 + ((a_half ^ ((hp >> 2) & 1)) << 4));
        uint32_t ah[4], al[4];
        ldsm_x4(ah, halo_s + off);
        ldsm_x4(al, halo_s + HP * 32 + off);
        const uint4* wb = w0 + ((size_t)(cs * 9 + tap) * NTILE) * 32 + lane;
#pragma unroll
        for (int nt = 0; nt < NTILE; ++nt) mma3(acc[nt], ah, al, __ldg(wb + nt * 32));
      }
    }

    // ---- + invariant (x_d3 half and b0), ReLU ----
    const int xa = x0 + g, xb = x0 + g + 8;
    const bool va = y < p.H && xa < p.W, vb = y < p.H && xb < p.W;
    const float* ip = p.inv + (size_t)b * HID * HW + (size_t)(va || vb ? y : 0) * p.W;
#pragma unroll
    for (int nt = 0; nt < NTILE; ++nt) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const size_t n = (size_t)(nt * 8 + 2 * q + e) * HW;
        const float ca = __fmul_rn(__fmul_rn(acc[nt][e], dc), dw0), cb = __fmul_rn(__fmul_rn(acc[nt][2 + e], dc), dw0);
        acc[nt][e] = va ? relu(__fadd_rn(ca, __ldg(ip + n + xa))) : 0.0f;
        acc[nt][2 + e] = vb ? relu(__fadd_rn(cb, __ldg(ip + n + xb))) : 0.0f;
      }
    }

    // SAVE: layer l's activations of the warp's valid pixels into plane l of the saved maps
    auto save_hidden = [&](int l) {
      float* hp = p.save + ((size_t)l * p.B + b) * HID * HW + (size_t)(va ? y * p.W + xa : 0) + (size_t)(2 * q) * HW;
      store_rows(hp, acc, HW, va, vb);
      __syncwarp();   // keeps ptxas from sinking the stores into the next layer's MMAs (which spills)
    };
    if constexpr (SAVE) save_hidden(0);
    hidden_layer(acc, w12, vec, sh_w1, lane);
    if constexpr (SAVE) save_hidden(1);
    hidden_layer(acc, w12 + G_LAYER / 16, vec + HID, sh_w2, lane);
    if constexpr (SAVE) save_hidden(2);

    // ---- 128 -> 2 on the CUDA cores, quad reduction, Gaussian update ----
    float r[4];                                          // (mu1, sigma1) of rows g and g+8
    out2_layer(acc, vec + 2 * HID, q, r);
    if (q < 2 && (q == 0 ? va : vb)) {                  // lane 0 of the quad writes pixel g, lane 1 pixel g+8
      const size_t o = (size_t)b * 2 * HW + (size_t)y * p.W + (q == 0 ? xa : xb);
      const float mu1 = __fadd_rn(q == 0 ? r[0] : r[2], vec[4 * HID]);
      const float s1 = __fadd_rn(q == 0 ? r[1] : r[3], vec[4 * HID + 1]);
      float mu, sg;
      gaussian_update(mu1, s1, __ldg(p.prev + o), __ldg(p.prev + o + HW), mu, sg);
      p.out[o] = mu;
      p.out[o + HW] = sg;
      if constexpr (SAVE) {
        float* rp = p.save + (size_t)3 * p.B * HID * HW;
        rp[o] = mu1;
        rp[o + HW] = s1;
      }
    }
  }
}

// ---- weight pack --------------------------------------------------------------------------------------------------
// CTA l of 3 writes the shift of layer l (W0 cost slice, W1, W2): largest finite |w| mapped into [2^14, 2^15).
__global__ void __launch_bounds__(1024) gnet_weight_scale_kernel(const float* __restrict__ w0, int n0,
                                                                 const float* __restrict__ w1,
                                                                 const float* __restrict__ w2,
                                                                 int* __restrict__ shifts) {
  const float* w = blockIdx.x == 0 ? w0 : blockIdx.x == 1 ? w1 : w2;
  const int n = blockIdx.x == 0 ? n0 : HID * HID;
  unsigned m = 0u;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const unsigned u = __float_as_uint(w[i]) & 0x7fffffffu;
    m = max(m, u >= 0x7f800000u ? 0u : u);
  }
  m = __reduce_max_sync(0xffffffffu, m);
  __shared__ unsigned red[32];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) m = max(m, red[i]);
    m = max(m, red[0]);
    shifts[blockIdx.x] = split16_shift(m);
  }
}

// One thread per 16-byte fragment of W1, W2 and W0 (in that order), then the fp32 vectors.  Fragment (k step, n tile,
// lane): n = 8*tile + lane/4, k = 16*step + 2*(lane%4) + {0, 1, 8, 9}.  W0's k step is (16-channel chunk, tap).
__global__ void __launch_bounds__(256) gnet_pack_kernel(const float* __restrict__ w0, const float* __restrict__ w1,
                                                        const float* __restrict__ b1, const float* __restrict__ w2,
                                                        const float* __restrict__ b2, const float* __restrict__ w3,
                                                        const float* __restrict__ b3, int D, int n_frag,
                                                        unsigned char* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int* shifts = reinterpret_cast<const int*>(dst + G_HDR);
  if (i < G_NVEC) {
    float* vec = reinterpret_cast<float*>(dst + G_VEC);
    vec[i] = i < HID ? b1[i] : i < 2 * HID ? b2[i - HID] : i < 4 * HID ? w3[i - 2 * HID] : b3[i - 4 * HID];
  }
  if (i >= n_frag) return;
  const int per_layer = (int)(G_LAYER / 16);
  const int layer = i < per_layer ? 1 : i < 2 * per_layer ? 2 : 0;
  const int f = layer == 1 ? i : layer == 2 ? i - per_layer : i - 2 * per_layer;
  const int lane = f & 31, nt = (f >> 5) % NTILE, step = (f >> 5) / NTILE;
  const int n = nt * 8 + (lane >> 2);
  const float s = pow2(shifts[layer]);
  float v[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int kk = 2 * (lane & 3) + (e & 1) + (e >> 1) * 8;            // 0,1 -> b0 ; 8,9 -> b1
    if (layer == 0) {
      const int cs = step / 9, tap = step - cs * 9, c = cs * CCH + kk;
      v[e] = c < D ? w0[((size_t)n * D + c) * 9 + tap] : 0.0f;
    } else {
      v[e] = (layer == 1 ? w1 : w2)[n * HID + step * 16 + kk];
    }
  }
  uint32_t h0, l0, h1, l1;
  split2(__fmul_rn(v[0], s), __fmul_rn(v[1], s), h0, l0);
  split2(__fmul_rn(v[2], s), __fmul_rn(v[3], s), h1, l1);
  const size_t base = layer == 1 ? G_W1 : layer == 2 ? G_W2 : G_W0;
  reinterpret_cast<uint4*>(dst + base)[f] = make_uint4(h0, h1, l0, l1);
}
}  // namespace

cudaError_t launch_gnet_pack(const float* w0, const float* w1, const float* b1, const float* w2, const float* b2,
                             const float* w3, const float* b3, int D, void* dst, cudaStream_t st) {
  unsigned char* d = static_cast<unsigned char*>(dst);
  gnet_weight_scale_kernel<<<3, 1024, 0, st>>>(w0, HID * D * 9, w1, w2, reinterpret_cast<int*>(d + G_HDR));
  const int n_frag = (int)((gnet_weights_bytes(D) - G_W1) / 16);
  gnet_pack_kernel<<<(n_frag + 255) / 256, 256, 0, st>>>(w0, w1, b1, w2, b2, w3, b3, D, n_frag, d);
  return cudaGetLastError();
}

namespace {
template <bool SAVE>
cudaError_t launch_gnet_head(int B, int D, int H, int W, const float* cost, const float* inv, const void* weights,
                             const float* prev, unsigned* scratch, float* out, float* save, cudaStream_t st) {
  static std::once_flag flags[64];
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  cudaError_t res = cudaSuccess;
  std::call_once(flags[dev & 63], [&] {
    res = cudaFuncSetAttribute(gnet_head_kernel<SAVE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S_TOTAL);
  });
  if (res != cudaSuccess) return res;
  if ((e = launch_absmax_f32(cost, (size_t)B * D * H * W, scratch, st)) != cudaSuccess) return e;
  GnetParams p;
  p.B = B; p.D = D; p.H = H; p.W = W;
  p.ncs = (D + CCH - 1) / CCH;
  p.tiles_x = (W + TX - 1) / TX;
  p.tiles_y = (H + TY - 1) / TY;
  p.ntiles = B * p.tiles_x * p.tiles_y;
  p.cost = cost; p.inv = inv; p.weights = static_cast<const unsigned char*>(weights); p.prev = prev;
  p.absmax = scratch; p.out = out; p.save = save;
  gnet_head_kernel<SAVE><<<std::min(p.ntiles, sm_count(dev)), NT, S_TOTAL, st>>>(p);   // persistent: one CTA per SM
  return cudaGetLastError();
}
}  // namespace

cudaError_t launch_gnet_update(int B, int D, int H, int W, const float* cost, const float* inv, const void* weights,
                               const float* prev, unsigned* scratch, float* out, cudaStream_t st) {
  return launch_gnet_head<false>(B, D, H, W, cost, inv, weights, prev, scratch, out, nullptr, st);
}

// ================================================ training (DESIGN §3.10) ==========================================
// Training pack: the inference pack, then W1^T and W2^T as B fragments of the same form (layer shifts of the header).
size_t gnet_train_weights_bytes(int D) { return gnet_weights_bytes(D) + 2 * G_LAYER; }
size_t gnet_saved_bytes(int B, int H, int W) { return (size_t)(3 * HID + 2) * B * H * W * 4; }

namespace {
constexpr int WG_KS = 32;            // pixels per shared-memory slab of the weight-gradient GEMMs
constexpr int WG_KC = 1024;          // pixels per CTA (one partial per CTA and output element)
constexpr int WG_M = 128, WG_N = 64; // CTA output tile
constexpr int WG_SA = WG_M + 8, WG_SB = WG_N + 8;   // row strides = 8 mod 32 banks: conflict-free fragment loads
constexpr size_t WG_SMEM = (size_t)2 * WG_KS * (WG_SA + WG_SB) * 4;

int wgrad_chunks(int P) { return (P + WG_KC - 1) / WG_KC; }
size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }
}  // namespace

// backward scratch: d_h2, d_h1 (B,128,H,W), d_raw (B,2,H,W), the GEMM partials (one set, reused by the four GEMMs)
size_t gnet_bwd_workspace_bytes(int B, int D, int H, int W) {
  const size_t map = (size_t)B * H * W * 4;
  const size_t ncols = (size_t)std::max(HID, 9 * D);
  return align256(2 * HID * map) + align256(2 * map) + align256((size_t)wgrad_chunks(B * H * W) * HID * (ncols + 1) * 4);
}

namespace {
// W1^T (layer 0 of the tail) and W2^T: Bmat[k][n] = W[k][n], fragment order as gnet_pack_kernel
__global__ void __launch_bounds__(256) gnet_pack_t_kernel(const float* __restrict__ w1, const float* __restrict__ w2,
                                                          unsigned char* __restrict__ dst, size_t tail) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int per_layer = (int)(G_LAYER / 16);
  if (i >= 2 * per_layer) return;
  const int layer = i / per_layer, f = i - layer * per_layer;
  const int lane = f & 31, nt = (f >> 5) % NTILE, step = (f >> 5) / NTILE;
  const int n = nt * 8 + (lane >> 2);
  const float* w = layer == 0 ? w1 : w2;
  const float s = pow2(reinterpret_cast<const int*>(dst + G_HDR)[1 + layer]);
  float v[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) v[e] = w[(step * 16 + 2 * (lane & 3) + (e & 1) + (e >> 1) * 8) * HID + n];
  uint32_t h0, l0, h1, l1;
  split2(__fmul_rn(v[0], s), __fmul_rn(v[1], s), h0, l0);
  split2(__fmul_rn(v[2], s), __fmul_rn(v[3], s), h1, l1);
  reinterpret_cast<uint4*>(dst + tail)[i] = make_uint4(h0, h1, l0, l1);
}

struct GnetBwdParams {
  int B, HW, gpi, ngroups;                   // gpi: 16-pixel groups per image
  const float* __restrict__ grad;            // (B,2,H,W) gradient of the updated Gaussian
  const float* __restrict__ prev;            // (B,2,H,W)
  const float* __restrict__ save;            // the training forward's h0, h1, h2, raw
  const unsigned char* __restrict__ weights; // training pack: header and fp32 vectors of its inference part ...
  const unsigned char* __restrict__ wt;      // ... and its tail, W1^T then W2^T
  float* __restrict__ grad_inv;              // (B,128,H,W) = d_h0
  float* __restrict__ dh;                    // d_h2, d_h1 (B,128,H,W), d_raw (B,2,H,W)
  float* __restrict__ grad_prev;             // (B,2,H,W) or NULL
};

// Per warp 16 consecutive pixels of one image (rows g and g+8 of the MMA): d_raw from the update's derivative,
// d_h2 = (W3^T d_raw) [h2 > 0] on the CUDA cores, d_h1 = (W2^T d_h2) [h1 > 0] and d_h0 = (W1^T d_h1) [h0 > 0] on the
// tensor cores.  Pixels past the image carry zeros.
__global__ void __launch_bounds__(NT, 1) gnet_bwd_chain_kernel(const GnetBwdParams p) {
  extern __shared__ __align__(16) unsigned char smem[];
  uint4* wt = reinterpret_cast<uint4*>(smem);                       // W1^T then W2^T, resident
  float* w3 = reinterpret_cast<float*>(smem + S_W12);               // W3 [2][128]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, q = lane & 3;
  {
    const uint4* src = reinterpret_cast<const uint4*>(p.wt);
    for (int i = tid; i < (int)(S_W12 / 16); i += NT) wt[i] = __ldg(src + i);
    const float* vs = reinterpret_cast<const float*>(p.weights + G_VEC) + 2 * HID;
    for (int i = tid; i < 2 * HID; i += NT) w3[i] = __ldg(vs + i);
  }
  __syncthreads();
  const int* shw = reinterpret_cast<const int*>(p.weights + G_HDR);
  const int sh_w1 = __ldg(shw + 1), sh_w2 = __ldg(shw + 2);
  const int HW = p.HW;
  const size_t plane = (size_t)p.B * HID * HW;
  const float* h0s = p.save;
  const float* h1s = p.save + plane;
  const float* h2s = p.save + 2 * plane;
  const float* raws = p.save + 3 * plane;
  float* dh2 = p.dh;
  float* dh1 = p.dh + plane;
  float* draw = p.dh + 2 * plane;

  for (int base = blockIdx.x * (NT / 32); base < p.ngroups; base += gridDim.x * (NT / 32)) {
    const int gi = base + warp;
    if (gi >= p.ngroups) break;
    const int b = gi / p.gpi, hw0 = (gi - b * p.gpi) * 16;
    const int pa = hw0 + g, pb = hw0 + g + 8;
    const bool va = pa < HW, vb = pb < HW;
    // ---- d_raw from the update's derivative ----
    float d[4] = {0.0f, 0.0f, 0.0f, 0.0f};     // (d_mu1, d_sigma1) of pixels pa, pb
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int px = r == 0 ? pa : pb;
      if (!(r == 0 ? va : vb)) continue;
      const size_t o = (size_t)b * 2 * HW + px;
      const float g_mu = __ldg(p.grad + o), g_sg = __ldg(p.grad + o + HW);
      const float mu1 = __ldg(raws + o), s1 = __ldg(raws + o + HW);
      gaussian_update_bwd(g_mu, g_sg, s1, __ldg(p.prev + o + HW), d[2 * r], d[2 * r + 1]);
      if (q == r) {
        draw[o] = d[2 * r];
        draw[o + HW] = d[2 * r + 1];
        if (p.grad_prev) {
          float d_mu0, d_s0;
          gaussian_update_bwd_prev(g_mu, g_sg, mu1, s1, d_mu0, d_s0);
          p.grad_prev[o] = d_mu0;
          p.grad_prev[o + HW] = d_s0;
        }
      }
    }
    // offset of channel 2q of pixel pa in a (B,128,H,W) map
    const size_t off = ((size_t)b * HID + 2 * q) * HW + (va ? pa : 0);
    // ---- d_h2 on the CUDA cores ----
    float acc[NTILE][4];
#pragma unroll
    for (int nt = 0; nt < NTILE; ++nt) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = nt * 8 + 2 * q + e;
        const float wm = w3[c], ws = w3[HID + c];
        acc[nt][e] = __fmaf_rn(ws, d[1], __fmul_rn(wm, d[0]));
        acc[nt][2 + e] = __fmaf_rn(ws, d[3], __fmul_rn(wm, d[2]));
      }
    }
    relu_mask(acc, h2s + off, HW, va, vb);
    store_rows(dh2 + off, acc, HW, va, vb);
    // ---- d_h1, d_h0 on the tensor cores ----
#pragma unroll 1
    for (int l = 0; l < 2; ++l) {
      grad_layer(acc, acc, wt + (l == 0 ? G_LAYER / 16 : 0), l == 0 ? sh_w2 : sh_w1, lane);
      relu_mask(acc, (l == 0 ? h1s : h0s) + off, HW, va, vb);
      store_rows((l == 0 ? dh1 : p.grad_inv) + off, acc, HW, va, vb);
    }
  }
}

// ---- weight gradients: out[m][n] = sum over pixels of A_m(p) B_n(p), 3xTF32 on the tensor cores ----
struct WgradParams {
  int HW, H, W, P, Ma, Nw, D, im2col;
  const float* __restrict__ a;      // (B, Ma, HW)
  const float* __restrict__ bsrc;   // dense: (B, Nw, HW); im2col: the cost volume (B, D, H, W), n = 9c + tap
  float* __restrict__ part_w;       // [chunk][Ma][Nw]
  float* __restrict__ part_b;       // [chunk][Ma] (sum of A over the pixels: the bias gradient) or NULL
};

__device__ __forceinline__ uint32_t tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void mma1688(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                        uint32_t b1) {
  asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// CTA (chunk, n block): its WG_KC pixels in slabs of WG_KS; each operand element is split x = hi + lo (tf32) once on
// its way into shared memory; per k8 step three products lo*hi + hi*lo + hi*hi into the fp32 accumulators.
__global__ void __launch_bounds__(256, 2) gnet_wgrad_kernel(const WgradParams p) {
  extern __shared__ __align__(16) float wsm[];
  uint32_t* ah = reinterpret_cast<uint32_t*>(wsm);
  uint32_t* al = ah + WG_KS * WG_SA;
  uint32_t* bh = al + WG_KS * WG_SA;
  uint32_t* bl = bh + WG_KS * WG_SB;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, q = lane & 3;
  const int wm = warp & 3, wn = warp >> 2;
  const int chunk = blockIdx.x, n0 = blockIdx.y * WG_N;
  const int k_begin = chunk * WG_KC, k_end = min(p.P, k_begin + WG_KC);
  const bool bias = p.part_b != nullptr && blockIdx.y == 0;
  float tot[2][4][4];        // the CTA's sums; each slab's MMAs accumulate from zero and are added here (IEEE adds)
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) tot[mt][nt][0] = tot[mt][nt][1] = tot[mt][nt][2] = tot[mt][nt][3] = 0.0f;
  float bsum[4] = {0.0f, 0.0f, 0.0f, 0.0f};
  const int lk = tid & 7, lr = tid >> 3;     // loader: pixel k = lk + 8*kk of the slab, row / column lr + 32*j
  const bool warp_live = wm * 32 < p.Ma;

  for (int k0 = k_begin; k0 < k_end; k0 += WG_KS) {
    int pb_[4], phw[4], py[4], px[4];
    bool pv[4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const int pix = k0 + lk + 8 * kk;
      pv[kk] = pix < k_end;
      pb_[kk] = pv[kk] ? pix / p.HW : 0;
      phw[kk] = pv[kk] ? pix - pb_[kk] * p.HW : 0;
      py[kk] = phw[kk] / p.W;
      px[kk] = phw[kk] - py[kk] * p.W;
    }
    __syncthreads();                                   // the previous slab is consumed
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = lr + 32 * j;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const float v = pv[kk] && m < p.Ma ? __ldg(p.a + ((size_t)pb_[kk] * p.Ma + m) * p.HW + phw[kk]) : 0.0f;
        bsum[j] = __fadd_rn(bsum[j], v);
        const uint32_t h = tf32(v);
        const int k = lk + 8 * kk;
        ah[k * WG_SA + m] = h;
        al[k * WG_SA + m] = tf32(__fsub_rn(v, __uint_as_float(h)));
      }
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int n = n0 + lr + 32 * j;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        float v = 0.0f;
        if (pv[kk] && n < p.Nw) {
          if (p.im2col) {
            const int c = n / 9, tap = n - 9 * c;
            const int yy = py[kk] + tap / 3 - 1, xx = px[kk] + tap % 3 - 1;
            if (yy >= 0 && yy < p.H && xx >= 0 && xx < p.W)
              v = __ldg(p.bsrc + ((size_t)pb_[kk] * p.D + c) * p.HW + (size_t)yy * p.W + xx);
          } else {
            v = __ldg(p.bsrc + ((size_t)pb_[kk] * p.Nw + n) * p.HW + phw[kk]);
          }
        }
        const uint32_t h = tf32(v);
        const int k = lk + 8 * kk;
        bh[k * WG_SB + n - n0] = h;
        bl[k * WG_SB + n - n0] = tf32(__fsub_rn(v, __uint_as_float(h)));
      }
    }
    __syncthreads();
    if (warp_live) {
      float acc[2][4][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) acc[mt][nt][0] = acc[mt][nt][1] = acc[mt][nt][2] = acc[mt][nt][3] = 0.0f;
#pragma unroll
      for (int ks = 0; ks < WG_KS / 8; ++ks) {
        const int r0 = (ks * 8 + q) * WG_SA, r1 = r0 + 4 * WG_SA;
        uint32_t fh[2][4], fl[2][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          const int m = wm * 32 + mt * 16 + g;
          fh[mt][0] = ah[r0 + m]; fh[mt][1] = ah[r0 + m + 8]; fh[mt][2] = ah[r1 + m]; fh[mt][3] = ah[r1 + m + 8];
          fl[mt][0] = al[r0 + m]; fl[mt][1] = al[r0 + m + 8]; fl[mt][2] = al[r1 + m]; fl[mt][3] = al[r1 + m + 8];
        }
        const int s0 = (ks * 8 + q) * WG_SB, s1 = s0 + 4 * WG_SB;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int n = wn * 32 + nt * 8 + g;
          const uint32_t b0h = bh[s0 + n], b1h = bh[s1 + n], b0l = bl[s0 + n], b1l = bl[s1 + n];
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            mma1688(acc[mt][nt], fl[mt][0], fl[mt][1], fl[mt][2], fl[mt][3], b0h, b1h);
            mma1688(acc[mt][nt], fh[mt][0], fh[mt][1], fh[mt][2], fh[mt][3], b0l, b1l);
            mma1688(acc[mt][nt], fh[mt][0], fh[mt][1], fh[mt][2], fh[mt][3], b0h, b1h);
          }
        }
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) tot[mt][nt][e] = __fadd_rn(tot[mt][nt][e], acc[mt][nt][e]);
    }
  }
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int m = wm * 32 + mt * 16 + g + (e >> 1) * 8, n = n0 + wn * 32 + nt * 8 + 2 * q + (e & 1);
        if (m < p.Ma && n < p.Nw) p.part_w[((size_t)chunk * p.Ma + m) * p.Nw + n] = tot[mt][nt][e];
      }
    }
  }
  if (bias) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float s = bsum[j];
      s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 1));
      s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 2));
      s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 4));
      const int m = lr + 32 * j;
      if (lk == 0 && m < p.Ma) p.part_b[(size_t)chunk * p.Ma + m] = s;
    }
  }
}

// fixed-order sum of the per-CTA partials
__global__ void __launch_bounds__(256) gnet_wgrad_reduce_kernel(const float* __restrict__ part, int nchunk, int count,
                                                                float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  float s = 0.0f;
  for (int c = 0; c < nchunk; ++c) s = __fadd_rn(s, __ldg(part + (size_t)c * count + i));
  out[i] = s;
}

cudaError_t launch_wgrad(int B, int H, int W, int Ma, const float* a, int Nw, int D, bool im2col, const float* bsrc,
                         float* part, float* out_w, float* out_b, cudaStream_t st) {
  WgradParams p;
  p.HW = H * W; p.H = H; p.W = W; p.P = B * H * W; p.Ma = Ma; p.Nw = Nw; p.D = D; p.im2col = im2col ? 1 : 0;
  p.a = a; p.bsrc = bsrc;
  const int nchunk = wgrad_chunks(p.P);
  p.part_w = part;
  p.part_b = out_b ? part + (size_t)nchunk * Ma * Nw : nullptr;
  gnet_wgrad_kernel<<<dim3(nchunk, (Nw + WG_N - 1) / WG_N), 256, WG_SMEM, st>>>(p);
  if (out_w) {
    const int count = Ma * Nw;
    gnet_wgrad_reduce_kernel<<<(count + 255) / 256, 256, 0, st>>>(part, nchunk, count, out_w);
  }
  if (out_b) gnet_wgrad_reduce_kernel<<<(Ma + 255) / 256, 256, 0, st>>>(p.part_b, nchunk, Ma, out_b);
  return cudaGetLastError();
}
}  // namespace

// The same weight-gradient GEMMs for the mask head's training (mask_head.cu): out_w[m][n] = sum over the B*H*W pixels
// of a[m] b[n] on dense (B, Ma, H, W) / (B, Nw, H, W) maps, Ma <= 128, out_b[m] = sum of a[m].  `part` holds
// head_wgrad_partial_floats(B, H, W, Ma, Nw) floats.
size_t head_wgrad_partial_floats(int B, int H, int W, int Ma, int Nw) {
  return (size_t)wgrad_chunks(B * H * W) * Ma * (Nw + 1);
}

cudaError_t launch_head_wgrad(int B, int H, int W, int Ma, const float* a, int Nw, const float* b, float* part,
                              float* out_w, float* out_b, cudaStream_t st) {
  static std::once_flag flags[64];
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  cudaError_t res = cudaSuccess;
  std::call_once(flags[dev & 63], [&] {
    res = cudaFuncSetAttribute(gnet_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WG_SMEM);
  });
  if (res != cudaSuccess) return res;
  return launch_wgrad(B, H, W, Ma, a, Nw, 0, false, b, part, out_w, out_b, st);
}

cudaError_t launch_gnet_pack_train(const float* w0, const float* w1, const float* b1, const float* w2, const float* b2,
                                   const float* w3, const float* b3, int D, void* dst, cudaStream_t st) {
  cudaError_t e = launch_gnet_pack(w0, w1, b1, w2, b2, w3, b3, D, dst, st);
  if (e != cudaSuccess) return e;
  const int n = (int)(2 * G_LAYER / 16);
  gnet_pack_t_kernel<<<(n + 255) / 256, 256, 0, st>>>(w1, w2, static_cast<unsigned char*>(dst), gnet_weights_bytes(D));
  return cudaGetLastError();
}

cudaError_t launch_gnet_train_fwd(int B, int D, int H, int W, const float* cost, const float* inv, const void* weights,
                                  const float* prev, unsigned* scratch, float* out, float* saved, cudaStream_t st) {
  return launch_gnet_head<true>(B, D, H, W, cost, inv, weights, prev, scratch, out, saved, st);
}

// Launches: the chain kernel, then per requested (weight, bias) pair one GEMM and one or two reductions.
cudaError_t launch_gnet_bwd(int B, int D, int H, int W, const float* cost, const float* prev, const void* weights,
                            const float* saved, const float* grad, void* workspace, float* grad_inv, float* gw0,
                            float* gw1, float* gb1, float* gw2, float* gb2, float* gw3, float* gb3, float* grad_prev,
                            cudaStream_t st, int* launches) {
  static std::once_flag flags[64];
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  cudaError_t res = cudaSuccess;
  std::call_once(flags[dev & 63], [&] {
    res = cudaFuncSetAttribute(gnet_bwd_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(S_W12 + 2 * HID * 4));
    if (res == cudaSuccess)
      res = cudaFuncSetAttribute(gnet_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WG_SMEM);
  });
  if (res != cudaSuccess) return res;
  const int HW = H * W;
  const size_t map = (size_t)B * HW;
  float* dh = static_cast<float*>(workspace);
  float* part = reinterpret_cast<float*>(static_cast<unsigned char*>(workspace) + align256(2 * HID * map * 4) +
                                         align256(2 * map * 4));
  const unsigned char* wb = static_cast<const unsigned char*>(weights);
  GnetBwdParams p;
  p.B = B; p.HW = HW; p.gpi = (HW + 15) / 16; p.ngroups = B * p.gpi;
  p.grad = grad; p.prev = prev; p.save = saved; p.weights = wb; p.wt = wb + gnet_weights_bytes(D);
  p.grad_inv = grad_inv; p.dh = dh; p.grad_prev = grad_prev;
  const int ctas = std::min((p.ngroups + NT / 32 - 1) / (NT / 32), sm_count(dev));
  gnet_bwd_chain_kernel<<<ctas, NT, S_W12 + 2 * HID * 4, st>>>(p);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  int n = 1;
  const size_t plane = (size_t)HID * map;
  const float* h0 = saved;
  const float* h1 = saved + plane;
  const float* h2 = saved + 2 * plane;
  auto pair = [&](float* w, float* bias) { return (w ? 1 : 0) + (bias ? 1 : 0) + 1; };
  if (gw1 || gb1) {          // dW1 = sum d_h1 h0^T, db1 = sum d_h1
    if ((e = launch_wgrad(B, H, W, HID, dh + plane, HID, D, false, h0, part, gw1, gb1, st)) != cudaSuccess) return e;
    n += pair(gw1, gb1);
  }
  if (gw2 || gb2) {          // dW2 = sum d_h2 h1^T, db2 = sum d_h2
    if ((e = launch_wgrad(B, H, W, HID, dh, HID, D, false, h1, part, gw2, gb2, st)) != cudaSuccess) return e;
    n += pair(gw2, gb2);
  }
  if (gw3 || gb3) {          // dW3 = sum d_raw h2^T, db3 = sum d_raw
    if ((e = launch_wgrad(B, H, W, 2, dh + 2 * plane, HID, D, false, h2, part, gw3, gb3, st)) != cudaSuccess) return e;
    n += pair(gw3, gb3);
  }
  if (gw0) {                 // dW0[o][c][tap] = sum d_h0[o] cost[c](p + tap)
    if ((e = launch_wgrad(B, H, W, HID, grad_inv, 9 * D, D, true, cost, part, gw0, nullptr, st)) != cudaSuccess) return e;
    n += 2;
  }
  *launches = n;
  return cudaSuccess;
}

}  // namespace magnet
