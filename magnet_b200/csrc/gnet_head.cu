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

#include "common.cuh"
#include "gaussian_common.cuh"

namespace magnet {

int sm_count(int dev);                                                                   // cost_mma.cu
cudaError_t launch_absmax_f32(const float* x, size_t n, unsigned* out, cudaStream_t st);  // cost_mma.cu

namespace {
constexpr int HID = 128;                       // hidden channels
constexpr int NTILE = HID / 8;                 // n8 tiles of one layer's output
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
};

__device__ __forceinline__ float pow2(int e) { return __uint_as_float((unsigned)(127 + e) << 23); }   // |e| <= 126
__device__ __forceinline__ float relu(float v) { return v < 0.0f ? 0.0f : v; }                       // NaN stays NaN

__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {       // a: lower K index
  return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}
// two consecutive K elements, already scaled: x = hi + lo
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half h0 = __float2half_rn(x0), h1 = __float2half_rn(x1);
  hi = pack_h2(h0, h1);
  lo = pack_h2(__float2half_rn(__fsub_rn(x0, __half2float(h0))), __float2half_rn(__fsub_rn(x1, __half2float(h1))));
}

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// the three SPLIT16 products, small terms first
__device__ __forceinline__ void mma3(float (&c)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], uint4 b) {
  mma16816(c, al, b.x, b.y);
  mma16816(c, ah, b.z, b.w);
  mma16816(c, ah, b.x, b.y);
}

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}

// One 128 -> 128 layer on the accumulator fragment of the previous one (already ReLU'd): per-row scale and split into
// the A fragments (the m16n8 C layout of n tiles 2k, 2k+1 is the m16k16 A layout of K step k), three products against
// the resident weights, descale, bias, ReLU.  Rows g and g+8 of the warp's 16 pixels.
__device__ __forceinline__ void hidden_layer(float (&acc)[NTILE][4], const uint4* __restrict__ wsm,
                                             const float* __restrict__ bias, int shw, int lane) {
  float m0 = 0.0f, m1 = 0.0f;
#pragma unroll
  for (int nt = 0; nt < NTILE; ++nt) {
    m0 = fmaxf(m0, fmaxf(acc[nt][0], acc[nt][1]));
    m1 = fmaxf(m1, fmaxf(acc[nt][2], acc[nt][3]));
  }
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {                    // the quad shares a row
    m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, o));
    m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, o));
  }
  const int sh0 = split16_shift(__float_as_uint(m0)), sh1 = split16_shift(__float_as_uint(m1));
  const float s0 = pow2(sh0), s1 = pow2(sh1);
  uint32_t ah[HID / 16][4], al[HID / 16][4];
#pragma unroll
  for (int kk = 0; kk < HID / 16; ++kk) {
    split2(__fmul_rn(acc[2 * kk][0], s0), __fmul_rn(acc[2 * kk][1], s0), ah[kk][0], al[kk][0]);
    split2(__fmul_rn(acc[2 * kk][2], s1), __fmul_rn(acc[2 * kk][3], s1), ah[kk][1], al[kk][1]);
    split2(__fmul_rn(acc[2 * kk + 1][0], s0), __fmul_rn(acc[2 * kk + 1][1], s0), ah[kk][2], al[kk][2]);
    split2(__fmul_rn(acc[2 * kk + 1][2], s1), __fmul_rn(acc[2 * kk + 1][3], s1), ah[kk][3], al[kk][3]);
  }
#pragma unroll
  for (int nt = 0; nt < NTILE; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.0f;
#pragma unroll
  for (int kk = 0; kk < HID / 16; ++kk) {
#pragma unroll
    for (int nt = 0; nt < NTILE; ++nt) mma3(acc[nt], ah[kk], al[kk], wsm[(kk * NTILE + nt) * 32 + lane]);
  }
  const float dw = pow2(-shw), d0 = pow2(-sh0), d1 = pow2(-sh1);
  const int q = lane & 3;
#pragma unroll
  for (int nt = 0; nt < NTILE; ++nt) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const float b = bias[nt * 8 + 2 * q + e];
      acc[nt][e] = relu(__fadd_rn(__fmul_rn(__fmul_rn(acc[nt][e], d0), dw), b));
      acc[nt][2 + e] = relu(__fadd_rn(__fmul_rn(__fmul_rn(acc[nt][2 + e], d1), dw), b));
    }
  }
}

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

    hidden_layer(acc, w12, vec, sh_w1, lane);
    hidden_layer(acc, w12 + G_LAYER / 16, vec + HID, sh_w2, lane);

    // ---- 128 -> 2 on the CUDA cores, quad reduction, Gaussian update ----
    const float* w3 = vec + 2 * HID;
    float r[4] = {0.0f, 0.0f, 0.0f, 0.0f};               // (mu1, sigma1) of rows g and g+8
#pragma unroll
    for (int nt = 0; nt < NTILE; ++nt) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = nt * 8 + 2 * q + e;
        const float wm = w3[n], ws = w3[HID + n];
        r[0] = __fmaf_rn(acc[nt][e], wm, r[0]);
        r[1] = __fmaf_rn(acc[nt][e], ws, r[1]);
        r[2] = __fmaf_rn(acc[nt][2 + e], wm, r[2]);
        r[3] = __fmaf_rn(acc[nt][2 + e], ws, r[3]);
      }
    }
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
#pragma unroll
      for (int i = 0; i < 4; ++i) r[i] = __fadd_rn(r[i], __shfl_xor_sync(0xffffffffu, r[i], o));
    }
    if (q < 2 && (q == 0 ? va : vb)) {                  // lane 0 of the quad writes pixel g, lane 1 pixel g+8
      const size_t o = (size_t)b * 2 * HW + (size_t)y * p.W + (q == 0 ? xa : xb);
      const float mu1 = __fadd_rn(q == 0 ? r[0] : r[2], vec[4 * HID]);
      const float s1 = __fadd_rn(q == 0 ? r[1] : r[3], vec[4 * HID + 1]);
      float mu, sg;
      gaussian_update(mu1, s1, __ldg(p.prev + o), __ldg(p.prev + o + HW), mu, sg);
      p.out[o] = mu;
      p.out[o + HW] = sg;
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

cudaError_t launch_gnet_update(int B, int D, int H, int W, const float* cost, const float* inv, const void* weights,
                               const float* prev, unsigned* scratch, float* out, cudaStream_t st) {
  static std::once_flag flags[64];
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  cudaError_t res = cudaSuccess;
  std::call_once(flags[dev & 63], [&] {
    res = cudaFuncSetAttribute(gnet_head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S_TOTAL);
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
  p.absmax = scratch; p.out = out;
  gnet_head_kernel<<<std::min(p.ntiles, sm_count(dev)), NT, S_TOTAL, st>>>(p);   // persistent: one CTA per SM
  return cudaGetLastError();
}

}  // namespace magnet
