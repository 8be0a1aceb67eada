// Mask head and learned upsampling of inference in one kernel (DESIGN §3.12): per 8x16 pixel tile, the ReLU of the
// hoisted first layer, the two 128 -> 128 layers, the 128 -> 144 layer, the softmax over the 9 taps and the convex
// combination of every prediction (upsample_depth_via_mask, MAGNET.py:15-27,111-118,172-173).  Neither a 128-channel
// map nor the 144-channel mask leaves the SM; the full-resolution Gaussians are written once.
//
// GEMMs run on the fp16 tensor cores in the SPLIT16 scheme of the G-Net head (head_common.cuh): one shift per layer
// for the weights (chosen by the pack), one per pixel for the activations, three products, exact descale.
#include <algorithm>
#include <mutex>

#include "head_common.cuh"
#include "upsample_common.cuh"

namespace magnet {

int sm_count(int dev);   // cost_mma.cu

namespace {
constexpr int K_UP = 4;                        // upsampling factor: 9 taps x 4 x 4 sub-pixels = 144 mask channels
constexpr int NOUT = 9 * K_UP * K_UP;
constexpr int NTILE3 = NOUT / 8;               // n8 tiles of the 144-channel layer; tile 2i+h = tap i, sub-pixels 8h..8h+7
constexpr int TY = 8, TX = 16;                 // pixel tile of a CTA: warp w owns row w (16 pixels = the MMA's M)
constexpr int HX = TX + 2, HP = (TY + 2) * HX; // the tile's 3x3 neighbourhood, 180 pixels
constexpr int NT = 32 * TY;
constexpr int MAX_PRED = MAGNET_MASK_MAX_PRED;

// Packed weight buffer (magnet_mask_pack_weights_f32): B fragments in the order the MMA consumes them, per (K step,
// n8 tile) 32 lanes x 16 bytes {hi(b0), hi(b1), lo(b0), lo(b1)}, as the G-Net pack.
constexpr size_t M_HDR = 0;                    // int32 shift of W1, W2, W3
constexpr size_t M_VEC = 256;                  // fp32 b1[128], b2[128], b3[144]
constexpr int M_NVEC = 2 * HID + NOUT;
constexpr size_t M_W1 = 4096;
constexpr size_t M_LAYER = (size_t)(HID / 16) * NTILE * 32 * 16;     // 64 KiB per 128x128 layer
constexpr size_t M_W2 = M_W1 + M_LAYER;
constexpr size_t M_W3 = M_W2 + M_LAYER;
constexpr size_t M_LAYER3 = (size_t)(HID / 16) * NTILE3 * 32 * 16;   // 72 KiB
constexpr size_t M_BYTES = M_W3 + M_LAYER3;

constexpr size_t S_W = M_BYTES - M_W1;                               // W1, W2, W3 resident
constexpr size_t S_VEC = ((M_NVEC * 4 + 15) / 16) * 16;
constexpr size_t S_NB = (size_t)2 * HP * 4;                          // per prediction: [mu, sigma][HP] fp32
static_assert(M_VEC + M_NVEC * 4 <= M_W1, "vectors fit before W1");
static_assert(S_W + S_VEC + MAX_PRED * S_NB <= 227 * 1024, "one CTA per SM");

size_t smem_bytes(int P) { return S_W + S_VEC + (size_t)P * S_NB; }

struct MaskParams {
  int B, H, W, P, tiles_x, tiles_y, ntiles;
  const float* __restrict__ pre0;
  const unsigned char* __restrict__ weights;
  const float* pred[MAX_PRED];
  float* out[MAX_PRED];
};

__global__ void __launch_bounds__(NT, 1) mask_upsample_kernel(const MaskParams p) {
  extern __shared__ __align__(16) unsigned char smem[];
  uint4* wsm = reinterpret_cast<uint4*>(smem);                          // W1, W2, W3
  float* vec = reinterpret_cast<float*>(smem + S_W);                    // b1, b2, b3
  float* nb = reinterpret_cast<float*>(smem + S_W + S_VEC);            // [P][mu, sigma][HP]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, q = lane & 3;
  const int H = p.H, W = p.W, HW = H * W;
  {
    const uint4* src = reinterpret_cast<const uint4*>(p.weights + M_W1);
    for (int i = tid; i < (int)(S_W / 16); i += NT) wsm[i] = __ldg(src + i);
    const float* vs = reinterpret_cast<const float*>(p.weights + M_VEC);
    for (int i = tid; i < M_NVEC; i += NT) vec[i] = __ldg(vs + i);
  }
  const int* shw = reinterpret_cast<const int*>(p.weights + M_HDR);
  const int sh_w1 = __ldg(shw + 0), sh_w2 = __ldg(shw + 1), sh_w3 = __ldg(shw + 2);
  const uint4* w3 = wsm + 2 * M_LAYER / 16;
  const float* b3 = vec + 2 * HID;
  const float dw3 = pow2(-sh_w3);
  const int per_img = p.tiles_x * p.tiles_y;

  for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
    const int b = tile / per_img, t = tile - b * per_img, ty = t / p.tiles_x;
    const int y0 = ty * TY, x0 = (t - ty * p.tiles_x) * TX, y = y0 + warp;

    // ---- the tile's 3x3 neighbourhood of every prediction, zeros outside the image ----
    __syncthreads();                                   // every warp is done with the previous tile's neighbourhood
#pragma unroll
    for (int pp = 0; pp < MAX_PRED; ++pp) {
      if (pp >= p.P) break;
      const float* src = p.pred[pp] + (size_t)b * 2 * HW;
      for (int i = tid; i < 2 * HP; i += NT) {
        const int c = i / HP, hp = i - c * HP;
        const int yy = y0 - 1 + hp / HX, xx = x0 - 1 + hp % HX;
        nb[pp * 2 * HP + i] = yy >= 0 && yy < H && xx >= 0 && xx < W ? __ldg(src + (size_t)c * HW + yy * W + xx) : 0.0f;
      }
    }

    // ---- h0 = ReLU(pre0), read once; the two hidden layers ----
    const int xa = x0 + g, xb = x0 + g + 8;
    const bool va = y < H && xa < W, vb = y < H && xb < W;
    const float* ip = p.pre0 + (size_t)b * HID * HW + (size_t)(va || vb ? y : 0) * W;
    float acc[NTILE][4];
#pragma unroll
    for (int nt = 0; nt < NTILE; ++nt) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const size_t n = (size_t)(nt * 8 + 2 * q + e) * HW;
        acc[nt][e] = va ? relu(__ldg(ip + n + xa)) : 0.0f;
        acc[nt][2 + e] = vb ? relu(__ldg(ip + n + xb)) : 0.0f;
      }
    }
    hidden_layer(acc, wsm, vec, sh_w1, lane);
    hidden_layer(acc, wsm + M_LAYER / 16, vec + HID, sh_w2, lane);
    uint32_t ah[HID / 16][4], al[HID / 16][4];
    int sh0, sh1;
    split_rows(acc, ah, al, sh0, sh1);
    const float d0 = pow2(-sh0), d1 = pow2(-sh1);
    __syncthreads();                                   // the neighbourhood is staged

    // ---- 128 -> 144 in two halves: tiles 2i+h hold tap i of sub-pixels 8h..8h+7, so each thread has all 9 taps of
    // sub-pixels s = 8h+2q+e (row ky = 2h + q/2, columns kx = 2(q&1)+e) of pixels xa and xb ----
#pragma unroll 1
    for (int h = 0; h < 2; ++h) {
      float lg[9][4];
#pragma unroll
      for (int i = 0; i < 9; ++i) lg[i][0] = lg[i][1] = lg[i][2] = lg[i][3] = 0.0f;
#pragma unroll
      for (int kk = 0; kk < HID / 16; ++kk) {
#pragma unroll
        for (int i = 0; i < 9; ++i) mma3(lg[i], ah[kk], al[kk], w3[(kk * NTILE3 + 2 * i + h) * 32 + lane]);
      }
#pragma unroll
      for (int i = 0; i < 9; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float bias = b3[(2 * i + h) * 8 + 2 * q + e];
          lg[i][e] = __fadd_rn(__fmul_rn(__fmul_rn(lg[i][e], d0), dw3), bias);
          lg[i][2 + e] = __fadd_rn(__fmul_rn(__fmul_rn(lg[i][2 + e], d1), dw3), bias);
        }
      }
      const int ky = 2 * h + (q >> 1), kx = 2 * (q & 1);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        if (!(r == 0 ? va : vb)) continue;
        const int xl = g + 8 * r, x = x0 + xl;
        float w[2][9];
#pragma unroll
        for (int e = 0; e < 2; ++e)
#pragma unroll
          for (int i = 0; i < 9; ++i) w[e][i] = lg[i][2 * r + e];
        const size_t o = ((size_t)b * 2 * H * K_UP + (size_t)y * K_UP + ky) * (size_t)(W * K_UP) + (size_t)x * K_UP + kx;
        const size_t cstride = (size_t)HW * K_UP * K_UP;
#pragma unroll
        for (int pp = 0; pp < MAX_PRED; ++pp) {
          if (pp >= p.P) break;
          const float* np = nb + pp * 2 * HP;
          auto tap = [&](int i, float& a, float& c) {
            const int yy = y + i / 3 - 1, xx = x + i % 3 - 1;
            const bool in = yy >= 0 && yy < H && xx >= 0 && xx < W;
            const int hp = (warp + i / 3) * HX + xl + i % 3;
            a = np[hp];
            c = np[HP + hp];
            return in;
          };
          float mu[2], sg[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (pp == 0) convex_gaussian(w[e], tap, mu[e], sg[e]);
            else convex_combine(w[e], tap, mu[e], sg[e]);
          }
          float* op = p.out[pp] + o;
          *reinterpret_cast<float2*>(op) = make_float2(mu[0], mu[1]);
          *reinterpret_cast<float2*>(op + cstride) = make_float2(sg[0], sg[1]);
        }
      }
    }
  }
}

// ---- weight pack --------------------------------------------------------------------------------------------------
// CTA l of 3 writes the shift of layer l + 1 (W1, W2, W3): largest finite |w| mapped into [2^14, 2^15).
__global__ void __launch_bounds__(1024) mask_weight_scale_kernel(const float* __restrict__ w1,
                                                                 const float* __restrict__ w2,
                                                                 const float* __restrict__ w3, int* __restrict__ shifts) {
  const float* w = blockIdx.x == 0 ? w1 : blockIdx.x == 1 ? w2 : w3;
  const int n = blockIdx.x == 2 ? NOUT * HID : HID * HID;
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

// One thread per 16-byte fragment of W1, W2 and W3, then the fp32 vectors.  Fragment (k step, n tile, lane):
// n = 8*tile + lane/4, k = 16*step + 2*(lane%4) + {0, 1, 8, 9}.
__global__ void __launch_bounds__(256) mask_pack_kernel(const float* __restrict__ w1, const float* __restrict__ b1,
                                                        const float* __restrict__ w2, const float* __restrict__ b2,
                                                        const float* __restrict__ w3, const float* __restrict__ b3,
                                                        unsigned char* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < M_NVEC) {
    float* vec = reinterpret_cast<float*>(dst + M_VEC);
    vec[i] = i < HID ? b1[i] : i < 2 * HID ? b2[i - HID] : b3[i - 2 * HID];
  }
  const int per_layer = (int)(M_LAYER / 16);
  if (i >= (int)(S_W / 16)) return;
  const int layer = i < per_layer ? 0 : i < 2 * per_layer ? 1 : 2;
  const int f = i - layer * per_layer;
  const int ntile = layer == 2 ? NTILE3 : NTILE;
  const int lane = f & 31, nt = (f >> 5) % ntile, step = (f >> 5) / ntile;
  const int n = nt * 8 + (lane >> 2);
  const float* w = layer == 0 ? w1 : layer == 1 ? w2 : w3;
  const float s = pow2(reinterpret_cast<const int*>(dst + M_HDR)[layer]);
  float v[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) v[e] = w[n * HID + step * 16 + 2 * (lane & 3) + (e & 1) + (e >> 1) * 8];
  uint32_t h0, l0, h1, l1;
  split2(__fmul_rn(v[0], s), __fmul_rn(v[1], s), h0, l0);
  split2(__fmul_rn(v[2], s), __fmul_rn(v[3], s), h1, l1);
  reinterpret_cast<uint4*>(dst + M_W1)[i] = make_uint4(h0, h1, l0, l1);
}
}  // namespace

size_t mask_weights_bytes() { return M_BYTES; }

cudaError_t launch_mask_pack(const float* w1, const float* b1, const float* w2, const float* b2, const float* w3,
                             const float* b3, void* dst, cudaStream_t st) {
  unsigned char* d = static_cast<unsigned char*>(dst);
  mask_weight_scale_kernel<<<3, 1024, 0, st>>>(w1, w2, w3, reinterpret_cast<int*>(d + M_HDR));
  const int n = (int)(S_W / 16);
  mask_pack_kernel<<<(n + 255) / 256, 256, 0, st>>>(w1, b1, w2, b2, w3, b3, d);
  return cudaGetLastError();
}

cudaError_t launch_mask_upsample(int P, int B, int H, int W, const float* pre0, const void* weights,
                                 const float* const* pred, float* const* out, cudaStream_t st) {
  static std::once_flag flags[64];
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  cudaError_t res = cudaSuccess;
  std::call_once(flags[dev & 63], [&] {
    res = cudaFuncSetAttribute(mask_upsample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)smem_bytes(MAX_PRED));
  });
  if (res != cudaSuccess) return res;
  MaskParams p;
  p.B = B; p.H = H; p.W = W; p.P = P;
  p.tiles_x = (W + TX - 1) / TX;
  p.tiles_y = (H + TY - 1) / TY;
  p.ntiles = B * p.tiles_x * p.tiles_y;
  p.pre0 = pre0;
  p.weights = static_cast<const unsigned char*>(weights);
  for (int i = 0; i < MAX_PRED; ++i) {
    p.pred[i] = i < P ? pred[i] : nullptr;
    p.out[i] = i < P ? out[i] : nullptr;
  }
  mask_upsample_kernel<<<std::min(p.ntiles, sm_count(dev)), NT, smem_bytes(P), st>>>(p);   // persistent
  return cudaGetLastError();
}

}  // namespace magnet
