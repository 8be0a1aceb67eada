// Mask head and learned upsampling of inference in one kernel (DESIGN §3.12): per 8x16 pixel tile, the ReLU of the
// hoisted first layer, the two 128 -> 128 layers, the 128 -> 144 layer, the softmax over the 9 taps and the convex
// combination of every prediction (upsample_depth_via_mask, MAGNET.py:15-27,111-118,172-173).  Neither a 128-channel
// map nor the 144-channel mask leaves the SM; the full-resolution Gaussians are written once.  With one hidden layer
// and activation_G on the upsampled second channel the same kernel is D-Net's mask head (DESIGN §3.15).
//
// GEMMs run on the fp16 tensor cores in the SPLIT16 scheme of the G-Net head (head_common.cuh): one shift per layer
// for the weights (chosen by the pack), one per pixel for the activations, three products, exact descale.
#include <algorithm>
#include <mutex>

#include "head_common.cuh"
#include "launchers.h"
#include "upsample_common.cuh"

namespace magnet {

namespace {
constexpr int K_UP = 4;                        // upsampling factor: 9 taps x 4 x 4 sub-pixels = 144 mask channels
constexpr int NOUT = 9 * K_UP * K_UP;
constexpr int NTILE3 = NOUT / 8;               // n8 tiles of the 144-channel layer; tile 2i+h = tap i, sub-pixels 8h..8h+7
constexpr int TY = 8, TX = 16;                 // pixel tile of a CTA: warp w owns row w (16 pixels = the MMA's M)
constexpr int HX = TX + 2, HP = (TY + 2) * HX; // the tile's 3x3 neighbourhood, 180 pixels
constexpr int NT = 32 * TY;
constexpr int MAX_PRED = MAGNET_MASK_MAX_PRED;

// Packed weight buffer (magnet_mask_pack_weights_f32) in the SPLIT16 pack format of head_common.cuh.
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

// The inference pack of a mask head with NHID 128 -> 128 layers: 2 for MaGNet's (MAGNET.py:111-118, the layout above),
// 1 for D-Net's (D_dense_depth.py:156-160).  Header shifts of W1, [W2,] W3; vectors b1, [b2,] b3; then the fragments.
template <int NHID>
struct MaskLayout {
  static constexpr int NVEC = NHID * HID + NOUT;
  static constexpr size_t W = NHID * M_LAYER + M_LAYER3;              // resident weights
  static constexpr size_t VEC = ((NVEC * 4 + 15) / 16) * 16;
  static constexpr size_t BYTES = M_W1 + W;
};
static_assert(MaskLayout<2>::W == S_W && MaskLayout<2>::VEC == S_VEC && MaskLayout<2>::BYTES == M_BYTES, "");
static_assert(MaskLayout<1>::W + MaskLayout<1>::VEC + S_NB <= 227 * 1024, "D-Net: one prediction");

struct MaskParams {
  int B, H, W, P, tiles_x, tiles_y, ntiles;
  const float* __restrict__ pre0;
  const unsigned char* __restrict__ weights;
  const float* pred[MAX_PRED];
  float* out[MAX_PRED];
};

// ACT_G: the upsampled second channel goes through D-Net's activation_G (activation_g), so out = [mu, var].
template <int NHID, bool ACT_G>
__global__ void __launch_bounds__(NT, 1) mask_upsample_kernel(const MaskParams p) {
  using L = MaskLayout<NHID>;
  extern __shared__ __align__(16) unsigned char smem[];
  uint4* wsm = reinterpret_cast<uint4*>(smem);                          // W1, [W2,] W3
  float* vec = reinterpret_cast<float*>(smem + L::W);                   // b1, [b2,] b3
  float* nb = reinterpret_cast<float*>(smem + L::W + L::VEC);           // [P][mu, sigma][HP]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, q = lane & 3;
  const int H = p.H, W = p.W, HW = H * W;
  {
    const uint4* src = reinterpret_cast<const uint4*>(p.weights + M_W1);
    for (int i = tid; i < (int)(L::W / 16); i += NT) wsm[i] = __ldg(src + i);
    const float* vs = reinterpret_cast<const float*>(p.weights + M_VEC);
    for (int i = tid; i < L::NVEC; i += NT) vec[i] = __ldg(vs + i);
  }
  const int* shw = reinterpret_cast<const int*>(p.weights + M_HDR);
  const int sh_w1 = __ldg(shw + 0), sh_w2 = NHID == 2 ? __ldg(shw + 1) : 0, sh_w3 = __ldg(shw + NHID);
  const uint4* w3 = wsm + NHID * M_LAYER / 16;
  const float* b3 = vec + NHID * HID;
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
    if constexpr (NHID == 2) hidden_layer(acc, wsm + M_LAYER / 16, vec + HID, sh_w2, lane);
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
            if constexpr (ACT_G) sg[e] = activation_g(sg[e]);
          }
          float* op = p.out[pp] + o;
          *reinterpret_cast<float2*>(op) = make_float2(mu[0], mu[1]);
          *reinterpret_cast<float2*>(op + cstride) = make_float2(sg[0], sg[1]);
        }
      }
    }
  }
}

// ---- weight pack (DESIGN §3.16) ----
// The inference pack at `base` of p: header shifts of W1, [W2,] W3; fragments of W1, [W2,] W3; vectors b1, [b2,] b3.
template <int NHID>
void add_pack(HeadPack& p, const float* w1, const float* b1, const float* w2, const float* b2, const float* w3,
              const float* b3, size_t base) {
  const float* w[2] = {w1, w2};
  const float* b[2] = {b1, b2};
  for (int l = 0; l < NHID; ++l) {
    p.add_scale(w[l], HID * HID, base + M_HDR + 4 * l);
    p.add_frags(w[l], PACK_ROWS, HID / 16, NTILE, 0, base + M_HDR + 4 * l, base + M_W1 + l * M_LAYER);
    p.add_vec(b[l], HID, base + M_VEC + l * HID * 4);
  }
  p.add_scale(w3, NOUT * HID, base + M_HDR + 4 * NHID);
  p.add_frags(w3, PACK_ROWS, HID / 16, NTILE3, 0, base + M_HDR + 4 * NHID, base + M_W1 + NHID * M_LAYER);
  p.add_vec(b3, NOUT, base + M_VEC + NHID * HID * 4);
}
}  // namespace

size_t mask_weights_bytes() { return M_BYTES; }

namespace {
template <int NHID, bool ACT_G>
cudaError_t launch_upsample(int P, int B, int H, int W, const float* pre0, const void* weights,
                            const float* const* pred, float* const* out, cudaStream_t st) {
  using L = MaskLayout<NHID>;
  static std::once_flag flags[64];
  int dev = 0;
  cudaError_t e = set_smem_once(mask_upsample_kernel<NHID, ACT_G>, flags, (int)(L::W + L::VEC + MAX_PRED * S_NB),
                                false, &dev);
  if (e != cudaSuccess) return e;
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
  mask_upsample_kernel<NHID, ACT_G><<<std::min(p.ntiles, sm_count(dev)), NT, L::W + L::VEC + P * S_NB, st>>>(p);   // persistent
  return cudaGetLastError();
}
}  // namespace

cudaError_t launch_mask_pack(const float* w1, const float* b1, const float* w2, const float* b2, const float* w3,
                             const float* b3, void* dst, cudaStream_t st) {
  HeadPack p;
  add_pack<2>(p, w1, b1, w2, b2, w3, b3, 0);
  return launch_head_pack(p, dst, st);
}

cudaError_t launch_mask_upsample(int P, int B, int H, int W, const float* pre0, const void* weights,
                                 const float* const* pred, float* const* out, cudaStream_t st) {
  return launch_upsample<2, false>(P, B, H, W, pre0, weights, pred, out, st);
}

// D-Net's mask head (one hidden layer), its learned upsampling of the raw (mu, v) and activation_G (DESIGN §3.15):
// `weights` is the mask-head part of the D-Net pack.
size_t dnet_mask_weights_bytes() { return MaskLayout<1>::BYTES; }

void add_dnet_mask_pack(HeadPack& p, const float* w1, const float* b1, const float* w3, const float* b3, size_t base) {
  add_pack<1>(p, w1, b1, nullptr, nullptr, w3, b3, base);
}

cudaError_t launch_dnet_upsample(int B, int H, int W, const float* pre_m, const void* weights, const float* raw,
                                 float* out, cudaStream_t st) {
  return launch_upsample<1, true>(1, B, H, W, pre_m, weights, &raw, &out, st);
}

// ================================================ training (DESIGN §3.13) ==========================================
// The mask head, the upsampling and the Gaussian NLL of MagnetLoss (utils/losses.py:34-50) in one forward kernel that
// also forms the loss's gradient with respect to the 144 logits and the predictions while they are on chip; a
// tensor-core backward chain through the three 1x1 layers; the weight gradients on the G-Net head's fixed-order GEMMs.

namespace {
// d_logits is stored as channels 0..127 (B,128,H,W) followed by channels 128..143 (B,16,H,W): the weight-gradient GEMM
// takes at most 128 rows, so dW3 is two GEMMs on two dense maps.
constexpr int NOUT_HI = NOUT - HID;
// Training pack: the inference pack, then W3^T (9 K steps of the 144 logits x 16 n8 tiles), W2^T and W1^T as B
// fragments of the same form, under the header's layer shifts.
constexpr size_t M_LAYER3T = (size_t)(NOUT / 16) * NTILE * 32 * 16;  // 72 KiB
constexpr size_t S_WT = M_LAYER3T + 2 * M_LAYER;                     // the chain kernel's resident weights
constexpr size_t S_GP = S_NB;                                         // per prediction: [d mu, d sigma][HP] fp32
static_assert(S_W + S_VEC + MAX_PRED * (S_NB + S_GP) + 32 * MAX_PRED * 4 <= 227 * 1024, "one CTA per SM");
static_assert(S_WT <= 227 * 1024, "W3^T, W2^T, W1^T resident");

size_t smem_train(int P) { return S_W + S_VEC + (size_t)P * (S_NB + S_GP); }

struct MaskTrainParams {
  int B, H, W, P, tiles_x, tiles_y, ntiles;
  const float* __restrict__ pre0;
  const unsigned char* __restrict__ weights;
  const float* __restrict__ gt;
  const unsigned char* __restrict__ gtm;
  const float* pred[MAX_PRED];
  float scale[MAX_PRED];              // gamma_p / count: the NLL's gradient of prediction p at unit upstream gradient
  float* __restrict__ partial;        // [ntiles][P] loss partials
  float* __restrict__ saved;          // h0, h1, h2 (B,128,H,W) each, or NULL
  float* __restrict__ dlog;           // d_logits (B,128,H,W) + (B,16,H,W), or NULL
  float* __restrict__ gpred;          // P x (B,2,H,W) prediction gradients, accumulated; or NULL
  const float* __restrict__ scale_dev;  // DEV_SCALE: P device floats read in place of `scale`
};

// The inference kernel's tiles, layers and logits (bit for bit), then per full-resolution sub-pixel where gt_mask is
// set: the convex upsampling of every prediction, its NLL and the NLL's derivative (upsample_nll_fwd / bwd_kernel's
// expressions), the logits' gradient d = sum_p w (t_p - <w, t_p>) in prediction order, and the gradient into each
// prediction's 3x3 neighbourhood, gathered per tile in shared memory and added to global memory once per tile.
// DEV_SCALE: the prediction scales are read from device memory (p.scale_dev) at run time, so that a captured graph takes
// them from memory; otherwise they are the kernel parameters p.scale.
template <bool DEV_SCALE>
__global__ void __launch_bounds__(NT, 1) mask_train_fwd_kernel(const MaskTrainParams p) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ float red[NT / 32][MAX_PRED];
  uint4* wsm = reinterpret_cast<uint4*>(smem);                          // W1, W2, W3
  float* vec = reinterpret_cast<float*>(smem + S_W);                    // b1, b2, b3
  float* nb = reinterpret_cast<float*>(smem + S_W + S_VEC);            // [P][mu, sigma][HP]
  float* gacc = nb + p.P * 2 * HP;                                      // [P][d mu, d sigma][HP]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, q = lane & 3;
  const int H = p.H, W = p.W, HW = H * W;
  {
    const uint4* src = reinterpret_cast<const uint4*>(p.weights + M_W1);
    for (int i = tid; i < (int)(S_W / 16); i += NT) wsm[i] = __ldg(src + i);
    const float* vs = reinterpret_cast<const float*>(p.weights + M_VEC);
    for (int i = tid; i < M_NVEC; i += NT) vec[i] = __ldg(vs + i);
  }
  const bool want_pg = p.gpred != nullptr;
  if (want_pg)
    for (int i = tid; i < p.P * 2 * HP; i += NT) gacc[i] = 0.0f;
  const int* shw = reinterpret_cast<const int*>(p.weights + M_HDR);
  const int sh_w1 = __ldg(shw + 0), sh_w2 = __ldg(shw + 1), sh_w3 = __ldg(shw + 2);
  const uint4* w3 = wsm + 2 * M_LAYER / 16;
  const float* b3 = vec + 2 * HID;
  const float dw3 = pow2(-sh_w3);
  const int per_img = p.tiles_x * p.tiles_y;

  for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
    const int b = tile / per_img, t = tile - b * per_img, ty = t / p.tiles_x;
    const int y0 = ty * TY, x0 = (t - ty * p.tiles_x) * TX, y = y0 + warp;

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
    // the hidden maps the weight gradients read
    auto save_hidden = [&](int l) {
      if (!p.saved) return;
      float* hp = p.saved + ((size_t)l * p.B + b) * HID * HW + (size_t)(va ? y * W + xa : 0) + (size_t)(2 * q) * HW;
      store_rows(hp, acc, HW, va, vb);
      __syncwarp();
    };
    save_hidden(0);
    hidden_layer(acc, wsm, vec, sh_w1, lane);
    save_hidden(1);
    hidden_layer(acc, wsm + M_LAYER / 16, vec + HID, sh_w2, lane);
    save_hidden(2);
    uint32_t ah[HID / 16][4], al[HID / 16][4];
    int sh0, sh1;
    split_rows(acc, ah, al, sh0, sh1);
    const float d0 = pow2(-sh0), d1 = pow2(-sh1);
    __syncthreads();                                   // the neighbourhood is staged

    float nll[MAX_PRED];
#pragma unroll
    for (int pp = 0; pp < MAX_PRED; ++pp) nll[pp] = 0.0f;
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
      // lg[i][2r+e] becomes the gradient of the loss with respect to that logit
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int xl = g + 8 * r, x = x0 + xl;
        const bool v = r == 0 ? va : vb;
        const size_t o = ((size_t)b * H * K_UP + (size_t)y * K_UP + ky) * (size_t)(W * K_UP) + (size_t)x * K_UP + kx;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float w[9], dl[9];
#pragma unroll
          for (int i = 0; i < 9; ++i) { w[i] = lg[i][2 * r + e]; dl[i] = 0.0f; }
          if (v && __ldg(p.gtm + o + e)) {
            const float gt = __ldg(p.gt + o + e);
#pragma unroll
            for (int pp = 0; pp < MAX_PRED; ++pp) {
              if (pp >= p.P) break;
              const float* np = nb + pp * 2 * HP;
              auto tap = [&](int i, float& a, float& c) {
                const int yy = y + i / 3 - 1, xx = x + i % 3 - 1;
                const int hp = (warp + i / 3) * HX + xl + i % 3;
                a = np[hp];
                c = np[HP + hp];
                return yy >= 0 && yy < H && xx >= 0 && xx < W;
              };
              float mu, sg;
              if (pp == 0) convex_gaussian(w, tap, mu, sg);
              else convex_combine(w, tap, mu, sg);
              const float var = fmaxf(sg * sg, 1e-10f), d = mu - gt;
              nll[pp] += (d * d) / (2.0f * var) + 0.5f * logf(var);
              const float s = DEV_SCALE ? __ldg(p.scale_dev + pp) : p.scale[pp];
              const float g_mu = s * d / var;
              // var[var < 1e-10] = 1e-10 (losses.py:45) cuts the gradient to sigma where it clamps
              const float g_sg = (sg * sg < 1e-10f) ? 0.0f : s * (1.0f / sg - (d * d) / (var * sg));
              float tt[9];
#pragma unroll
              for (int i = 0; i < 9; ++i) {
                float a, c;
                tt[i] = 0.0f;
                if (tap(i, a, c)) {
                  tt[i] = __fmaf_rn(g_sg, c, g_mu * a);
                  if (want_pg) {
                    const int hp = (warp + i / 3) * HX + xl + i % 3;
                    atomicAdd(gacc + pp * 2 * HP + hp, g_mu * w[i]);
                    atomicAdd(gacc + pp * 2 * HP + HP + hp, g_sg * w[i]);
                  }
                }
              }
              float dot = 0.0f;
#pragma unroll
              for (int i = 0; i < 9; ++i) dot = __fmaf_rn(w[i], tt[i], dot);
#pragma unroll
              for (int i = 0; i < 9; ++i) dl[i] = __fadd_rn(dl[i], w[i] * (tt[i] - dot));
            }
          }
#pragma unroll
          for (int i = 0; i < 9; ++i) lg[i][2 * r + e] = dl[i];
        }
      }
      if (p.dlog) {
#pragma unroll
        for (int i = 0; i < 9; ++i) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int ch = (2 * i + h) * 8 + 2 * q + e;
            float* c = ch < HID ? p.dlog + ((size_t)b * HID + ch) * HW
                                : p.dlog + (size_t)p.B * HID * HW + ((size_t)b * NOUT_HI + ch - HID) * HW;
            if (va) c[y * W + xa] = lg[i][e];
            if (vb) c[y * W + xb] = lg[i][2 + e];
          }
        }
      }
    }

    // ---- the tile's loss partial of every prediction, in a fixed order ----
#pragma unroll
    for (int pp = 0; pp < MAX_PRED; ++pp) {
      if (pp >= p.P) break;
      float s = nll[pp];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
      if (lane == 0) red[warp][pp] = s;
    }
    __syncthreads();                                   // partials and neighbourhood gradients complete
    if (tid < p.P) {
      float s = 0.0f;
#pragma unroll
      for (int w = 0; w < NT / 32; ++w) s = __fadd_rn(s, red[w][tid]);
      p.partial[(size_t)tile * p.P + tid] = s;
    }
    if (want_pg) {
      for (int i = tid; i < p.P * 2 * HP; i += NT) {
        const int pp = i / (2 * HP), j = i - pp * 2 * HP, c = j / HP, hp = j - c * HP;
        const int yy = y0 - 1 + hp / HX, xx = x0 - 1 + hp % HX;
        const float v = gacc[i];
        gacc[i] = 0.0f;
        if (v != 0.0f && yy >= 0 && yy < H && xx >= 0 && xx < W)
          atomicAdd(p.gpred + ((size_t)pp * p.B + b) * 2 * HW + (size_t)c * HW + yy * W + xx, v);
      }
    }
  }
}

struct MaskBwdParams {
  int B, HW, gpi, ngroups, depth;            // gpi: 16-pixel groups per image; depth: layers of the chain (1..3)
  const float* __restrict__ saved;           // the training forward's h0, h1, h2, d_logits
  const unsigned char* __restrict__ weights; // training pack: header ...
  const unsigned char* __restrict__ wt;      // ... and its tail, W3^T, W2^T, W1^T
  const float* __restrict__ gscale;          // upstream gradient of the loss
  float* __restrict__ dh;                    // d_h2, d_h1 (B,128,H,W)
  float* __restrict__ grad_pre0;             // (B,128,H,W) when depth == 3
};

// Per warp 16 consecutive pixels of one image (rows g and g+8 of the MMA): d_h2 = (W3^T d_logits) [h2 > 0] with 9 K
// steps, d_h1 = (W2^T d_h2) [h1 > 0], grad_pre0 = (W1^T d_h1) [h0 > 0] times the upstream gradient, all on the tensor
// cores.  Pixels past the image carry zeros.
__global__ void __launch_bounds__(NT, 1) mask_bwd_chain_kernel(const MaskBwdParams p) {
  extern __shared__ __align__(16) unsigned char smem[];
  uint4* wt = reinterpret_cast<uint4*>(smem);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, q = lane & 3;
  {
    const uint4* src = reinterpret_cast<const uint4*>(p.wt);
    for (int i = tid; i < (int)(S_WT / 16); i += NT) wt[i] = __ldg(src + i);
  }
  __syncthreads();
  const int* shw = reinterpret_cast<const int*>(p.weights + M_HDR);
  const int sh_w1 = __ldg(shw + 0), sh_w2 = __ldg(shw + 1), sh_w3 = __ldg(shw + 2);
  const float gs = __ldg(p.gscale);
  const int HW = p.HW;
  const size_t plane = (size_t)p.B * HID * HW;
  const float* h0s = p.saved;
  const float* h1s = p.saved + plane;
  const float* h2s = p.saved + 2 * plane;
  const float* dlo = p.saved + 3 * plane;
  const float* dhi = p.saved + 4 * plane;
  float* dh2 = p.dh;
  float* dh1 = p.dh + plane;

  for (int base = blockIdx.x * (NT / 32); base < p.ngroups; base += gridDim.x * (NT / 32)) {
    const int gi = base + warp;
    if (gi >= p.ngroups) break;
    const int b = gi / p.gpi, hw0 = (gi - b * p.gpi) * 16;
    const int pa = hw0 + g, pb = hw0 + g + 8;
    const bool va = pa < HW, vb = pb < HW;
    const size_t off = ((size_t)b * HID + 2 * q) * HW + (va ? pa : 0);
    float acc[NTILE][4];
    {
      float dl[NOUT / 8][4];
      const int hw = opaque(HW);
#pragma unroll
      for (int nt = 0; nt < NOUT / 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int ch = nt * 8 + 2 * q + e;
          const float* c = nt < NTILE ? dlo + ((size_t)b * HID + ch) * hw : dhi + ((size_t)b * NOUT_HI + ch - HID) * hw;
          dl[nt][e] = va ? __ldg(c + pa) : 0.0f;
          dl[nt][2 + e] = vb ? __ldg(c + pb) : 0.0f;
        }
      }
      grad_layer(dl, acc, wt, sh_w3, lane);
    }
    relu_mask(acc, h2s + off, HW, va, vb);
    store_rows(dh2 + off, acc, HW, va, vb);
#pragma unroll 1
    for (int l = 1; l < p.depth; ++l) {
      grad_layer(acc, acc, wt + (M_LAYER3T + (l - 1) * M_LAYER) / 16, l == 1 ? sh_w2 : sh_w1, lane);
      relu_mask(acc, (l == 1 ? h1s : h0s) + off, HW, va, vb);
      if (l == 2) {
#pragma unroll
        for (int nt = 0; nt < NTILE; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[nt][e] = __fmul_rn(acc[nt][e], gs);
      }
      store_rows((l == 1 ? dh1 : p.grad_pre0) + off, acc, HW, va, vb);
    }
  }
}

// out[i] = in[i] * upstream gradient for up to 16 (in, out, n) triples, one per blockIdx.y
struct ScaleList {
  const float* in[16];
  float* out[16];
  int n[16];
};
__global__ void __launch_bounds__(256) scale_grads_kernel(const ScaleList l, const float* __restrict__ gscale) {
  const int j = blockIdx.y;
  const float s = __ldg(gscale);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < l.n[j]; i += gridDim.x * blockDim.x)
    l.out[j][i] = __fmul_rn(l.in[j][i], s);
}
}  // namespace

size_t mask_train_weights_bytes() { return M_BYTES + S_WT; }
int mask_train_partials(int B, int H, int W) { return B * ((H + TY - 1) / TY) * ((W + TX - 1) / TX); }
size_t mask_saved_bytes(int P, int B, int H, int W) { return (size_t)(3 * HID + NOUT + 2 * P) * B * H * W * 4; }
size_t mask_bwd_workspace_bytes(int B, int H, int W) {
  return align256((size_t)2 * HID * B * H * W * 4) + head_wgrad_partial_floats(B, H, W, HID, HID) * 4;
}

// the inference pack, then W3^T (9 K steps), W2^T and W1^T under the same shifts
cudaError_t launch_mask_pack_train(const float* w1, const float* b1, const float* w2, const float* b2, const float* w3,
                                   const float* b3, void* dst, cudaStream_t st) {
  HeadPack p;
  add_pack<2>(p, w1, b1, w2, b2, w3, b3, 0);
  p.add_frags(w3, PACK_COLS, NOUT / 16, NTILE, 0, M_HDR + 8, M_BYTES);
  p.add_frags(w2, PACK_COLS, HID / 16, NTILE, 0, M_HDR + 4, M_BYTES + M_LAYER3T);
  p.add_frags(w1, PACK_COLS, HID / 16, NTILE, 0, M_HDR, M_BYTES + M_LAYER3T + M_LAYER);
  return launch_head_pack(p, dst, st);
}

cudaError_t launch_mask_train_fwd(int P, int B, int H, int W, const float* pre0, const void* weights,
                                  const float* const* pred, const float* gt, const unsigned char* gtm,
                                  const float* scale, bool scale_on_device, bool save_maps, bool pred_grad,
                                  float* partial, float* saved, cudaStream_t st, int* launches) {
  static std::once_flag flags[2][64];
  int dev = 0;
  const auto kern = scale_on_device ? mask_train_fwd_kernel<true> : mask_train_fwd_kernel<false>;
  cudaError_t e = set_smem_once(kern, flags[scale_on_device], (int)smem_train(MAX_PRED), false, &dev);
  if (e != cudaSuccess) return e;
  const size_t map = (size_t)B * H * W;
  MaskTrainParams p;
  p.B = B; p.H = H; p.W = W; p.P = P;
  p.tiles_x = (W + TX - 1) / TX;
  p.tiles_y = (H + TY - 1) / TY;
  p.ntiles = B * p.tiles_x * p.tiles_y;
  p.pre0 = pre0;
  p.weights = static_cast<const unsigned char*>(weights);
  p.gt = gt; p.gtm = gtm;
  for (int i = 0; i < MAX_PRED; ++i) {
    p.pred[i] = i < P ? pred[i] : nullptr;
    p.scale[i] = i < P && !scale_on_device ? scale[i] : 0.0f;
  }
  p.scale_dev = scale_on_device ? scale : nullptr;
  p.partial = partial;
  // saved: P x (B,2,H,W) prediction gradients, then h0, h1, h2 and d_logits (mask_saved_floats)
  float* maps = saved + (size_t)2 * P * map;
  p.saved = save_maps ? maps : nullptr;
  p.dlog = save_maps ? maps + 3 * HID * map : nullptr;
  p.gpred = pred_grad ? saved : nullptr;
  *launches = 1;
  if (pred_grad) {
    if ((e = cudaMemsetAsync(p.gpred, 0, (size_t)P * 2 * map * 4, st)) != cudaSuccess) return e;
    ++*launches;
  }
  kern<<<std::min(p.ntiles, sm_count(dev)), NT, smem_train(P), st>>>(p);   // persistent
  return cudaGetLastError();
}

// Launches: the chain kernel (when a gradient below the logits is asked for), per requested (weight, bias) pair of
// layers 2 and 1 one GEMM and its reductions, for layer 3 two of each (logit rows 0..127 and 128..143), and one
// kernel applying the upstream gradient to the weight, bias and prediction gradients.
cudaError_t launch_mask_bwd(int P, int B, int H, int W, const void* weights, const float* saved, const float* gscale,
                            void* workspace, float* grad_pre0, float* gw1, float* gb1, float* gw2, float* gb2,
                            float* gw3, float* gb3, float* const* grad_pred, cudaStream_t st, int* launches) {
  static std::once_flag flags[64];
  int dev = 0;
  cudaError_t e = set_smem_once(mask_bwd_chain_kernel, flags, (int)S_WT, false, &dev);
  if (e != cudaSuccess) return e;
  const int HW = H * W;
  const size_t map = (size_t)B * HW, plane = (size_t)HID * map;
  float* dh = static_cast<float*>(workspace);
  float* part = reinterpret_cast<float*>(static_cast<unsigned char*>(workspace) + align256(2 * plane * 4));
  const float* gp = saved;                                  // P x (B,2,H,W) prediction gradients, unit scale
  saved += (size_t)2 * P * map;                             // h0, h1, h2, d_logits
  const float* h0 = saved;
  const float* h1 = saved + plane;
  const float* h2 = saved + 2 * plane;
  const float* dlo = saved + 3 * plane;
  const float* dhi = saved + 4 * plane;
  int n = 0;
  const int depth = grad_pre0 ? 3 : (gw1 || gb1) ? 2 : (gw2 || gb2) ? 1 : 0;
  if (depth > 0) {
    MaskBwdParams p;
    p.B = B; p.HW = HW; p.gpi = (HW + 15) / 16; p.ngroups = B * p.gpi; p.depth = depth;
    p.saved = saved;
    p.weights = static_cast<const unsigned char*>(weights);
    p.wt = p.weights + M_BYTES;
    p.gscale = gscale; p.dh = dh; p.grad_pre0 = grad_pre0;
    const int ctas = std::min((p.ngroups + NT / 32 - 1) / (NT / 32), sm_count(dev));
    mask_bwd_chain_kernel<<<ctas, NT, S_WT, st>>>(p);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    ++n;
  }
  auto pair = [&](float* w, float* bias) { return (w ? 1 : 0) + (bias ? 1 : 0) + 1; };
  if (gw3 || gb3) {          // dW3 = sum d_logits h2^T, db3 = sum d_logits, in two row blocks
    if ((e = launch_head_wgrad(B, H, W, HID, dlo, HID, h2, part, gw3, gb3, st)) != cudaSuccess) return e;
    if ((e = launch_head_wgrad(B, H, W, NOUT_HI, dhi, HID, h2, part, gw3 ? gw3 + HID * HID : nullptr,
                               gb3 ? gb3 + HID : nullptr, st)) != cudaSuccess) return e;
    n += 2 * pair(gw3, gb3);
  }
  if (gw2 || gb2) {          // dW2 = sum d_h2 h1^T, db2 = sum d_h2
    if ((e = launch_head_wgrad(B, H, W, HID, dh, HID, h1, part, gw2, gb2, st)) != cudaSuccess) return e;
    n += pair(gw2, gb2);
  }
  if (gw1 || gb1) {          // dW1 = sum d_h1 h0^T, db1 = sum d_h1
    if ((e = launch_head_wgrad(B, H, W, HID, dh + plane, HID, h0, part, gw1, gb1, st)) != cudaSuccess) return e;
    n += pair(gw1, gb1);
  }
  ScaleList l;
  int cnt = 0, most = 0;
  auto add = [&](const float* in, float* out, int count) {
    if (!out) return;
    l.in[cnt] = in; l.out[cnt] = out; l.n[cnt] = count;
    most = std::max(most, count);
    ++cnt;
  };
  add(gw1, gw1, HID * HID); add(gb1, gb1, HID); add(gw2, gw2, HID * HID); add(gb2, gb2, HID);
  add(gw3, gw3, NOUT * HID); add(gb3, gb3, NOUT);
  for (int i = 0; i < P; ++i) add(gp + (size_t)i * 2 * map, grad_pred ? grad_pred[i] : nullptr, (int)(2 * map));
  if (cnt > 0) {
    scale_grads_kernel<<<dim3(std::min((most + 255) / 256, 4 * sm_count(dev)), cnt), 256, 0, st>>>(l, gscale);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    ++n;
  }
  *launches = n;
  return cudaSuccess;
}

}  // namespace magnet
