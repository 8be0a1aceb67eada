// D-Net's depth head after its 3x3 convolution in one kernel (DESIGN §3.15): per pixel the ReLU of the hoisted first
// layer, the 128 -> 128 layer on the fp16 tensor cores (SPLIT16, as the G-Net and mask heads, head_common.cuh), ReLU,
// and the 128 -> 2 layer on the CUDA cores (G-Net's output layer); optionally activation_G_magnet (DNET.py:62-67).
// The 128-channel hidden map never leaves the SM.  D-Net's mask head and upsampling run in mask_head.cu's kernel with
// one hidden layer; this file also describes the pack both kernels read.
#include <algorithm>
#include <mutex>

#include "head_common.cuh"
#include "launchers.h"

namespace magnet {

namespace {
constexpr int NT = 256;
constexpr int WARPS = NT / 32;
// 66 KiB of shared memory would let three CTAs share an SM, but the layer needs more than 128 registers per thread
// (at two CTAs per SM ptxas spills 180-224 bytes), so one CTA of 8 warps per SM
constexpr int CTAS_PER_SM = 1;

// D-Net pack: the depth head, then (k = 4) the mask head in mask_head.cu's one-hidden-layer layout.
constexpr size_t D_HDR = 0;                    // int32 shift of W1
constexpr size_t D_VEC = 256;                  // fp32 b1[128], W2[2][128], b2[2]
constexpr int D_NVEC = 3 * HID + 2;
constexpr size_t D_W1 = 4096;
constexpr size_t D_LAYER = (size_t)(HID / 16) * NTILE * 32 * 16;    // 64 KiB
constexpr size_t D_BYTES = D_W1 + D_LAYER;                          // offset of the mask-head part
constexpr size_t S_VEC = ((D_NVEC * 4 + 15) / 16) * 16;
constexpr size_t S_TOTAL = D_LAYER + S_VEC;
static_assert(D_VEC + D_NVEC * 4 <= D_W1, "vectors fit before W1");
static_assert(CTAS_PER_SM * S_TOTAL <= 227 * 1024, "CTAs per SM");

struct DnetParams {
  int B, HW, gpi, ngroups;                     // gpi: 16-pixel groups per image
  const float* __restrict__ pre;
  const unsigned char* __restrict__ weights;
  float* __restrict__ out;
};

// Per warp 16 consecutive pixels of one image (rows g and g+8 of the MMA); pixels past the image carry zeros and are
// not written.  SIGMA: out = [mu, sqrt(activation_G(v))] (mono_gmms of MAGNET.forward), else the raw [mu, v].
template <bool SIGMA>
__global__ void __launch_bounds__(NT, CTAS_PER_SM) dnet_depth_kernel(const DnetParams p) {
  extern __shared__ __align__(16) unsigned char smem[];
  uint4* wsm = reinterpret_cast<uint4*>(smem);                          // W1
  float* vec = reinterpret_cast<float*>(smem + D_LAYER);                // b1, W2, b2
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, q = lane & 3;
  {
    const uint4* src = reinterpret_cast<const uint4*>(p.weights + D_W1);
    for (int i = tid; i < (int)(D_LAYER / 16); i += NT) wsm[i] = __ldg(src + i);
    const float* vs = reinterpret_cast<const float*>(p.weights + D_VEC);
    for (int i = tid; i < D_NVEC; i += NT) vec[i] = __ldg(vs + i);
  }
  __syncthreads();
  const int sh_w1 = __ldg(reinterpret_cast<const int*>(p.weights + D_HDR));
  const int HW = p.HW;

  for (int base = blockIdx.x * WARPS; base < p.ngroups; base += gridDim.x * WARPS) {
    const int gi = base + warp;
    if (gi >= p.ngroups) break;
    const int b = gi / p.gpi, hw0 = (gi - b * p.gpi) * 16;
    const int pa = hw0 + g, pb = hw0 + g + 8;
    const bool va = pa < HW, vb = pb < HW;
    const float* ip = p.pre + (size_t)b * HID * HW;
    float acc[NTILE][4];
#pragma unroll
    for (int nt = 0; nt < NTILE; ++nt) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const size_t n = (size_t)(nt * 8 + 2 * q + e) * HW;
        acc[nt][e] = va ? relu(__ldg(ip + n + pa)) : 0.0f;
        acc[nt][2 + e] = vb ? relu(__ldg(ip + n + pb)) : 0.0f;
      }
    }
    hidden_layer(acc, wsm, vec, sh_w1, lane);
    float r[4];                                          // (mu, v) of rows g and g+8
    out2_layer(acc, vec + HID, q, r);
    if (q < 2 && (q == 0 ? va : vb)) {                  // lane 0 of the quad writes pixel g, lane 1 pixel g+8
      const size_t o = (size_t)b * 2 * HW + (q == 0 ? pa : pb);
      const float mu = __fadd_rn(q == 0 ? r[0] : r[2], vec[3 * HID]);
      float v = __fadd_rn(q == 0 ? r[1] : r[3], vec[3 * HID + 1]);
      if constexpr (SIGMA) v = sqrtf(activation_g(v));
      p.out[o] = mu;
      p.out[o + HW] = v;
    }
  }
}

template <bool SIGMA>
cudaError_t launch_depth(int B, int H, int W, const float* pre, const void* weights, float* out, cudaStream_t st) {
  static std::once_flag flags[64];
  int dev = 0;
  cudaError_t e = set_smem_once(dnet_depth_kernel<SIGMA>, flags, (int)S_TOTAL, false, &dev);
  if (e != cudaSuccess) return e;
  DnetParams p;
  p.B = B; p.HW = H * W; p.gpi = (p.HW + 15) / 16; p.ngroups = B * p.gpi;
  p.pre = pre; p.weights = static_cast<const unsigned char*>(weights); p.out = out;
  const int ctas = std::min((p.ngroups + WARPS - 1) / WARPS, CTAS_PER_SM * sm_count(dev));   // persistent
  dnet_depth_kernel<SIGMA><<<ctas, NT, S_TOTAL, st>>>(p);
  return cudaGetLastError();
}
}  // namespace

// k = 0: the depth head only; k = 4: both heads.
size_t dnet_weights_bytes(bool with_mask) { return D_BYTES + (with_mask ? dnet_mask_weights_bytes() : 0); }

// DESIGN §3.16: the depth head's W1 shift, fragments and vectors b1, W2, b2; then the mask head's pack at D_BYTES.
cudaError_t launch_dnet_pack(const float* dw1, const float* db1, const float* dw2, const float* db2, const float* mw1,
                             const float* mb1, const float* mw3, const float* mb3, bool with_mask, void* dst,
                             cudaStream_t st) {
  HeadPack p;
  p.add_scale(dw1, HID * HID, D_HDR);
  p.add_frags(dw1, PACK_ROWS, HID / 16, NTILE, 0, D_HDR, D_W1);
  p.add_vec(db1, HID, D_VEC);
  p.add_vec(dw2, 2 * HID, D_VEC + HID * 4);
  p.add_vec(db2, 2, D_VEC + 3 * HID * 4);
  if (with_mask) add_dnet_mask_pack(p, mw1, mb1, mw3, mb3, D_BYTES);
  return launch_head_pack(p, dst, st);
}

cudaError_t launch_dnet_depth(int B, int H, int W, const float* pre_d, const void* weights, bool sigma, float* out,
                              cudaStream_t st) {
  return sigma ? launch_depth<true>(B, H, W, pre_d, weights, out, st)
               : launch_depth<false>(B, H, W, pre_d, weights, out, st);
}

cudaError_t launch_dnet_upsample_packed(int B, int H, int W, const float* pre_m, const void* weights, const float* raw,
                                        float* out, cudaStream_t st) {
  return launch_dnet_upsample(B, H, W, pre_m, static_cast<const unsigned char*>(weights) + D_BYTES, raw, out, st);
}

}  // namespace magnet
