// Device code shared by the fused heads on the fp16 tensor cores: the G-Net head (gnet_head.cu, DESIGN §3.8) and the
// mask head with the learned upsampling (mask_head.cu, DESIGN §3.12).  SPLIT16 products on mma.sync m16n8k16 with fp32
// accumulation: x*s = hi + lo with a power-of-two s, three products hi*hi + hi*lo + lo*hi, exact descale.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "gaussian_common.cuh"        // activation_g

namespace magnet {

constexpr int HID = 128;                       // hidden channels
constexpr int NTILE = HID / 8;                 // n8 tiles of one layer's output

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

// The accumulator fragment of a 128-channel layer (already ReLU'd) as the A fragments of the next GEMM: per-row scale
// (largest value of the row; sh0 / sh1 for rows g and g+8), split into hi and lo.  The m16n8 C layout of n tiles 2k,
// 2k+1 is the m16k16 A layout of K step k.
__device__ __forceinline__ void split_rows(const float (&acc)[NTILE][4], uint32_t (&ah)[HID / 16][4],
                                           uint32_t (&al)[HID / 16][4], int& sh0, int& sh1) {
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
  sh0 = split16_shift(__float_as_uint(m0));
  sh1 = split16_shift(__float_as_uint(m1));
  const float s0 = pow2(sh0), s1 = pow2(sh1);
#pragma unroll
  for (int kk = 0; kk < HID / 16; ++kk) {
    split2(__fmul_rn(acc[2 * kk][0], s0), __fmul_rn(acc[2 * kk][1], s0), ah[kk][0], al[kk][0]);
    split2(__fmul_rn(acc[2 * kk][2], s1), __fmul_rn(acc[2 * kk][3], s1), ah[kk][1], al[kk][1]);
    split2(__fmul_rn(acc[2 * kk + 1][0], s0), __fmul_rn(acc[2 * kk + 1][1], s0), ah[kk][2], al[kk][2]);
    split2(__fmul_rn(acc[2 * kk + 1][2], s1), __fmul_rn(acc[2 * kk + 1][3], s1), ah[kk][3], al[kk][3]);
  }
}

// One 128 -> 128 layer on the accumulator fragment of the previous one (already ReLU'd): split_rows, three products
// against the resident weights, descale, bias, ReLU.  Rows g and g+8 of the warp's 16 pixels.
__device__ __forceinline__ void hidden_layer(float (&acc)[NTILE][4], const uint4* __restrict__ wsm,
                                             const float* __restrict__ bias, int shw, int lane) {
  uint32_t ah[HID / 16][4], al[HID / 16][4];
  int sh0, sh1;
  split_rows(acc, ah, al, sh0, sh1);
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

// The 128 -> 2 layer on the CUDA cores (G-Net's output layer, D-Net's depth head): w = [W(0, :), W(1, :)] fp32, 32
// sequential FMAs per lane, then the quad's two-step butterfly.  r = (out0, out1) of row g, then of row g+8, bias not
// yet added; every lane of the quad holds the sums.
__device__ __forceinline__ void out2_layer(const float (&acc)[NTILE][4], const float* __restrict__ w, int q,
                                           float (&r)[4]) {
  r[0] = r[1] = r[2] = r[3] = 0.0f;
#pragma unroll
  for (int nt = 0; nt < NTILE; ++nt) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int n = nt * 8 + 2 * q + e;
      const float wm = w[n], ws = w[HID + n];
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
}

// ---- training (DESIGN §3.10, §3.13) --------------------------------------------------------------------------------
// The accumulator fragment of rows g, g+8 (pixels x, x+8 of one image row) into a (128, H, W) map: p points at channel
// 2q of pixel x.  Pixel x+8 is only valid when x is.
// The channel stride goes through an opaque copy: otherwise the compiler keeps the 32 channel addresses of one call
// live for the next call, across a layer's MMAs, and spills.
__device__ __forceinline__ int opaque(int v) {
  int r;
  asm volatile("mov.b32 %0, %1;" : "=r"(r) : "r"(v));
  return r;
}
__device__ __forceinline__ void store_rows(float* __restrict__ p, const float (&acc)[NTILE][4], int HW, bool va, bool vb) {
  HW = opaque(HW);
#pragma unroll
  for (int nt = 0; nt < NTILE; ++nt) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float* c = p + (size_t)(nt * 8 + e) * HW;
      if (va) c[0] = acc[nt][e];
      if (vb) c[8] = acc[nt][2 + e];
    }
  }
}

// One layer of the backward chain on a gradient fragment of KT n8 tiles (any sign; KT even) into 128 channels: per-row
// scale from max |x|, split, three products against resident transposed weights of KT/2 K steps, descale.  `in` is
// read completely before `out` is written, so both may name one array.  The caller applies the ReLU mask.
template <int KT>
__device__ __forceinline__ void grad_layer(const float (&in)[KT][4], float (&out)[NTILE][4], const uint4* __restrict__ wsm,
                                           int shw, int lane) {
  float m0 = 0.0f, m1 = 0.0f;
#pragma unroll
  for (int nt = 0; nt < KT; ++nt) {
    m0 = fmaxf(m0, fmaxf(fabsf(in[nt][0]), fabsf(in[nt][1])));
    m1 = fmaxf(m1, fmaxf(fabsf(in[nt][2]), fabsf(in[nt][3])));
  }
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, o));
    m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, o));
  }
  const int sh0 = split16_shift(__float_as_uint(m0)), sh1 = split16_shift(__float_as_uint(m1));
  const float s0 = pow2(sh0), s1 = pow2(sh1);
  uint32_t ah[KT / 2][4], al[KT / 2][4];
#pragma unroll
  for (int kk = 0; kk < KT / 2; ++kk) {
    split2(__fmul_rn(in[2 * kk][0], s0), __fmul_rn(in[2 * kk][1], s0), ah[kk][0], al[kk][0]);
    split2(__fmul_rn(in[2 * kk][2], s1), __fmul_rn(in[2 * kk][3], s1), ah[kk][1], al[kk][1]);
    split2(__fmul_rn(in[2 * kk + 1][0], s0), __fmul_rn(in[2 * kk + 1][1], s0), ah[kk][2], al[kk][2]);
    split2(__fmul_rn(in[2 * kk + 1][2], s1), __fmul_rn(in[2 * kk + 1][3], s1), ah[kk][3], al[kk][3]);
  }
#pragma unroll
  for (int nt = 0; nt < NTILE; ++nt) out[nt][0] = out[nt][1] = out[nt][2] = out[nt][3] = 0.0f;
#pragma unroll
  for (int kk = 0; kk < KT / 2; ++kk) {
#pragma unroll
    for (int nt = 0; nt < NTILE; ++nt) mma3(out[nt], ah[kk], al[kk], wsm[(kk * NTILE + nt) * 32 + lane]);
  }
  const float dw = pow2(-shw), d0 = pow2(-sh0), d1 = pow2(-sh1);
#pragma unroll
  for (int nt = 0; nt < NTILE; ++nt) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      out[nt][e] = __fmul_rn(__fmul_rn(out[nt][e], d0), dw);
      out[nt][2 + e] = __fmul_rn(__fmul_rn(out[nt][2 + e], d1), dw);
    }
  }
}

// ReLU backward on the fragment, as torch's threshold_backward: zero where the saved activation is <= 0 (a NaN
// activation passes the gradient); h as store_rows addresses it
__device__ __forceinline__ void relu_mask(float (&acc)[NTILE][4], const float* __restrict__ h, int HW, bool va, bool vb) {
  HW = opaque(HW);
#pragma unroll
  for (int nt = 0; nt < NTILE; ++nt) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const float* c = h + (size_t)(nt * 8 + e) * HW;
      acc[nt][e] = va && !(__ldg(c) <= 0.0f) ? acc[nt][e] : 0.0f;
      acc[nt][2 + e] = vb && !(__ldg(c + 8) <= 0.0f) ? acc[nt][2 + e] : 0.0f;
    }
  }
}

// ---- the weight pack (DESIGN §3.16) --------------------------------------------------------------------------------
// A pack is described by where each piece goes, and launch_head_pack (head_pack.cu) writes it in two launches: one CTA
// per scale entry writes split16_shift(largest finite |w|) as an int32 at dst + shift_off; then one thread per 16-byte
// B fragment {hi b0, hi b1, lo b0, lo b1} (K step, n8 tile, lane: n = 8 tile + lane/4, k = 16 step + 2 (lane%4) +
// {0, 1, 8, 9}) of the fragment segments, scaled by the shift at dst + shift_off, and the fp32 vectors copied as they are.
enum PackKind {
  PACK_ROWS,      // W[n K + k]: a 1x1 layer (N, K)
  PACK_COLS,      // W[k N + n]: its transpose, for the backward chains
  PACK_CONV3X3,   // W0[(n D + c) 9 + tap], K step = 9 chunk + tap, c = 16 chunk + k % 16, zero for c >= D
};
struct PackScale { const float* w; int n; size_t shift_off; };
struct PackFrags { const float* w; PackKind kind; int k_steps, n_tiles, D; size_t shift_off, dst_off; int first; };
struct PackVec { const float* src; int n; size_t dst_off; int first; };

struct HeadPack {
  PackScale scale[3];
  PackFrags frag[6];
  PackVec vec[5];
  int nscale = 0, nfrag = 0, nvec = 0, frag_total = 0, vec_total = 0;   // first: index of the segment's first thread

  void add_scale(const float* w, int n, size_t shift_off) { scale[nscale++] = {w, n, shift_off}; }
  void add_frags(const float* w, PackKind kind, int k_steps, int n_tiles, int D, size_t shift_off, size_t dst_off) {
    frag[nfrag++] = {w, kind, k_steps, n_tiles, D, shift_off, dst_off, frag_total};
    frag_total += k_steps * n_tiles * 32;
  }
  void add_vec(const float* src, int n, size_t dst_off) {
    vec[nvec++] = {src, n, dst_off, vec_total};
    vec_total += n;
  }
};
cudaError_t launch_head_pack(const HeadPack& p, void* dst, cudaStream_t st);
// the mask-head part of D-Net's pack, at byte `base` of it
void add_dnet_mask_pack(HeadPack& p, const float* w1, const float* b1, const float* w3, const float* b3, size_t base);

}  // namespace magnet
