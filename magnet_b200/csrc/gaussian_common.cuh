// Device code of the Gaussian update shared by the stand-alone update kernel (aux_kernels.cu) and the fused G-Net
// head (gnet_head.cu), so both produce the same bits from the same G-Net output; and D-Net's variance activation,
// shared by the fused D-Net heads (dnet_head.cu, mask_head.cu) and the D-Net loss (aux_kernels.cu).
#pragma once
#include <cmath>

namespace magnet {

// MAGNET.py:60,65-69: mu' = mu0 + mu1*sigma0 ; sigma' = (elu(sigma1) + 1 + 1e-10)*sigma0.
// torch's ELU evaluates exp(x) - 1 on the negative side (not expm1).
__device__ __forceinline__ void gaussian_update(float mu1, float s1, float mu0, float s0, float& mu, float& sg) {
  const float elu = s1 > 0.0f ? s1 : __fsub_rn(expf(s1), 1.0f);
  mu = __fadd_rn(mu0, __fmul_rn(mu1, s0));
  sg = __fmul_rn(__fadd_rn(__fadd_rn(elu, 1.0f), 1e-10f), s0);
}

// Its derivative w.r.t. the G-Net output (mu1, sigma1), shared by the stand-alone backward (aux_kernels.cu) and the
// fused head's backward (gnet_head.cu): d_mu1 = g_mu*sigma0 ; d_sigma1 = g_sigma*elu'(sigma1)*sigma0.
__device__ __forceinline__ void gaussian_update_bwd(float g_mu, float g_sg, float s1, float s0, float& d_mu1,
                                                    float& d_s1) {
  d_mu1 = __fmul_rn(g_mu, s0);
  const float delu = s1 > 0.0f ? 1.0f : expf(s1);
  d_s1 = __fmul_rn(__fmul_rn(g_sg, delu), s0);
}

// ... and w.r.t. the previous Gaussian (mu0, sigma0), for callers whose prev_gmm is not detached.
__device__ __forceinline__ void gaussian_update_bwd_prev(float g_mu, float g_sg, float mu1, float s1, float& d_mu0,
                                                         float& d_s0) {
  const float elu = s1 > 0.0f ? s1 : __fsub_rn(expf(s1), 1.0f);
  d_mu0 = g_mu;
  d_s0 = __fadd_rn(__fmul_rn(g_mu, mu1), __fmul_rn(g_sg, __fadd_rn(__fadd_rn(elu, 1.0f), 1e-10f)));
}

// D-Net's activation_G (models/DNET.py:56-60) on the raw variance channel, in torch's order: F.elu as ATen's CUDA kernel
// evaluates it (x <= 0 ? expm1(x) : x), then + 1.0 and + 1e-10 as two fp32 additions.  NaN stays NaN.
__device__ __forceinline__ float activation_g(float v) {
  const float e = v <= 0.0f ? expm1f(v) : v;
  return __fadd_rn(__fadd_rn(e, 1.0f), 1e-10f);
}

}  // namespace magnet
