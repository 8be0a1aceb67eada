// Device code of the Gaussian update shared by the stand-alone update kernel (aux_kernels.cu) and the fused G-Net
// head (gnet_head.cu), so both produce the same bits from the same G-Net output.
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

}  // namespace magnet
