// The SPLIT16 weight pack of the fused heads (DESIGN §3.16): the scales, then every B fragment and fp32 vector of a
// HeadPack (head_common.cuh) in one kernel each.
#include <algorithm>

#include "head_common.cuh"

namespace magnet {

namespace {
// CTA s writes the shift of scale entry s: largest finite |w| mapped into [2^14, 2^15).
__global__ void __launch_bounds__(1024) head_scale_kernel(const __grid_constant__ HeadPack p,
                                                          unsigned char* __restrict__ dst) {
  const PackScale& s = p.scale[blockIdx.x];
  unsigned m = 0u;
  for (int i = threadIdx.x; i < s.n; i += blockDim.x) {
    const unsigned u = __float_as_uint(s.w[i]) & 0x7fffffffu;
    m = max(m, u >= 0x7f800000u ? 0u : u);
  }
  m = __reduce_max_sync(0xffffffffu, m);
  __shared__ unsigned red[32];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) m = max(m, red[i]);
    m = max(m, red[0]);
    *reinterpret_cast<int*>(dst + s.shift_off) = split16_shift(m);
  }
}

// Thread i writes fragment i of the concatenated segments and, below the vector count, vector element i.
__global__ void __launch_bounds__(256) head_pack_kernel(const __grid_constant__ HeadPack p,
                                                        unsigned char* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < p.vec_total) {
    int v = 0;
    while (v + 1 < p.nvec && i >= p.vec[v + 1].first) ++v;
    const PackVec& s = p.vec[v];
    reinterpret_cast<float*>(dst + s.dst_off)[i - s.first] = s.src[i - s.first];
  }
  if (i >= p.frag_total) return;
  int g = 0;
  while (g + 1 < p.nfrag && i >= p.frag[g + 1].first) ++g;
  const PackFrags& s = p.frag[g];
  const int f = i - s.first;
  const int lane = f & 31, nt = (f >> 5) % s.n_tiles, step = (f >> 5) / s.n_tiles;
  const int n = nt * 8 + (lane >> 2);
  const float sc = pow2(*reinterpret_cast<const int*>(dst + s.shift_off));
  float w[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int kk = 2 * (lane & 3) + (e & 1) + (e >> 1) * 8;           // 0,1 -> b0 ; 8,9 -> b1
    if (s.kind == PACK_CONV3X3) {
      const int cs = step / 9, tap = step - cs * 9, c = cs * 16 + kk;
      w[e] = c < s.D ? s.w[((size_t)n * s.D + c) * 9 + tap] : 0.0f;
    } else {
      const int k = step * 16 + kk;
      w[e] = s.kind == PACK_ROWS ? s.w[n * s.k_steps * 16 + k] : s.w[k * s.n_tiles * 8 + n];
    }
  }
  uint32_t h0, l0, h1, l1;
  split2(__fmul_rn(w[0], sc), __fmul_rn(w[1], sc), h0, l0);
  split2(__fmul_rn(w[2], sc), __fmul_rn(w[3], sc), h1, l1);
  reinterpret_cast<uint4*>(dst + s.dst_off)[f] = make_uint4(h0, h1, l0, l1);
}
}  // namespace

cudaError_t launch_head_pack(const HeadPack& p, void* dst, cudaStream_t st) {
  unsigned char* d = static_cast<unsigned char*>(dst);
  head_scale_kernel<<<p.nscale, 1024, 0, st>>>(p, d);
  const int n = std::max(p.frag_total, p.vec_total);
  head_pack_kernel<<<(n + 255) / 256, 256, 0, st>>>(p, d);
  return cudaGetLastError();
}

}  // namespace magnet
