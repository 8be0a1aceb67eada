// MAGNET_SRC_SPLIT16 / MAGNET_SRC_HALF16 producer (the buffers of the tensor-core kernels, packed_layout.cuh) and the
// absmax reduction it starts with.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "launchers.h"
#include "packed_layout.cuh"

namespace magnet {

// MAGNET_SRC_SPLIT16 producer: (N, 64, H, W) fp32 [+ (N, 2, H, W) Gaussians] -> header | fp16 planes (N, 2, H, W, 64):
//   hi = fp16(x*s), lo = fp16(x*s - hi) | table (N, H, W + 1, 4), entry x + 1 = (mu[x], sigma[x], mu[x+1], sigma[x+1]),
//   zeros outside the row
// MAGNET_SRC_HALF16 producer: (N, 64, H, W) fp16 / bf16 -> the same header and table around ONE plane fp16(x*s): the
// same kernels with T = __half / __nv_bfloat16 and PLANES = 1 (exact for every element above the threshold of DESIGN
// §3.7, so the plane equals the hi plane of the fp32 split of x.float(), whose lo plane is zero)

// bits of |x|, 0 for inf / NaN: the scale is chosen from the finite values, non-finite elements poison only their own
// products
__device__ __forceinline__ unsigned finite_abs_bits(float x) {
  const unsigned u = __float_as_uint(x) & 0x7fffffffu;
  return u >= 0x7f800000u ? 0u : u;
}
__device__ __forceinline__ float to_f32(float x) { return x; }
__device__ __forceinline__ float to_f32(__half x) { return __half2float(x); }
__device__ __forceinline__ float to_f32(__nv_bfloat16 x) { return __bfloat162float(x); }

template <class T> __device__ __forceinline__ unsigned finite_abs_bits16(uint4 r) {   // one 16-byte vector of T
  const T* h = reinterpret_cast<const T*>(&r);
  unsigned m = 0u;
#pragma unroll
  for (int e = 0; e < (int)(16 / sizeof(T)); ++e) m = max(m, finite_abs_bits(to_f32(h[e])));   // half types: exact in fp32
  return m;
}

// Reduction slots of absmax_kernel (work slots, common.cuh): the running maximum and the count of finished blocks of
// one launch, re-armed by the launch's last block.
__device__ unsigned g_absmax_max[WORK_SLOTS];
__device__ unsigned g_absmax_done[WORK_SLOTS];
static SlotTickets absmax_tickets;

// Largest finite |x| of x: n16 16-byte vectors of T, then ntail < 16 / sizeof(T) elements at `tail`.  Grid-stride over
// the vectors, four loads in flight per thread; one atomicMax per block into the slot, and the last block to finish
// writes the result: HEADER = the whole 256-byte Split16Header (absmax bits, scale and 1 / scale of the SPLIT16 rule,
// zeros) at `out`, otherwise the absmax bits alone.
template <class T, bool HEADER>
__global__ void __launch_bounds__(256) absmax_kernel(const T* __restrict__ x, size_t n16, const T* __restrict__ tail,
                                                     int ntail, unsigned* __restrict__ out, int slot) {
  constexpr int U = 4;
  __shared__ unsigned red[8];
  __shared__ bool last;
  const uint4* v = reinterpret_cast<const uint4*>(x);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned m = 0u;
  for (; i + (U - 1) * stride < n16; i += U * stride) {
    uint4 r[U];
#pragma unroll
    for (int u = 0; u < U; ++u) r[u] = __ldg(v + i + u * stride);
#pragma unroll
    for (int u = 0; u < U; ++u) m = max(m, finite_abs_bits16<T>(r[u]));
  }
  for (; i < n16; i += stride) m = max(m, finite_abs_bits16<T>(__ldg(v + i)));
  if (blockIdx.x == 0 && (int)threadIdx.x < ntail) m = max(m, finite_abs_bits(to_f32(tail[threadIdx.x])));
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) m = max(m, red[w]);
    if (m != 0u) atomicMax(&g_absmax_max[slot], m);
    last = slot_last_cta(g_absmax_done, slot);           // the maximum is visible before the block counts as done
  }
  __syncthreads();
  if (!last) return;
  if (threadIdx.x == 0) {                                  // every other block's maximum is in the slot: read and re-arm
    __threadfence();
    red[0] = atomicExch(&g_absmax_max[slot], 0u);
    g_absmax_done[slot] = 0u;
  }
  __syncthreads();
  m = red[0];
  if constexpr (HEADER) {
    static_assert(sizeof(Split16Header) == 12 && SPLIT16_HEADER == 256, "header words below");
    const int sh = split16_shift(m);
    const unsigned word = threadIdx.x == 0 ? (unsigned)(127 + sh) << 23     // scale
                        : threadIdx.x == 1 ? (unsigned)(127 - sh) << 23     // 1 / scale
                        : threadIdx.x == 2 ? m : 0u;                        // absmax bits, then zeros
    if (threadIdx.x < SPLIT16_HEADER / 4) out[threadIdx.x] = word;
  } else if (threadIdx.x == 0) {
    *out = m;
  }
}

// One CTA per SPX pixels of one image: channel planes are read coalesced along the pixels (16-byte loads of fp32, 8-byte
// loads of fp16 / bf16, when the image size allows; all of a thread's loads in flight together), transposed through
// shared memory (as fp32: exact), and the PLANES fp16 planes are written as contiguous 128-byte pixel rows.
// The vector loads of the map and the plane stores are evict-first in L2 (ld / st .cs): lines the kernel has re-read or
// written do not push out the ones absmax_kernel left in L2 that it has still to re-read.
template <class T> __device__ __forceinline__ float4 ldg_x4(const T* p) {   // 4 consecutive elements, 4 * sizeof(T) aligned
  if constexpr (std::is_same<T, float>::value) {
    return __ldcs(reinterpret_cast<const float4*>(p));
  } else {
    const uint2 r = __ldcs(reinterpret_cast<const uint2*>(p));
    const T* h = reinterpret_cast<const T*>(&r);
    return make_float4(to_f32(h[0]), to_f32(h[1]), to_f32(h[2]), to_f32(h[3]));
  }
}

template <class T, int PLANES, int SPX, bool VEC>
__global__ void __launch_bounds__(256) split16_repack_kernel(const T* __restrict__ src, const float* __restrict__ gmm,
                                                             unsigned char* __restrict__ dst, int N, int HW, int W) {
  constexpr int C = 64;
  __shared__ float t[SPX * (C + 1)];
  const float s = reinterpret_cast<const Split16Header*>(dst)->scale;   // written by absmax_kernel<T, true>
  // blocks are dispatched in blockIdx order: walk the images and pixel blocks from the end of the map back to its
  // start, the reverse of absmax_kernel's grid stride, so the first re-reads find the lines it touched last in L2 (and
  // image 0, which the first work items of the cost kernel read, is written last).  The kernel does not know the batch
  // size, so the other images of the first items (v * B) get no place of their own; in a step the reference repack
  // follows the source repack and replaces most of what the latter left in L2 anyway.
  const size_t img = gridDim.y - 1 - blockIdx.y;
  const int p0 = (gridDim.x - 1 - blockIdx.x) * SPX;
  if constexpr (VEC) {                                     // HW % 4 == 0, src 16-byte aligned
    static_assert(SPX == 128, "thread mapping below");
    constexpr int CPI = 8;                                 // channels per iteration
    // a warp reads 4 channel rows x 8 float4 (4 x 128 contiguous bytes); this way its transposed stores hit 32 banks
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int q4 = (warp & 3) * 8 + (lane & 7), c0 = (warp >> 2) * 4 + (lane >> 3);
    float4 v[C / CPI];
#pragma unroll
    for (int e = 0; e < C / CPI; ++e) {
      const int c = c0 + e * CPI, pix = p0 + 4 * q4;
      v[e] = pix < HW ? ldg_x4(src + (img * C + c) * HW + pix) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int e = 0; e < C / CPI; ++e) {
      const int c = c0 + e * CPI;
      t[(4 * q4 + 0) * (C + 1) + c] = v[e].x;
      t[(4 * q4 + 1) * (C + 1) + c] = v[e].y;
      t[(4 * q4 + 2) * (C + 1) + c] = v[e].z;
      t[(4 * q4 + 3) * (C + 1) + c] = v[e].w;
    }
  } else {
    const int xi = threadIdx.x % SPX, cy = threadIdx.x / SPX;
    for (int c = cy; c < C; c += 256 / SPX) t[xi * (C + 1) + c] = p0 + xi < HW ? to_f32(src[(img * C + c) * HW + p0 + xi]) : 0.0f;
  }
  __syncthreads();
  __half* planes = packed_planes(dst);
  float4* meta = packed_table(dst, (size_t)N, (size_t)HW, PLANES);
#pragma unroll
  for (int itw = 0; itw < SPX * 8 / 256; ++itw) {
    const int item = itw * 256 + threadIdx.x;
    const int pl = item >> 3, q = item & 7;                // pixel of the group, 8-channel chunk
    if (p0 + pl < HW) {
      __align__(16) __half hi[8], lo[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float v = t[pl * (C + 1) + q * 8 + e] * s;
        hi[e] = __float2half_rn(v);
        if constexpr (PLANES == 2) lo[e] = __float2half_rn(v - __half2float(hi[e]));
      }
      const size_t o = (size_t)(p0 + pl) * 64 + q * 8;
      __stcs(reinterpret_cast<uint4*>(planes + (img * PLANES + 0) * (size_t)HW * 64 + o), *reinterpret_cast<const uint4*>(hi));
      if constexpr (PLANES == 2)
        __stcs(reinterpret_cast<uint4*>(planes + (img * 2 + 1) * (size_t)HW * 64 + o), *reinterpret_cast<const uint4*>(lo));
    }
  }
  if (threadIdx.x < SPX && p0 + threadIdx.x < HW) {       // my (mu, sigma): first half of entry x + 1, second half of entry x
    const int pix = p0 + threadIdx.x;
    const int y = pix / W, x = pix - y * W;
    float2 ms = make_float2(0.0f, 0.0f);
    if (gmm != nullptr) ms = make_float2(gmm[(img * 2 + 0) * HW + pix], gmm[(img * 2 + 1) * HW + pix]);
    float2* row = reinterpret_cast<float2*>(meta + (img * (HW / W) + y) * (size_t)(W + 1));
    row[2 * (x + 1)] = ms;
    row[2 * x + 1] = ms;
    if (x == 0) row[0] = make_float2(0.0f, 0.0f);          // entry 0 = (outside, pixel 0)
    if (x == W - 1) row[2 * W + 1] = make_float2(0.0f, 0.0f);   // entry W = (pixel W-1, outside)
  }
}

// T = float: MAGNET_SRC_SPLIT16 (two planes); T = __half / __nv_bfloat16: MAGNET_SRC_HALF16 (one plane)
template <class T>
static cudaError_t launch_repack_planes(const T* src, const float* gmm, void* dst, int N, int C, int H, int W,
                                       cudaStream_t st, int* launches) {
  constexpr int PLANES = std::is_same<T, float>::value ? 2 : 1;
  constexpr size_t VEC = 16 / sizeof(T);                   // elements per 16-byte load of the reduction
  if (C != 64) return cudaErrorInvalidValue;
  const int HW = H * W;
  const size_t n = (size_t)N * C * HW;
  const size_t n16 = n / VEC;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const int blocks = (int)std::min<size_t>((size_t)sm_count(dev) * 8, (n16 + 255) / 256 + 1);
  absmax_kernel<T, true><<<blocks, 256, 0, st>>>(src, n16, src + n16 * VEC, (int)(n - n16 * VEC),
                                                 static_cast<unsigned*>(dst), work_slot(absmax_tickets, st));
  dim3 block(256);
  if (HW % 4 == 0 && reinterpret_cast<uintptr_t>(src) % 16 == 0) {
    dim3 grid((HW + 127) / 128, N);
    split16_repack_kernel<T, PLANES, 128, true><<<grid, block, 0, st>>>(src, gmm, static_cast<unsigned char*>(dst), N, HW, W);
  } else {
    dim3 grid((HW + 31) / 32, N);
    split16_repack_kernel<T, PLANES, 32, false><<<grid, block, 0, st>>>(src, gmm, static_cast<unsigned char*>(dst), N, HW, W);
  }
  *launches = 2;
  return cudaGetLastError();
}

// *out = bits of the largest finite |x[i]|, i < n (x 16-byte aligned): one reduction kernel
cudaError_t launch_absmax_f32(const float* x, size_t n, unsigned* out, cudaStream_t st) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const size_t n16 = n / 4;
  const int blocks = (int)std::min<size_t>((size_t)sm_count(dev) * 8, (n16 + 255) / 256 + 1);
  absmax_kernel<float, false><<<blocks, 256, 0, st>>>(x, n16, x + n16 * 4, (int)(n - n16 * 4), out, work_slot(absmax_tickets, st));
  return cudaGetLastError();
}

cudaError_t launch_repack_split16(const float* src, const float* gmm, void* dst, int N, int C, int H, int W,
                                  cudaStream_t st, int* launches) {
  return launch_repack_planes(src, gmm, dst, N, C, H, W, st, launches);
}

// dtype: MAGNET_DTYPE_F16 or MAGNET_DTYPE_BF16 (checked by the caller)
cudaError_t launch_repack_half16(const void* src, int dtype, const float* gmm, void* dst, int N, int C, int H, int W,
                                 cudaStream_t st, int* launches) {
  if (dtype == MAGNET_DTYPE_F16)
    return launch_repack_planes(static_cast<const __half*>(src), gmm, dst, N, C, H, W, st, launches);
  return launch_repack_planes(static_cast<const __nv_bfloat16*>(src), gmm, dst, N, C, H, W, st, launches);
}

size_t split16_buffer_bytes(int N, int H, int W) { return split16_bytes((size_t)N, (size_t)H, (size_t)W); }
size_t half16_buffer_bytes(int N, int H, int W) { return half16_bytes((size_t)N, (size_t)H, (size_t)W); }

}  // namespace magnet
