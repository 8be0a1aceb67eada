// Layout of a MAGNET_SRC_SPLIT16 / MAGNET_SRC_HALF16 buffer of N images (H x W, 64 channels), and the tensor maps the
// tensor-core kernels read it through:
//   header (256 bytes: Split16Header, then zeros)
//   | fp16 planes (N, PLANES, H, W, 64): SPLIT16 hi = fp16(x*s), lo = fp16(x*s - hi); HALF16 the one plane fp16(x*s)
//   | (mu, sigma) table (N, H, W + 1, 4): entry x + 1 of a row = (mu, sigma)[x], (mu, sigma)[x + 1] with zeros outside
//     the row — both horizontal taps of a bilinear cell in ONE 16-byte read
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stddef.h>

#include "launchers.h"

namespace magnet {

struct Split16Header {
  float scale;       // s = 2^k
  float inv_scale;   // 2^-k
  unsigned absmax;   // bits of max |x|
};
constexpr size_t SPLIT16_HEADER = 256;

__host__ __device__ inline size_t split16_bytes(size_t N, size_t H, size_t W) {
  return SPLIT16_HEADER + N * H * W * 256 + N * H * (W + 1) * 16;
}
__host__ __device__ inline size_t half16_bytes(size_t N, size_t H, size_t W) {
  return SPLIT16_HEADER + N * H * W * 128 + N * H * (W + 1) * 16;
}

// the fp16 planes and the (mu, sigma) table of a buffer of N images of HW pixels with `planes` planes
__host__ __device__ inline __half* packed_planes(void* buf) {
  return reinterpret_cast<__half*>(static_cast<unsigned char*>(buf) + SPLIT16_HEADER);
}
__host__ __device__ inline float4* packed_table(void* buf, size_t N, size_t HW, int planes) {
  return reinterpret_cast<float4*>(static_cast<unsigned char*>(buf) + SPLIT16_HEADER + N * HW * 128 * planes);
}
__host__ __device__ inline const float4* packed_table(const void* buf, size_t N, size_t HW, int planes) {
  return packed_table(const_cast<void*>(buf), N, HW, planes);
}

// rank-5 map over the fp16 planes of `buf`: (64 channels, W, H, planes, N); box = 8 pixels of one row (window segment,
// box_rows 1) or an 8x8 tile (reference, box_rows 8), every plane; 128-byte swizzle = the canonical K-major wgmma
// layout (cost_f_bwd_mma.cu reads the same boxes as MN-major operands)
inline cudaError_t make_planes_map(CUtensorMap* tm, const void* buf, int N, int H, int W, int box_rows, int nplanes) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) return cudaErrorNotSupported;
  const cuuint64_t dims[5] = {64, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)nplanes, (cuuint64_t)N};
  const cuuint64_t strides[4] = {128, (cuuint64_t)W * 128, (cuuint64_t)H * W * 128, (cuuint64_t)H * W * 128 * nplanes};
  const cuuint32_t box[5] = {64u, 8u, (cuuint32_t)box_rows, (cuuint32_t)nplanes, 1u};
  const cuuint32_t estr[5] = {1u, 1u, 1u, 1u, 1u};
  const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, packed_planes(const_cast<void*>(buf)), dims, strides,
                         box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

// rank-4 map over the (mu, sigma) table of `buf`: (4 floats, W + 1, H, N), box = 8 entries of one row
inline cudaError_t make_meta_map(CUtensorMap* tm, const void* buf, int N, int H, int W, int nplanes) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) return cudaErrorNotSupported;
  const cuuint64_t dims[4] = {4, (cuuint64_t)W + 1, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t strides[3] = {16, ((cuuint64_t)W + 1) * 16, (cuuint64_t)H * (W + 1) * 16};
  const cuuint32_t box[4] = {4u, 8u, 1u, 1u};
  const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  const void* meta = packed_table(buf, (size_t)N, (size_t)H * W, nplanes);
  const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<void*>(meta), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

}  // namespace magnet
