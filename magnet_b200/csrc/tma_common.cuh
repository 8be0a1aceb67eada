// sm_90a primitives as inline PTX: mbarrier + TMA (cp.async.bulk[.tensor]) for cost_tma.cu / cost_mma.cu, and
// warpgroup MMA (wgmma.mma_async) for cost_mma.cu.
#pragma once
#include <cuda.h>   // CUtensorMap and its enums (types only — cuTensorMapEncodeTiled is resolved at run time)
#include <stdint.h>

namespace magnet {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t arrivals) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(arrivals) : "memory");
}
// make the barrier initialisation visible to the async proxy (TMA) before the first copy is issued
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// one arrival + the number of bytes the async copies of this phase will deliver
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(bar), "r"(parity) : "memory");
}

__device__ __forceinline__ void mbar_wait_or_trap(uint32_t bar, uint32_t parity) {
  // bounded spin: a protocol error must surface as a launch failure, not as a hung GPU
#pragma unroll 1
  for (int it = 0; it < (1 << 22); ++it) {
    uint32_t done;
    // the suspend-time hint lets the hardware park the warp instead of spinning on issue slots the other CTA needs
    asm volatile("{\n.reg .pred P1;\nmbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2, %3;\nselp.u32 %0, 1, 0, P1;\n}"
                 : "=r"(done) : "r"(bar), "r"(parity), "r"(20000u) : "memory");
    if (done) return;
  }
  __trap();
}

// TMA tiled load of one box of a rank-4 tensor map into shared memory (UTMALDG); out-of-range elements are
// zero-filled by the copy engine, coordinates are signed.
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* tmap, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
      ::"r"(dst), "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar) : "memory");
}

// rank-5 variant (cost_mma.cu: (channel, x, y, hi/lo plane, image))
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* tmap, uint32_t bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
      ::"r"(dst), "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "r"(bar) : "memory");
}

// order generic-proxy accesses of shared memory (ld/st.shared) before later async-proxy accesses (TMA writes, wgmma reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// 1-D bulk copy global -> shared (UBLKCP); bytes % 16 == 0, both addresses 16-byte aligned
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar) : "memory");
}

__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}

// ---- wgmma: one warpgroup (128 threads), fp16 operands from shared memory, fp32 accumulator in registers ----------
// Shared-memory matrix descriptor of a K-major operand in the canonical 128-byte-swizzle layout (what TMA's
// CU_TENSOR_MAP_SWIZZLE_128B writes): rows of 128 bytes (64 fp16 of K), 8-row atoms of 1024 bytes, `sbo` bytes between
// consecutive atoms.  Bit fields as cute::GMMA::GmmaDescriptor: start address >> 4 [0,14), leading byte offset >> 4
// [16,30) (unused for swizzled K-major, set to 1), stride byte offset >> 4 [32,46), base offset [49,52) = 0 (atoms are
// 1024-byte aligned), layout type SWIZZLE_128B = 1 [62,64).  A K step of 16 fp16 (32 bytes) inside the swizzle row is
// start address + 2.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t saddr, uint32_t sbo) {
  return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)1 << 16) | ((uint64_t)((sbo >> 4) & 0x3FFFu) << 32) |
         ((uint64_t)1 << 62);
}
// orders this warpgroup's register / shared-memory accesses before the wgmma instructions that follow
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, both K-major in shared memory.  Accumulator fragment of thread t of the
// warpgroup: d[4j + {0,1}] = D[16 (t/32) + (t%32)/4][8j + 2 (t%4) + {0,1}], d[4j + {2,3}] = the same columns 8 rows down.
__device__ __forceinline__ void wgmma_m64n128k16_f16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}

// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T, both K-major: the narrow form of m64n128k16 (fragment as there, j < 8)
__device__ __forceinline__ void wgmma_m64n64k16_f16(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}

// D[64 x 64] += A[64 x 16] * B[16 x 64] with either operand K-major (TA / TB = 0) or MN-major (= 1, the transposed
// form: rows of the 128-byte-swizzle atom are K indices holding 64 contiguous M / N elements; the descriptor's stride
// byte offset is then the distance between consecutive 8-row K groups).  Accumulator fragment as m64n128k16, j < 8.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16_f16(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %34, %35;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "n"(TA), "n"(TB)
      : "memory");
}

}  // namespace magnet
