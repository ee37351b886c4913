// Hopper warpgroup MMA (wgmma.mma_async, sm_90a) wrappers used by the tensor-core GEMMs (gemm_oz.cu, gemm_tc32.cu).
// B comes from shared memory through a matrix descriptor, A from shared memory too or (wgmma_s8_ra) from registers; the accumulator fragment of an m64nN shape is held by
// the 128 threads of the warpgroup, N / 2 32-bit registers each: register i of thread t is element
//     row = 16 (t / 32) + (t % 32) / 4 + 8 ((i / 2) % 2),   col = 8 (i / 4) + 2 (t % 4) + (i % 2)
// so the fragment of columns [32 j, 32 j + 32) is registers [16 j, 16 j + 16): an m64n(32 k) accumulator is k m64n32
// accumulators side by side.  Also the tensor-map encoder both GEMMs build their TMA descriptors with.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace gpk {

// cuTensorMapEncodeTiled, looked up once through the runtime (the library does not link the driver API); nullptr if absent
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeTiledFn encode_tiled_fn() {
  static const EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess) return (EncodeTiledFn) nullptr;
    return (EncodeTiledFn)p;
  }();
  return fn;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory");
}

// K-major shared-memory matrix descriptor: start address >> 4 (bits 0-13), leading byte offset >> 4 (bits 16-29; unused by
// swizzled K-major layouts, 1), stride byte offset >> 4 = distance between 8-row groups (bits 32-45), swizzle mode (bits
// 62-63: 1 = 128 B, 2 = 64 B, 3 = 32 B).  The tile must start on a swizzle-pattern boundary (1024 B / 512 B); a K step
// inside the swizzled row is a plain byte offset added to the start address.
template <int SWIZZLE_BYTES>
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr) {
  static_assert(SWIZZLE_BYTES == 128 || SWIZZLE_BYTES == 64, "swizzle");
  constexpr uint64_t mode = SWIZZLE_BYTES == 128 ? 1 : 2;
  constexpr uint64_t sbo = (8 * SWIZZLE_BYTES) >> 4;
  return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | (1ull << 16) | (sbo << 32) | (mode << 62);
}

// D(64 x N, s32) (+)= A(64 x 32, s8, K-major) * B(N x 32, s8, K-major)^T; exact integer arithmetic
template <int N>
__device__ __forceinline__ void wgmma_s8(uint32_t* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate);
template <>
__device__ __forceinline__ void wgmma_s8<32>(uint32_t* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p;\n}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_s8<64>(uint32_t* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p;\n}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// Same with A from registers: the warpgroup's m64k32 s8 fragment, 4 registers per thread.  Warp w holds rows 16 w .. 16 w + 15;
// register j of lane l is the 4 bytes of row 16 w + l / 4 + 8 (j % 2), columns 4 (l % 4) + 16 (j / 2) .. + 3 (the layout
// ldmatrix.x4 produces).  The registers must stay untouched until a wgmma wait shows the MMA complete.
template <int N>
__device__ __forceinline__ void wgmma_s8_ra(uint32_t* d, const uint32_t* a, uint64_t bdesc, uint32_t accumulate);
template <>
__device__ __forceinline__ void wgmma_s8_ra<32>(uint32_t* d, const uint32_t* a, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p;\n}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_s8_ra<64>(uint32_t* d, const uint32_t* a, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p;\n}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t* r, uint32_t smem_addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_addr)
               : "memory");
}
// D(64 x 128, f32) (+)= A(64 x 8, tf32, K-major) * B(128 x 8, tf32, K-major)^T
__device__ __forceinline__ void wgmma_tf32_n128(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

}  // namespace gpk
