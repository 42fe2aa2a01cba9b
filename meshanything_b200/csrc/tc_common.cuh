// tc_common.cuh -- Hopper tensor-core building blocks (wgmma + TMA 2-D tensor maps) shared by gemm_tc.cu, gemm_ws.cu and
// attention_tc.cu.
//
// wgmma.mma_async is issued by a whole warpgroup (4 consecutive warps, the first one's index a multiple of 4) and keeps
// its fp32 accumulator in registers.  Accumulator layout of an m64nN tile: warp w of the warpgroup, lane l holds
//   d[4i + 0..1] = D[16w + l/4    ][8i + 2(l%4) + 0..1]
//   d[4i + 2..3] = D[16w + l/4 + 8][8i + 2(l%4) + 0..1]          i = 0 .. N/8 - 1.
#pragma once
#include <cuda.h>

#include "canon.cuh"

namespace ma {

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}

// shared-memory matrix descriptor: K-major tile, rows of 128 bytes, SWIZZLE_128B, 8-row groups 1024 bytes apart.
// The tile base must be 1024-byte aligned; +2 on the descriptor = 32 bytes (16 halfs) further along K.
__device__ __forceinline__ uint64_t gmma_desc(const void* smem_ptr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_u32(smem_ptr) & 0x3FFFF) >> 4);  // start address
  d |= (uint64_t)1 << 16;                                // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;                      // stride byte offset
  d |= (uint64_t)1 << 62;                                // SWIZZLE_128B
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// the accumulator registers must not be touched by the compiler while an asynchronous wgmma may still write them
template <int NR>
__device__ __forceinline__ void wgmma_reg_fence(float* d) {
#pragma unroll
  for (int i = 0; i < NR; i++) asm volatile("" : "+f"(d[i])::"memory");
}

#define MA_F4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define MA_F16(i) MA_F4(i), MA_F4(i + 4), MA_F4(i + 8), MA_F4(i + 12)

// D[64][N] (+)= A[64][16] * B[N][16]^T, fp16 in, fp32 accumulate; A and B K-major in shared memory.
// accum = 0 overwrites D.
template <int N>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t ad, uint64_t bd, uint32_t accum);

template <>
__device__ __forceinline__ void wgmma_ss<16>(float* d, uint64_t ad, uint64_t bd, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : MA_F4(0), MA_F4(4)
      : "l"(ad), "l"(bd), "r"(accum));
}
template <>
__device__ __forceinline__ void wgmma_ss<32>(float* d, uint64_t ad, uint64_t bd, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : MA_F16(0)
      : "l"(ad), "l"(bd), "r"(accum));
}
template <>
__device__ __forceinline__ void wgmma_ss<64>(float* d, uint64_t ad, uint64_t bd, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,"
      "%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : MA_F16(0), MA_F16(16)
      : "l"(ad), "l"(bd), "r"(accum));
}
template <>
__device__ __forceinline__ void wgmma_ss<128>(float* d, uint64_t ad, uint64_t bd, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,"
      "%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,"
      "%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : MA_F16(0), MA_F16(16), MA_F16(32), MA_F16(48)
      : "l"(ad), "l"(bd), "r"(accum));
}
// D[64][64] += A[64][16] * B[64][16]^T with A in registers (4 x 2 packed halfs per thread, the layout of 16 columns
// of an accumulator tile: a[0] = D-row l/4 cols 2(l%4).., a[1] = row +8, a[2] = cols +8, a[3] = row +8 cols +8)
__device__ __forceinline__ void wgmma_rs64(float* d, const uint32_t* a, uint64_t bd) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,"
      "%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, 0;\n\t}"
      : MA_F16(0), MA_F16(16)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bd));
}
#undef MA_F16
#undef MA_F4

// non-transaction arrive (count 1) on a CTA-local mbarrier
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// ---- host: tensor maps through the driver entry point (gemm_tc.cu) -------------------------------------------------
// 2-D fp16 tensor [rows][cols] with row pitch `ld` elements, box [box_rows][box_cols], 128-byte swizzle.
int tc_make_map(CUtensorMap* map, const void* base, long rows, long cols, long ld, int box_rows, int box_cols);

}  // namespace ma
