// canon.cuh -- device-side pieces of the canonical arithmetic (DESIGN.md section 3).
//
// Every floating-point operation whose result is part of the parity contract is spelled with an
// explicit round-to-nearest intrinsic (__fmaf_rn / __fmul_rn / __fadd_rn / __fsub_rn / __fdiv_rn /
// __fsqrt_rn) so that nvcc can neither contract a*b+c into an FMA nor split one.  The CPU oracle
// (oracle/decoder_oracle.c, built with -ffp-contract=off) performs the same operations in the same
// order with scalar loops over virtual lanes.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ma_canon_constants.h"

namespace ma {

__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float ffma(float a, float b, float c) { return __fmaf_rn(a, b, c); }

// exp(x) for x <= 0 (softmax arguments); see include/ma_canon_constants.h
__device__ __forceinline__ float ma_exp(float x) {
  if (x < MA_EXP_FLUSH) return 0.0f;
  float y = fmul(x, MA_LOG2E);
  float n = rintf(y);
  float f = fsub(y, n);
  float p = MA_EXP2_C6;
  p = ffma(p, f, MA_EXP2_C5);
  p = ffma(p, f, MA_EXP2_C4);
  p = ffma(p, f, MA_EXP2_C3);
  p = ffma(p, f, MA_EXP2_C2);
  p = ffma(p, f, MA_EXP2_C1);
  p = ffma(p, f, MA_EXP2_C0);
  int bits = __float_as_int(p) + (((int)n) << 23);
  return __int_as_float(bits);
}

// 8 fp16 values of a 16-byte load -> fp32 (exact)
__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; i++) {
    float2 t = __half22float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

// acc + sum_j w[j] * x[j], j = 0..7 sequentially (the canonical per-lane chain): fp16 -> fp32 is exact, so each
// product-and-add is one fp32 FMA with one rounding
__device__ __forceinline__ float dot8(const uint4& w, const uint4& x, float acc) {
  float wf[8], xf[8];
  unpack8(w, wf);
  unpack8(x, xf);
#pragma unroll
  for (int j = 0; j < 8; j++) acc = ffma(wf[j], xf[j], acc);
  return acc;
}
// o[j] = float(p) * float(v[j]) + o[j], j = 0..7 (the P.V step of the canonical attention: P already rounded to fp16)
__device__ __forceinline__ void pv8(__half p, const uint4& v, float* o) {
  const float pf = __half2float(p);
  float vf[8];
  unpack8(v, vf);
#pragma unroll
  for (int j = 0; j < 8; j++) o[j] = ffma(pf, vf[j], o[j]);
}

__device__ __forceinline__ uint4 ldg_nc16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

// xor-16,8,4,2,1 butterfly: every lane ends with the canonical sum of the 32 lane partials
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fadd(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Transposing butterfly: each lane holds 32 partials v[0..31] (one per output); on return lane l
// holds in v[0] the canonical (xor-16,8,4,2,1) sum over lanes of partial l.  31 shuffles.
__device__ __forceinline__ float transpose_reduce32(float* v, int lane) {
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) {
    const bool up = (lane & s) != 0;
#pragma unroll
    for (int i = 0; i < s; i++) {
      float mine = up ? v[i + s] : v[i];
      float other = up ? v[i] : v[i + s];
      float recv = __shfl_xor_sync(0xffffffffu, other, s);
      v[i] = fadd(mine, recv);
    }
  }
  return v[0];
}

// pairwise left-to-right tree over n (<= 8) warp sums held in shared memory
__device__ __forceinline__ float warp_tree(const float* s, int n) {
  float b[8];
#pragma unroll
  for (int i = 0; i < 8; i++) b[i] = (i < n) ? s[i] : 0.0f;
  if (n == 8) return fadd(fadd(fadd(b[0], b[1]), fadd(b[2], b[3])), fadd(fadd(b[4], b[5]), fadd(b[6], b[7])));
  if (n == 6) return fadd(fadd(fadd(b[0], b[1]), fadd(b[2], b[3])), fadd(b[4], b[5]));
  if (n == 4) return fadd(fadd(b[0], b[1]), fadd(b[2], b[3]));
  if (n == 2) return fadd(b[0], b[1]);
  // generic (n in {1,3,5,7}): level by level, odd element carried
  int m = n;
  while (m > 1) {
    int k = 0;
    for (int i = 0; i + 1 < m; i += 2) b[k++] = fadd(b[i], b[i + 1]);
    if (m & 1) b[k++] = b[m - 1];
    m = k;
  }
  return b[0];
}

// Canonical block sum over W = 4*blockDim.x values: thread t contributes (x0+x1)+(x2+x3) of its own
// four elements; warp butterfly; warp tree.  `red` = shared scratch of >= 8 floats.  All threads
// return the sum.  Contains two __syncthreads().
__device__ __forceinline__ float block_sum4(float x0, float x1, float x2, float x3, float* red) {
  float p = fadd(fadd(x0, x1), fadd(x2, x3));
  p = warp_sum(p);
  const int nw = blockDim.x >> 5;
  __syncthreads();  // protect `red` against a previous use
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = p;
  __syncthreads();
  return warp_tree(red, nw);
}

// LayerNorm of a row of W = 4*blockDim.x fp32 values, thread t owns elements 4t..4t+3; g / b = this thread's four
// gamma / beta values, loaded by the caller (a PDL kernel loads them before its grid dependency resolves).
__device__ __forceinline__ void layernorm4(float* x, const float4& g, const float4& b, float eps, int W, float* red) {
  const float inv = __fdiv_rn(1.0f, (float)W);
  float mean = fmul(block_sum4(x[0], x[1], x[2], x[3], red), inv);
  float d0 = fsub(x[0], mean), d1 = fsub(x[1], mean), d2 = fsub(x[2], mean), d3 = fsub(x[3], mean);
  float var = fmul(block_sum4(fmul(d0, d0), fmul(d1, d1), fmul(d2, d2), fmul(d3, d3), red), inv);
  float rstd = __fdiv_rn(1.0f, __fsqrt_rn(fadd(var, eps)));
  x[0] = ffma(fmul(d0, rstd), g.x, b.x);
  x[1] = ffma(fmul(d1, rstd), g.y, b.y);
  x[2] = ffma(fmul(d2, rstd), g.z, b.z);
  x[3] = ffma(fmul(d3, rstd), g.w, b.w);
}

// ---- mbarrier / bulk-copy (TMA 1-D) wrappers -------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// global -> shared bulk copy; bytes % 16 == 0, both addresses 16-byte aligned
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---- programmatic dependent launch -----------------------------------------------------------
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

}  // namespace ma
