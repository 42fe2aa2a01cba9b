// gemm_canon.cu -- y = fp16(x W^T + b) in the canonical accumulation order, any number of rows M.
//
// Replaces nn.Linear under fp16 autocast (cuBLAS GEMM/GEMV in the reference: SURVEY.md 2.2 G1/G6).
// One warp owns R weight rows x T activation rows.  The 32 lanes split K exactly as the canonical
// dot product prescribes (lane l owns k = 256 g + 8 l + j), so every lane streams 16-byte pieces of
// the weight and activation rows, keeps R*T fp32 partial sums in registers, and the partials are
// combined with the transposing butterfly (canon.cuh) -- 31 shuffles per 32 outputs.
// This is CUDA-core work on purpose: the result must be bit-identical for every M (batch
// invariance) and to the CPU oracle; DESIGN.md section 3 explains why the tensor cores cannot give that.
// SEG = 64 / 256: the segmented order of the decoder's out_proj (K = 1024) / fc2 (K = 4096) -- the order the
// persistent decode kernel produces with its split-K partition (decode_mega.cu): every 256-wide group is reduced on
// its own (seg 64: xor-4,2,1 inside a 64-element segment first, then the 4 segments as a tree; seg 256: the plain
// butterfly) and the 16 segment dots are added with a balanced binary tree in index order.
#include "canon.cuh"
#include "internal.h"

namespace ma {

constexpr int GEMM_WARPS = 4;

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

template <int R, int T, bool PIPE, int SEG>
__global__ void __launch_bounds__(GEMM_WARPS * 32)
    gemm_canon_kernel(const __half* __restrict__ W, const __half* __restrict__ bias, const __half* __restrict__ x,
                      int ldx, __half* __restrict__ y, int ldy, int M, int N, int K, int epi) {
  static_assert((R * T) % 32 == 0, "R*T must be a multiple of 32");
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * T;
  const int n0 = (blockIdx.y * GEMM_WARPS + warp) * R;
  if (n0 >= N) return;

  float acc[R * T];
#pragma unroll
  for (int i = 0; i < R * T; i++) acc[i] = 0.0f;

  // element offsets of this lane's slice of each row (clamped: out-of-range rows repeat the last row)
  long woff[R], xoff[T];
#pragma unroll
  for (int r = 0; r < R; r++) woff[r] = (long)min(n0 + r, N - 1) * K + 8 * lane;
#pragma unroll
  for (int t = 0; t < T; t++) xoff[t] = (long)min(m0 + t, M - 1) * ldx + 8 * lane;

  // Software pipeline over the 256-wide K groups: the raw 16-byte pieces of group g+1 are requested while group g
  // is multiplied (x right after its conversion, each weight row right after its own conversion), so a warp hides
  // its own load latency -- at small M there are fewer than two warps per scheduler to hide it otherwise.
  const int G = K >> 8;
  if constexpr (SEG != 0) {
    // segmented order: per group, partial dots from 0 -> transposing butterfly -> tree over the groups
    constexpr int NS = (R * T) / 32;
    float lv[NS][4], tot[NS];
#pragma unroll
    for (int s = 0; s < NS; s++) tot[s] = 0.0f;
#pragma unroll 1
    for (int g = 0; g < G; g++) {
      uint4 xc[T];
#pragma unroll
      for (int t = 0; t < T; t++) xc[t] = *reinterpret_cast<const uint4*>(x + xoff[t] + 256 * g);
#pragma unroll
      for (int r = 0; r < R; r++) {
        const uint4 wc = ldg_nc16(W + woff[r] + 256 * g);
#pragma unroll
        for (int t = 0; t < T; t++) acc[r * T + t] = dot8(wc, xc[t], 0.0f);
      }
#pragma unroll
      for (int s = 0; s < NS; s++) {
        const float v = transpose_reduce32o<SEG == 64 ? 1 : 0>(acc + 32 * s, lane);
        // seg 64: the transposing butterfly already added the 4 segments of the group as a tree (levels 1-2 of the
        // 16-leaf tree); the 4 group values are levels 3-4.  seg 256: one leaf per group
        tot[s] = (SEG == 64) ? tree4_push(v, g, lv[s]) : tree16_push(v, g, lv[s]);
      }
    }
#pragma unroll
    for (int s = 0; s < NS; s++) {
      const int a = 32 * s + transpose_owner<SEG == 64 ? 1 : 0>(lane);
      const int r = a / T, t = a % T;
      const int n = n0 + r, m = m0 + t;
      if (n < N && m < M) {
        float bf = bias ? __half2float(bias[n]) : 0.0f;
        __half h = __float2half_rn(fadd(tot[s], bf));
        if (epi == MA_EPI_RELU) {
          if (__half2float(h) < 0.0f) h = __float2half_rn(0.0f);
        } else if (epi == MA_EPI_GELU) {
          h = __float2half_rn(gelu_erf(__half2float(h)));
        }
        y[(long)m * ldy + n] = h;
      }
    }
    return;
  }
  if constexpr (PIPE) {
    uint4 xr[T], wr[R];
#pragma unroll
    for (int t = 0; t < T; t++) xr[t] = *reinterpret_cast<const uint4*>(x + xoff[t]);
#pragma unroll
    for (int r = 0; r < R; r++) wr[r] = ldg_nc16(W + woff[r]);
    for (int g = 0; g < G; g++) {
      const int gn = 256 * min(g + 1, G - 1);   // the last group re-requests itself (no branch, no out-of-range read)
      float xf[T][8];
#pragma unroll
      for (int t = 0; t < T; t++) {
        unpack8(xr[t], xf[t]);
        xr[t] = *reinterpret_cast<const uint4*>(x + xoff[t] + gn);
      }
#pragma unroll
      for (int r = 0; r < R; r++) {
        float wf[8];
        unpack8(wr[r], wf);
        wr[r] = ldg_nc16(W + woff[r] + gn);
#pragma unroll
        for (int t = 0; t < T; t++) {
          float a = acc[r * T + t];
#pragma unroll
          for (int j = 0; j < 8; j++) a = ffma(wf[j], xf[t][j], a);
          acc[r * T + t] = a;
        }
      }
    }
  } else {
    for (int g = 0; g < G; g++) {
      float xf[T][8];
#pragma unroll
      for (int t = 0; t < T; t++) {
        uint4 u = *reinterpret_cast<const uint4*>(x + xoff[t] + 256 * g);
        unpack8(u, xf[t]);
      }
#pragma unroll
      for (int r = 0; r < R; r++) {
        uint4 u = ldg_nc16(W + woff[r] + 256 * g);
        float wf[8];
        unpack8(u, wf);
#pragma unroll
        for (int t = 0; t < T; t++) {
          float a = acc[r * T + t];
#pragma unroll
          for (int j = 0; j < 8; j++) a = ffma(wf[j], xf[t][j], a);
          acc[r * T + t] = a;
        }
      }
    }
  }

  // accumulator index a = r*T + t ; after the transposing butterfly lane l holds accumulator 32*s + l
#pragma unroll
  for (int s = 0; s < (R * T) / 32; s++) {
    float v = transpose_reduce32(acc + 32 * s, lane);
    const int a = 32 * s + lane;
    const int r = a / T, t = a % T;
    const int n = n0 + r, m = m0 + t;
    if (n < N && m < M) {
      float bf = bias ? __half2float(bias[n]) : 0.0f;
      __half h = __float2half_rn(fadd(v, bf));
      if (epi == MA_EPI_RELU) {
        if (__half2float(h) < 0.0f) h = __float2half_rn(0.0f);
      } else if (epi == MA_EPI_GELU) {
        h = __float2half_rn(gelu_erf(__half2float(h)));
      }
      y[(long)m * ldy + n] = h;
    }
  }
}

template <int SEG>
static void launch_seg(const __half* W, const __half* bias, const __half* x, int ldx, __half* y, int ldy, int M, int N,
                       int K, int epi, cudaStream_t st) {
  if (M <= 4) {
    constexpr int R = 8, T = 4;
    dim3 grid((M + T - 1) / T, (N + GEMM_WARPS * R - 1) / (GEMM_WARPS * R));
    gemm_canon_kernel<R, T, true, SEG><<<grid, GEMM_WARPS * 32, 0, st>>>(W, bias, x, ldx, y, ldy, M, N, K, epi);
  } else {
    constexpr int R = 8, T = 8;
    dim3 grid((M + T - 1) / T, (N + GEMM_WARPS * R - 1) / (GEMM_WARPS * R));
    gemm_canon_kernel<R, T, true, SEG><<<grid, GEMM_WARPS * 32, 0, st>>>(W, bias, x, ldx, y, ldy, M, N, K, epi);
  }
}

int launch_linear(const __half* W, const __half* bias, const __half* x, int ldx, __half* y, int ldy, int M, int N,
                  int K, int epi_flags, cudaStream_t st) {
  if (M <= 0 || N <= 0) return 0;
  const int epi = epi_flags & 0xf, seg = (epi_flags & MA_LIN_SEG64) ? 64 : (epi_flags & MA_LIN_SEG256) ? 256 : 0;
  if (seg && K != 16 * seg) {
    set_error("ma_linear_f16: segmented order %d needs K = %d, got %d", seg, 16 * seg, K);
    return 1;
  }
  if (K <= 0 || (K & 255)) {
    set_error("ma_linear_f16: K=%d is not a positive multiple of 256", K);
    return 1;
  }
  if ((ldx & 7) || ((uintptr_t)x & 15) || ((uintptr_t)W & 15)) {
    set_error("ma_linear_f16: x/W must be 16-byte aligned and ldx a multiple of 8");
    return 1;
  }
  // PIPE (254 registers, 2 CTAs/SM) for grids of a few waves at most (decode steps); the 3-CTA/SM plain loop for
  // prefill sizes
  const bool pipe = M <= 512;
  if (seg == 64) {
    launch_seg<64>(W, bias, x, ldx, y, ldy, M, N, K, epi, st);
  } else if (seg == 256) {
    launch_seg<256>(W, bias, x, ldx, y, ldy, M, N, K, epi, st);
  } else if (M <= 4) {
    constexpr int R = 8, T = 4;
    dim3 grid((M + T - 1) / T, (N + GEMM_WARPS * R - 1) / (GEMM_WARPS * R));
    gemm_canon_kernel<R, T, true, 0><<<grid, GEMM_WARPS * 32, 0, st>>>(W, bias, x, ldx, y, ldy, M, N, K, epi);
  } else {
    constexpr int R = 8, T = 8;
    dim3 grid((M + T - 1) / T, (N + GEMM_WARPS * R - 1) / (GEMM_WARPS * R));
    if (pipe) gemm_canon_kernel<R, T, true, 0><<<grid, GEMM_WARPS * 32, 0, st>>>(W, bias, x, ldx, y, ldy, M, N, K, epi);
    else gemm_canon_kernel<R, T, false, 0><<<grid, GEMM_WARPS * 32, 0, st>>>(W, bias, x, ldx, y, ldy, M, N, K, epi);
  }
  count_launch();
  return check_launch("gemm_canon_kernel") ? 0 : 1;
}

}  // namespace ma
