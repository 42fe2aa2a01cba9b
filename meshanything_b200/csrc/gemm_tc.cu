// gemm_tc.cu -- y = act(x W^T + b) on the Hopper tensor cores: wgmma.mma_async with fp32 accumulators in registers,
// operands staged in shared memory by TMA (cp.async.bulk.tensor, 128-byte swizzle), mbarrier pipeline.
//
// Used for the dense contractions of the stages that are compared under a tolerance (encoder a1-a8, detokenizer
// a17-a18: SURVEY.md 2.2 G5/G6, ~200 GFLOP per shape).  The decoder keeps the canonical CUDA-core kernels: the
// tensor core sums each K=16 slab in a hardware-defined order that a CPU oracle cannot restate bit for bit
// (DESIGN.md section 3).
//
// One CTA = one 128x128 output tile, 288 threads:
//   warps 0-7  two consumer warpgroups: warpgroup g owns output rows m0 + 64g .. +63 and issues
//              4 x wgmma m64n128k16 per stage (one wgmma group kept in flight; the stage before it is released)
//   warp 8     TMA producer (one elected lane): A tile [128 rows x 64 halfs], B tile [128 x 64] per stage, 4 stages
// Both operands are K-major ([rows][K] row-major), so D = A * B^T needs no transpose.  TMA zero-fills rows beyond M.
#include "internal.h"
#include "tc_common.cuh"

namespace ma {

constexpr int TC_BM = 128, TC_BN = 128, TC_BK = 64, TC_STAGES = 4, TC_THREADS = 288, TC_CONSUMER_WARPS = 8;
constexpr uint32_t TC_STAGE_BYTES = (TC_BM + TC_BN) * TC_BK * 2;  // 32 KB

struct alignas(1024) TcSmem {
  __half a[TC_STAGES][TC_BM * TC_BK];
  __half b[TC_STAGES][TC_BN * TC_BK];
  uint64_t full[TC_STAGES], empty[TC_STAGES];
};

__device__ __forceinline__ float gelu_erf_tc(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

__global__ void __launch_bounds__(TC_THREADS, 1)
    gemm_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                   const __half* __restrict__ bias, __half* __restrict__ y, int ldy, int M, int N, int K, int epi) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  TcSmem& sm = *reinterpret_cast<TcSmem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.y * TC_BM, n0 = blockIdx.x * TC_BN;
  const int nk = K / TC_BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < TC_STAGES; s++) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.empty[s], TC_CONSUMER_WARPS);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == TC_CONSUMER_WARPS) {
    // ---------------- TMA producer
    if (elect_one()) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
      for (int kb = 0; kb < nk; kb++) {
        const int s = kb % TC_STAGES;
        const uint32_t ph = (kb / TC_STAGES) & 1;
        mbar_wait(&sm.empty[s], ph ^ 1);  // first pass: passes immediately (barrier is in phase 0)
        mbar_expect_tx(&sm.full[s], TC_STAGE_BYTES);
        tma_load_2d(sm.a[s], &map_a, kb * TC_BK, m0, &sm.full[s]);
        tma_load_2d(sm.b[s], &map_b, kb * TC_BK, n0, &sm.full[s]);
      }
    }
    return;
  }
  // ---------------- consumers: warpgroup g = rows 64g .. 64g+63 of the tile
  const int g = warp >> 2;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; i++) acc[i] = 0.0f;
  for (int kb = 0; kb < nk; kb++) {
    const int s = kb % TC_STAGES;
    mbar_wait(&sm.full[s], (kb / TC_STAGES) & 1);
    const uint64_t ad = gmma_desc(sm.a[s] + 64 * g * TC_BK), bd = gmma_desc(sm.b[s]);
    wgmma_reg_fence<64>(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < TC_BK / 16; k++)  // 32 bytes (16 halfs) further along K inside the 128-byte swizzle row
      wgmma_ss<TC_BN>(acc, ad + (uint64_t)(k * 2), bd + (uint64_t)(k * 2), (kb | k) ? 1u : 0u);
    wgmma_commit();
    wgmma_reg_fence<64>(acc);
    wgmma_wait<1>();                                        // the previous stage's wgmmas are complete
    if (kb > 0 && lane == 0) mbar_arrive(&sm.empty[(kb - 1) % TC_STAGES]);
  }
  wgmma_wait<0>();
  wgmma_reg_fence<64>(acc);
  // ---------------- epilogue straight from the accumulator registers
  const int r0 = m0 + 64 * g + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int m = r0 + 8 * h;
    if (m >= M) continue;
#pragma unroll
    for (int i = 0; i < TC_BN / 8; i++) {
      const int n = n0 + 8 * i + 2 * (lane & 3);
      __half out[2];
#pragma unroll
      for (int e = 0; e < 2; e++) {
        float v = acc[4 * i + 2 * h + e] + (bias ? __half2float(bias[n + e]) : 0.0f);
        __half hv = __float2half_rn(v);
        if (epi == MA_EPI_RELU) {
          if (__half2float(hv) < 0.0f) hv = __float2half_rn(0.0f);
        } else if (epi == MA_EPI_GELU) {
          hv = __float2half_rn(gelu_erf_tc(__half2float(hv)));
        }
        out[e] = hv;
      }
      *reinterpret_cast<__half2*>(y + (long)m * ldy + n) = __halves2half2(out[0], out[1]);
    }
  }
}

// ---- host side: tensor maps through the driver entry point (no link-time dependency on libcuda) ------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;

static int tc_init() {
  if (g_encode) return 0;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) {
    set_error("cuTensorMapEncodeTiled not available");
    cudaGetLastError();
    return 1;
  }
  g_encode = (EncodeTiledFn)fn;
  return 0;
}

int tc_make_map(CUtensorMap* map, const void* base, long rows, long cols, long ld, int box_rows, int box_cols) {
  if (tc_init()) return 1;
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  const cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d)", (int)r);
    return 1;
  }
  return 0;
}

bool linear_tc_supported(int M, int N, int K, int ldx, int ldy, const void* x, const void* W, const void* y) {
  return M >= 64 && (N % TC_BN) == 0 && (K % TC_BK) == 0 && (ldx % 8) == 0 && (ldy % 8) == 0 &&
         ((uintptr_t)x % 16) == 0 && ((uintptr_t)W % 16) == 0 && ((uintptr_t)y % 16) == 0;
}

int launch_linear_tc(const __half* W, const __half* bias, const __half* x, int ldx, __half* y, int ldy, int M, int N,
                     int K, int epi, cudaStream_t st) {
  static bool attr_done = false;
  if (!attr_done) {
    cudaFuncSetAttribute(gemm_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TcSmem) + 1024);
    attr_done = true;
  }
  CUtensorMap ma, mb;
  if (tc_make_map(&ma, x, M, K, ldx, TC_BM, TC_BK) || tc_make_map(&mb, W, N, K, K, TC_BN, TC_BK)) return 1;
  dim3 grid(N / TC_BN, (M + TC_BM - 1) / TC_BM);
  gemm_tc_kernel<<<grid, TC_THREADS, sizeof(TcSmem) + 1024, st>>>(ma, mb, bias, y, ldy, M, N, K, epi);
  count_launch();
  return check_launch("gemm_tc_kernel") ? 0 : 1;
}

}  // namespace ma
