// attention_tc.cu -- dense (non-causal) attention softmax(q K^T * scale) V on the Hopper tensor cores, for the
// stages compared under a tolerance: the Perceiver cross-attention (257 queries x 4096 keys x 12 heads,
// transformer_blocks.py:166-185), the 24 Michelangelo self-attention layers (:57-74) and the 6 BERT layers of the
// detokenizer (meshanything.py:50-80).  The decoder keeps the canonical CUDA-core attention (DESIGN.md section 3).
//
// One CTA = 128 queries of one (slot, head); loop over blocks of 128 keys (flash-attention recurrence).  Consumer
// warpgroup g (warps 4g .. 4g+3) owns query rows 64g .. 64g+63:
//   S = Q K_j^T          wgmma m64n128k16 x4 from shared memory (Q, K_j: K-major tiles [rows][64 halfs], TMA, 128-byte
//                        swizzle); S stays in registers (a thread holds 2 rows x 32 columns)
//   P = exp2((S - m) * scale * log2 e)  running max / sum per row over the 4 threads of a quad, P rounded to fp16
//                        and packed in registers in the A-operand layout of the next wgmma
//   O = O * alpha + P V_j  wgmma m64n64k16 x8 with A = P from registers, B = V_j^T from shared memory (two
//                        [64 d][64 keys] tiles; V is kept TRANSPOSED in global memory ([slot][head][64][Tpad]) so that
//                        it is K-major too)
// 288 threads: warps 0-7 the two consumer warpgroups, warp 8 TMA producer.  K/V^T double-buffered; mbarriers q_full,
// kv_full[2] (TMA transactions), kv_empty[2] (one arrival per consumer warp).
#include "internal.h"
#include "tc_common.cuh"

namespace ma {

constexpr int FA_BQ = 128, FA_BK = 128, FA_STAGES = 2, FA_THREADS = 288, FA_CONSUMER_WARPS = 8;
constexpr uint32_t FA_SPIN_LIMIT = 1u << 27;  // bounded polls (a few seconds): a protocol bug traps instead of hanging the GPU

struct alignas(1024) FaSmem {
  __half q[FA_BQ * 64];                   // 16 KB
  __half k[FA_STAGES][FA_BK * 64];        // 16 KB each
  __half vt[FA_STAGES][2][64 * 64];       // per stage: V^T for keys 0..63 and 64..127 of the block, 8 KB each
  uint64_t q_full, kv_full[FA_STAGES], kv_empty[FA_STAGES];
};

__device__ __forceinline__ void fa_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0;
  for (uint32_t spin = 0; spin < FA_SPIN_LIMIT; spin++) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (done) return;
  }
  __trap();
}

__device__ __forceinline__ uint32_t pack_half2(__half lo, __half hi) {
  __half2 v = __halves2half2(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

struct FaArgs {
  __half* out;
  int ldo, H, rows_per_slot, nkeys;
  long T;       // key capacity per (slot, head) in the K tensor
  float sl2;    // scale * log2(e)
};

__global__ void __launch_bounds__(FA_THREADS, 1)
    attention_tc_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                        const __grid_constant__ CUtensorMap map_vt, FaArgs a) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  FaSmem& sm = *reinterpret_cast<FaSmem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x, hd = blockIdx.y, slot = blockIdx.z;
  const int row0 = slot * a.rows_per_slot + qt * FA_BQ;          // first query row of this tile (global row index)
  const int valid_rows = min(FA_BQ, a.rows_per_slot - qt * FA_BQ);
  const int nb = (a.nkeys + FA_BK - 1) / FA_BK;
  const long head = (long)slot * a.H + hd;

  if (threadIdx.x == 0) {
    mbar_init(&sm.q_full, 1);
    for (int s = 0; s < FA_STAGES; s++) {
      mbar_init(&sm.kv_full[s], 1);
      mbar_init(&sm.kv_empty[s], FA_CONSUMER_WARPS);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == FA_CONSUMER_WARPS) {
    // ---------------- TMA producer
    if (elect_one()) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&map_q) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&map_k) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&map_vt) : "memory");
      mbar_expect_tx(&sm.q_full, FA_BQ * 64 * 2);
      tma_load_2d(sm.q, &map_q, 64 * hd, row0, &sm.q_full);
      for (int j = 0; j < nb; j++) {
        const int s = j % FA_STAGES;
        const uint32_t ph = (j / FA_STAGES) & 1;
        fa_wait(&sm.kv_empty[s], ph ^ 1);
        mbar_expect_tx(&sm.kv_full[s], (FA_BK * 64 + 2 * 64 * 64) * 2);
        tma_load_2d(sm.k[s], &map_k, 0, (int)(head * a.T + (long)j * FA_BK), &sm.kv_full[s]);
        tma_load_2d(sm.vt[s][0], &map_vt, j * FA_BK, (int)(head * 64), &sm.kv_full[s]);
        tma_load_2d(sm.vt[s][1], &map_vt, j * FA_BK + 64, (int)(head * 64), &sm.kv_full[s]);
      }
    }
    return;
  }
  // ---------------- consumers: thread holds query rows rr and rr + 8 of the tile, key / d columns 8i + 2(lane%4) + e
  const int g = warp >> 2;
  const int rr = 64 * g + 16 * (warp & 3) + (lane >> 2);
  const uint64_t qd = gmma_desc(sm.q + 64 * g * 64);
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.0f, 0.0f};
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; i++) o[i] = 0.0f;
  fa_wait(&sm.q_full, 0);
  for (int j = 0; j < nb; j++) {
    const int s = j % FA_STAGES;
    const int nvalid = min(FA_BK, a.nkeys - j * FA_BK);
    fa_wait(&sm.kv_full[s], (j / FA_STAGES) & 1);
    float sc[64];
    const uint64_t kd = gmma_desc(sm.k[s]);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; k++) wgmma_ss<FA_BK>(sc, qd + (uint64_t)(k * 2), kd + (uint64_t)(k * 2), k ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence<64>(sc);

    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 16; i++)
#pragma unroll
      for (int e = 0; e < 2; e++)
        if (8 * i + 2 * (lane & 3) + e < nvalid)
#pragma unroll
          for (int h = 0; h < 2; h++) mx[h] = fmaxf(mx[h], sc[4 * i + 2 * h + e]);
    float alpha[2], m_new[2], psum[2] = {0.0f, 0.0f};
#pragma unroll
    for (int h = 0; h < 2; h++) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      m_new[h] = fmaxf(m_run[h], mx[h]);   // nvalid >= 1, so m_new is finite
      alpha[h] = (m_run[h] == -INFINITY) ? 0.0f : exp2f((m_run[h] - m_new[h]) * a.sl2);
    }
    // P in the A-operand layout of wgmma: chunk kk (keys 16kk .. 16kk+15), register q = accumulator pair 8kk + 2q
    uint32_t pa[8][4];
#pragma unroll
    for (int kk = 0; kk < 8; kk++)
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const int idx = 8 * kk + 2 * q, h = q & 1;
        const int c = 8 * (idx >> 2) + 2 * (lane & 3);
        __half p2[2];
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const float p = (c + e < nvalid) ? exp2f((sc[idx + e] - m_new[h]) * a.sl2) : 0.0f;
          p2[e] = __float2half_rn(p);
          psum[h] += __half2float(p2[e]);
        }
        pa[kk][q] = pack_half2(p2[0], p2[1]);
      }
#pragma unroll
    for (int h = 0; h < 2; h++) {
      psum[h] += __shfl_xor_sync(0xffffffffu, psum[h], 1);
      psum[h] += __shfl_xor_sync(0xffffffffu, psum[h], 2);
      l_run[h] = l_run[h] * alpha[h] + psum[h];
      m_run[h] = m_new[h];
    }
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
      for (int e = 0; e < 4; e++) o[4 * i + e] *= alpha[e >> 1];
    wgmma_reg_fence<32>(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; kk++) wgmma_rs64(o, pa[kk], gmma_desc(sm.vt[s][kk >> 2]) + (uint64_t)((kk & 3) * 2));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence<32>(o);
    if (lane == 0) mbar_arrive(&sm.kv_empty[s]);   // this warp is done with K_j / V_j
  }
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int r = rr + 8 * h;
    if (r < valid_rows) {
      const float inv = 1.0f / l_run[h];
      __half* dst = a.out + (long)(row0 + r) * a.ldo + 64 * hd + 2 * (lane & 3);
#pragma unroll
      for (int i = 0; i < 8; i++)
        *reinterpret_cast<__half2*>(dst + 8 * i) =
            __halves2half2(__float2half_rn(o[4 * i + 2 * h] * inv), __float2half_rn(o[4 * i + 2 * h + 1] * inv));
    }
  }
}

bool attention_tc_supported(int ldq, int ldo, long T, long Tpad, int nkeys, const void* q, const void* K, const void* Vt,
                            const void* out) {
  return nkeys >= 1 && nkeys <= T && Tpad >= ((nkeys + FA_BK - 1) / FA_BK) * FA_BK && (Tpad % 64) == 0 &&
         (ldq % 8) == 0 && (ldo % 8) == 0 && ((uintptr_t)q % 16) == 0 && ((uintptr_t)K % 16) == 0 &&
         ((uintptr_t)Vt % 16) == 0 && ((uintptr_t)out % 16) == 0;
}

// q [n_slots*rows_per_slot][ldq] (head h at columns 64h..), K [n_slots][H][T][64], Vt [n_slots][H][64][Tpad] (zero beyond
// nkeys), every query of a slot attends to the first nkeys keys of that slot; out [rows][ldo] (head h at 64h..).
int launch_attention_tc(const __half* q, int ldq, const __half* K, const __half* Vt, long T, long Tpad, int H,
                        int rows_per_slot, int n_slots, int nkeys, float scale, __half* out, int ldo,
                        cudaStream_t st) {
  if (n_slots <= 0 || rows_per_slot <= 0) return 0;
  if (!attention_tc_supported(ldq, ldo, T, Tpad, nkeys, q, K, Vt, out)) {
    set_error("attention_tc: unsupported shape/alignment (nkeys=%d T=%ld Tpad=%ld ldq=%d ldo=%d)", nkeys, T, Tpad, ldq,
              ldo);
    return 1;
  }
  static bool attr_done = false;
  if (!attr_done) {
    cudaFuncSetAttribute(attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FaSmem) + 1024);
    attr_done = true;
  }
  CUtensorMap mq, mk, mv;
  const long rows = (long)n_slots * rows_per_slot;
  if (tc_make_map(&mq, q, rows, (long)H * 64, ldq, FA_BQ, 64) ||
      tc_make_map(&mk, K, (long)n_slots * H * T, 64, 64, FA_BK, 64) ||
      tc_make_map(&mv, Vt, (long)n_slots * H * 64, Tpad, Tpad, 64, 64))
    return 1;
  FaArgs a;
  a.out = out; a.ldo = ldo; a.H = H; a.rows_per_slot = rows_per_slot; a.nkeys = nkeys; a.T = T;
  a.sl2 = scale * 1.4426950408889634f;
  dim3 grid((rows_per_slot + FA_BQ - 1) / FA_BQ, H, n_slots);
  attention_tc_kernel<<<grid, FA_THREADS, sizeof(FaSmem) + 1024, st>>>(mq, mk, mv, a);
  count_launch();
  return check_launch("attention_tc_kernel") ? 0 : 1;
}

// V^T for the kernel above: dst[((slot*H + h)*64 + d)*Tpad + t] = src[m*ld + col0 + h*head_stride + d] (t < n), 0 beyond;
// m = slot*n + t.  One CTA per (64-key block, head, slot).
__global__ void __launch_bounds__(256)
    scatter_heads_t_kernel(const __half* __restrict__ src, int ld, int col0, int head_stride, int H, int n, long Tpad,
                           __half* __restrict__ dst) {
  __shared__ __half tile[64][72];  // [key][d], padded
  const int kb = blockIdx.x, h = blockIdx.y, slot = blockIdx.z, tid = threadIdx.x;
#pragma unroll
  for (int it = 0; it < 2; it++) {
    const int idx = tid + 256 * it, key = idx >> 3, piece = idx & 7;
    const int t = kb * 64 + key;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (t < n) u = *reinterpret_cast<const uint4*>(src + ((long)slot * n + t) * ld + col0 + h * head_stride + 8 * piece);
    *reinterpret_cast<uint4*>(&tile[key][8 * piece]) = u;
  }
  __syncthreads();
#pragma unroll
  for (int it = 0; it < 2; it++) {
    const int idx = tid + 256 * it, d = idx >> 3, piece = idx & 7;
    __half v[8];
#pragma unroll
    for (int i = 0; i < 8; i++) v[i] = tile[8 * piece + i][d];
    *reinterpret_cast<uint4*>(dst + (((long)slot * H + h) * 64 + d) * Tpad + kb * 64 + 8 * piece) =
        *reinterpret_cast<const uint4*>(v);
  }
}

int launch_scatter_heads_t(const __half* src, int ld, int col0, int head_stride, int H, int n, long Tpad, int n_slots,
                           __half* dst, cudaStream_t st) {
  if (Tpad % 64) {
    set_error("scatter_heads_t: Tpad=%ld is not a multiple of 64", Tpad);
    return 1;
  }
  dim3 grid((unsigned)(Tpad / 64), H, n_slots);
  scatter_heads_t_kernel<<<grid, 256, 0, st>>>(src, ld, col0, head_stride, H, n, Tpad, dst);
  count_launch();
  return check_launch("scatter_heads_t_kernel") ? 0 : 1;
}

}  // namespace ma
