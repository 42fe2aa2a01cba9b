// gemm_ws.cu -- weight-streaming GEMM for FEW activation rows (M <= 128) on the Hopper tensor cores:
// y = act(x W^T + b) with the roles of the operands swapped ("swap-AB"): a 128-row block of the WEIGHT matrix is the
// M operand of wgmma (two warpgroups of 64 rows), the M <= 128 activation rows are its N operand (padded to
// 16 / 32 / 64 / 128), so a decode step of a batch of sequences streams every weight exactly once through TMA at full
// tile efficiency instead of spending fp32 FMAs on it.
//
// The decoder's matrices have only 8..65 row blocks, fewer than the 132 SMs of an H100, so the K dimension is split
// across CTAs as well (grid = row blocks x K slices ~ one CTA per SM).  Two ways to add the slices, both in slice
// order, so the result never depends on timing:
//   * cluster mode (default): the K slices of a row block are ONE thread-block cluster (2 / 4 / 8 CTAs).  Every CTA
//     parks its fp32 tile in its own shared memory (the drained pipeline stages), the cluster synchronises, and CTA r
//     finishes activation rows r, r + ks, ... by reading the ks tiles over distributed shared memory
//     (ld.shared::cluster.v4) -- no round trip through L2, no tickets, no serialised last CTA;
//   * ticket mode (MA_B200_WS_CLUSTER=0, ma_linear_ws_set_mode): fp32 partial tiles in an L2-resident scratch area and
//     the LAST CTA of a row block (atomic ticket) adds them and applies bias / activation / fp16 rounding.
//
// Used by the batched decode step and (with gemm_tc_kernel for the 257-row prefill passes) wherever the decoder runs
// with a logits TOLERANCE instead of bit-exact ids: sampling (BASELINE configs 3-5) or MA_GEN_TC.  The tensor core adds
// each K = 16 slab in a hardware-defined order, so these results agree with the canonical kernels to fp32 rounding,
// not bit for bit (DESIGN.md section 3).
//
// CTA = 288 threads: warps 0-7 two consumer warpgroups (warpgroup g: weight rows n0 + 64g .. +63, 4 x wgmma
// m64 n=MP k16 per stage, accumulator [64 weight rows x MP activation rows] in registers), warp 8 TMA producer
// (W tile [128 x 64], x tile [MP x 64] per stage, 6-8 stages).
#include <stdlib.h>

#include "internal.h"
#include "tc_common.cuh"

namespace ma {

constexpr int WS_BN = 128, WS_BK = 64, WS_THREADS = 288, WS_CONSUMER_WARPS = 8;
// pipeline depth: as many 16 KB weight tiles in flight as shared memory holds
template <int MP> struct WsStages { static constexpr int value = MP <= 64 ? 8 : 6; };

template <int MP>
struct alignas(1024) WsSmem {
  static constexpr int ST = WsStages<MP>::value;
  __half a[ST][WS_BN * WS_BK];
  __half b[ST][MP * WS_BK];
  uint64_t full[ST], empty[ST];
  int last;
};

__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// the 256 consumer threads only (the producer warp does not take part)
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
// 16 bytes from the shared memory of CTA `rank` of this cluster, at the same offset as `addr` in this CTA
__device__ __forceinline__ float4 ld_dsmem_f4(uint32_t addr, uint32_t rank) {
  uint32_t ra;
  float4 v;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(addr), "r"(rank));
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(ra) : "memory");
  return v;
}

__device__ __forceinline__ float gelu_erf_ws(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

__device__ __forceinline__ __half ws_epilogue(float v, const __half* bias, int n, int epi) {
  v += bias ? __half2float(bias[n]) : 0.0f;
  __half h = __float2half_rn(v);
  if (epi == MA_EPI_RELU) {
    if (__half2float(h) < 0.0f) h = __float2half_rn(0.0f);
  } else if (epi == MA_EPI_GELU) {
    h = __float2half_rn(gelu_erf_ws(__half2float(h)));
  }
  return h;
}

template <int MP>
__global__ void __launch_bounds__(WS_THREADS, 1)
    gemm_ws_kernel(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_x,
                   const __half* __restrict__ bias, __half* __restrict__ y, int ldy, int M, int N, int nkb_total, int epi,
                   float* __restrict__ part, unsigned* __restrict__ tickets, int npad, int cluster) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  WsSmem<MP>& sm = *reinterpret_cast<WsSmem<MP>*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr uint32_t STAGE_BYTES = (WS_BN + MP) * WS_BK * 2;
  constexpr int WS_STAGES = WsStages<MP>::value;
  constexpr int NACC = MP / 2;   // accumulator registers per thread of an m64 nMP tile
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * WS_BN;
  const int ks = gridDim.y, ky = blockIdx.y;
  const int kb0 = (int)(((long)nkb_total * ky) / ks), kb1 = (int)(((long)nkb_total * (ky + 1)) / ks);
  const int nk = kb1 - kb0;
  // fp32 tile red[m][128] parked in the drained pipeline stages once every wgmma that read them has completed
  float* red = reinterpret_cast<float*>(sm.a);

  if (threadIdx.x == 0) {
    for (int s = 0; s < WS_STAGES; s++) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.empty[s], WS_CONSUMER_WARPS);
    }
    mbar_fence_init();
  }
  __syncthreads();

  pdl_trigger();   // the next kernel may start its prologue (and, if it is a GEMM, its own weight tiles)
  if (warp == WS_CONSUMER_WARPS) {
    // ---------------- TMA producer: this CTA's K slice of the weight row block (+ the matching columns of x).
    // The weights do not depend on the previous kernel: the first ring of weight tiles goes out BEFORE the grid
    // dependency resolves (programmatic dependent launch), the activation tiles after it.
    if (elect_one()) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
      const int first = min(nk, WS_STAGES);
      for (int i = 0; i < first; i++) {
        mbar_expect_tx(&sm.full[i], STAGE_BYTES);
        tma_load_2d(sm.a[i], &map_w, (kb0 + i) * WS_BK, n0, &sm.full[i]);   // rows beyond N are zero-filled
      }
      pdl_wait();
      for (int i = 0; i < first; i++)
        tma_load_2d(sm.b[i], &map_x, (kb0 + i) * WS_BK, 0, &sm.full[i]);    // rows beyond M are zero-filled
      for (int i = first; i < nk; i++) {
        const int s = i % WS_STAGES;
        const uint32_t ph = (i / WS_STAGES) & 1;
        mbar_wait(&sm.empty[s], ph ^ 1);
        mbar_expect_tx(&sm.full[s], STAGE_BYTES);
        tma_load_2d(sm.a[s], &map_w, (kb0 + i) * WS_BK, n0, &sm.full[s]);
        tma_load_2d(sm.b[s], &map_x, (kb0 + i) * WS_BK, 0, &sm.full[s]);
      }
    }
  } else {
    // ---------------- consumers: D[64 weight rows][MP activation rows] += Wtile * xtile^T per warpgroup
    const int g = warp >> 2, t = threadIdx.x;
    float acc[NACC];
#pragma unroll
    for (int i = 0; i < NACC; i++) acc[i] = 0.0f;
    for (int i = 0; i < nk; i++) {
      const int s = i % WS_STAGES;
      mbar_wait(&sm.full[s], (i / WS_STAGES) & 1);
      const uint64_t ad = gmma_desc(sm.a[s] + 64 * g * WS_BK), bd = gmma_desc(sm.b[s]);
      wgmma_reg_fence<NACC>(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < WS_BK / 16; k++) wgmma_ss<MP>(acc, ad + (uint64_t)(k * 2), bd + (uint64_t)(k * 2), (i | k) ? 1u : 0u);
      wgmma_commit();
      wgmma_reg_fence<NACC>(acc);
      wgmma_wait<1>();
      if (i > 0 && lane == 0) mbar_arrive(&sm.empty[(i - 1) % WS_STAGES]);
    }
    wgmma_wait<0>();
    wgmma_reg_fence<NACC>(acc);
    consumers_sync();   // every wgmma of both warpgroups has read its last stage: the stages may be overwritten
    {
      const int et = 64 * g + 16 * (warp & 3) + (lane >> 2);   // weight row inside the tile (+8 for h = 1)
#pragma unroll
      for (int i = 0; i < MP / 8; i++)
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
          for (int e = 0; e < 2; e++) red[(8 * i + 2 * (lane & 3) + e) * WS_BN + et + 8 * h] = acc[4 * i + 2 * h + e];
    }
    consumers_sync();
    if (!cluster) {
      const int et = t & (WS_BN - 1), n = n0 + et;
      if (n < N) {
        for (int m = t >> 7; m < M; m += 2) {
          const float v = red[m * WS_BN + et];
          if (ks == 1) y[(long)m * ldy + n] = ws_epilogue(v, bias, n, epi);
          else part[((long)ky * M + m) * npad + n] = v;
        }
      }
    }
    if (ks > 1 && !cluster) {
      // last CTA of this row block adds the K slices in slice order (deterministic) and finishes the rows
      __threadfence();
      consumers_sync();
      if (t == 0) {
        const unsigned old = atomicAdd(&tickets[blockIdx.x], 1u);
        sm.last = (old == (unsigned)ks - 1u);
        if (sm.last) tickets[blockIdx.x] = 0u;   // ready for the next launch
      }
      consumers_sync();
      if (sm.last && t < 128) {
        // 128 threads = 32 column quads x 4 row groups; 4 rows x 4 K slices of float4 loads in flight per thread (one
        // load at a time would serialise M * ks L2 round trips).  Slices are added in slice order.
        __threadfence();
        const int et = t;
        const int nq = n0 + 4 * (et & 31), mg = et >> 5;
        for (int m = mg; m < M; m += 16) {
          float4 acc4[4];
#pragma unroll
          for (int u = 0; u < 4; u++) acc4[u] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
#pragma unroll 4
          for (int k = 0; k < ks; k++) {
#pragma unroll
            for (int u = 0; u < 4; u++) {
              const int mm = m + 4 * u;
              if (mm < M) {
                const float4 pv = __ldcg(reinterpret_cast<const float4*>(part + ((long)k * M + mm) * npad + nq));
                acc4[u].x += pv.x; acc4[u].y += pv.y; acc4[u].z += pv.z; acc4[u].w += pv.w;
              }
            }
          }
#pragma unroll
          for (int u = 0; u < 4; u++) {
            const int mm = m + 4 * u;
            if (mm < M) {
              const float v4[4] = {acc4[u].x, acc4[u].y, acc4[u].z, acc4[u].w};
#pragma unroll
              for (int i = 0; i < 4; i++)
                if (nq + i < N) y[(long)mm * ldy + nq + i] = ws_epilogue(v4[i], bias, nq + i, epi);
            }
          }
        }
      }
    }
  }
  if (cluster) {
    // K slices of this row block = the CTAs of this cluster.  Barrier 1: every tile is parked; barrier 2: every CTA is
    // done reading its peers' shared memory (no CTA may exit before that).
    __syncwarp();
    cluster_sync_all();
    if (warp < WS_CONSUMER_WARPS) {
      uint32_t rank;
      asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
      const int et = threadIdx.x;
      const int nq = 4 * (et & 31), mg = et >> 5;      // 32 column quads x 8 row groups
      const uint32_t red0 = smem_u32(sm.a);
      // CTA `rank` finishes activation rows rank, rank + ks, ...; its 8 row groups take every 8th of those
      for (int m = (int)rank + ks * mg; m < M; m += 8 * ks) {
        float4 acc = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        float4 pv[8];
#pragma unroll
        for (int k = 0; k < 8; k++)
          if (k < ks) pv[k] = ld_dsmem_f4(red0 + (uint32_t)((m * WS_BN + nq) * 4), (uint32_t)k);
#pragma unroll
        for (int k = 0; k < 8; k++)
          if (k < ks) { acc.x += pv[k].x; acc.y += pv[k].y; acc.z += pv[k].z; acc.w += pv[k].w; }   // slice order
        const float v4[4] = {acc.x, acc.y, acc.z, acc.w};
        const int n = n0 + nq;
        if (n + 3 < N && (ldy & 3) == 0) {
          __half2 h01 = __halves2half2(ws_epilogue(v4[0], bias, n, epi), ws_epilogue(v4[1], bias, n + 1, epi));
          __half2 h23 = __halves2half2(ws_epilogue(v4[2], bias, n + 2, epi), ws_epilogue(v4[3], bias, n + 3, epi));
          uint2 u;
          u.x = *reinterpret_cast<uint32_t*>(&h01);
          u.y = *reinterpret_cast<uint32_t*>(&h23);
          *reinterpret_cast<uint2*>(y + (long)m * ldy + n) = u;
        } else {
#pragma unroll
          for (int i = 0; i < 4; i++)
            if (n + i < N) y[(long)m * ldy + n + i] = ws_epilogue(v4[i], bias, n + i, epi);
        }
      }
    }
    __syncwarp();
    cluster_sync_all();
  }
}

size_t linear_ws_scratch_bytes() { return (size_t)16 << 20; }   // fp32 partial tiles of one GEMM (+ tickets at the end)
constexpr size_t WS_TICKETS = 256;

bool linear_ws_supported(int M, int N, int K, int ldx, const void* x, const void* W) {
  return M >= 1 && M <= 128 && N >= 1 && (K % WS_BK) == 0 && (ldx % 8) == 0 && ((uintptr_t)x % 16) == 0 &&
         ((uintptr_t)W % 16) == 0 && (N + WS_BN - 1) / WS_BN <= (int)WS_TICKETS;
}

template <int MP>
static int launch_ws(const CUtensorMap& mw, const CUtensorMap& mx, const __half* bias, __half* y, int ldy, int M, int N,
                     int nkb, int epi, float* part, unsigned* tickets, int npad, dim3 grid, int cluster, bool pdl,
                     cudaStream_t st) {
  const size_t smem = sizeof(WsSmem<MP>) + 1024;
  static bool attr_done = false;
  if (!attr_done) {
    cudaFuncSetAttribute(gemm_ws_kernel<MP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr_done = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(WS_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[2];
  int na = 0;
  if (cluster) {
    at[na].id = cudaLaunchAttributeClusterDimension;
    at[na].val.clusterDim.x = 1;
    at[na].val.clusterDim.y = grid.y;   // the K slices of a row block are one cluster
    at[na].val.clusterDim.z = 1;
    na++;
  }
  if (pdl) {
    at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[na].val.programmaticStreamSerializationAllowed = 1;
    na++;
  }
  cfg.attrs = at;
  cfg.numAttrs = na;
  cudaLaunchKernelEx(&cfg, gemm_ws_kernel<MP>, mw, mx, bias, y, ldy, M, N, nkb, epi, part, tickets, npad, cluster);
  count_launch();
  return check_launch("gemm_ws_kernel") ? 0 : 1;
}

static int g_ws_cluster = [] {
  const char* e = getenv("MA_B200_WS_CLUSTER");
  return (e && e[0] == '0') ? 0 : 1;
}();
void linear_ws_set_mode(int cluster) { g_ws_cluster = cluster ? 1 : 0; }
int linear_ws_mode() { return g_ws_cluster; }

// scratch: linear_ws_scratch_bytes() bytes, its last WS_TICKETS words zero on first use (they return to zero)
int launch_linear_ws(const __half* W, const __half* bias, const __half* x, int ldx, __half* y, int ldy, int M, int N,
                     int K, int epi, void* scratch, cudaStream_t st, bool pdl) {
  if (!linear_ws_supported(M, N, K, ldx, x, W)) {
    set_error("ma_linear_ws_f16: unsupported shape M=%d N=%d K=%d ldx=%d", M, N, K, ldx);
    return 1;
  }
  const int tiles = (N + WS_BN - 1) / WS_BN, nkb = K / WS_BK;
  const int npad = tiles * WS_BN;
  const size_t avail = linear_ws_scratch_bytes() - WS_TICKETS * sizeof(unsigned);
  int ks, cluster = 0;
  if (g_ws_cluster) {
    // cluster mode: the largest cluster of 8 / 4 / 2 K slices whose clusters are all resident at once.  On an H100
    // (132 SMs) cudaOccupancyMaxActiveClusters gives 15 clusters of 8, 30 of 4 and 66 of 2 for this kernel at every MP
    // (149-199 KB of shared memory, 1 CTA per SM): a cluster never straddles a GPC.
    ks = 1;
    if (tiles <= 15 && nkb >= 16) ks = 8;               // out_proj, fc2: 8 row blocks -> 64 CTAs
    else if (tiles <= 30 && nkb >= 8) ks = 4;           // qkv 24 -> 96
    else if (tiles <= 66 && nkb >= 4) ks = 2;           // fc1 32 -> 64, lm_head 65 -> 130
    cluster = ks > 1;
  } else {
    // ticket mode: K is split only for matrices with few row blocks (out_proj, fc2: 8): the last-CTA fix-up costs about
    // a microsecond per K slice, more than a deep pipeline gains on 16+ CTAs
    ks = tiles >= 16 ? 1 : 132 / tiles;
    if (ks > 4) ks = 4;
    if (ks > nkb) ks = nkb;
    if (ks < 1) ks = 1;
    while (ks > 1 && (size_t)ks * M * npad * sizeof(float) > avail) ks--;
  }
  float* part = reinterpret_cast<float*>(scratch);
  unsigned* tickets = reinterpret_cast<unsigned*>(reinterpret_cast<char*>(scratch) + avail);
  const int MP = M <= 16 ? 16 : M <= 32 ? 32 : M <= 64 ? 64 : 128;
  CUtensorMap mw, mx;
  if (tc_make_map(&mw, W, N, K, K, WS_BN, WS_BK) || tc_make_map(&mx, x, M, K, ldx, MP, WS_BK)) return 1;
  const dim3 grid(tiles, ks);
  switch (MP) {
    case 16: return launch_ws<16>(mw, mx, bias, y, ldy, M, N, nkb, epi, part, tickets, npad, grid, cluster, pdl, st);
    case 32: return launch_ws<32>(mw, mx, bias, y, ldy, M, N, nkb, epi, part, tickets, npad, grid, cluster, pdl, st);
    case 64: return launch_ws<64>(mw, mx, bias, y, ldy, M, N, nkb, epi, part, tickets, npad, grid, cluster, pdl, st);
    default: return launch_ws<128>(mw, mx, bias, y, ldy, M, N, nkb, epi, part, tickets, npad, grid, cluster, pdl, st);
  }
}

}  // namespace ma
