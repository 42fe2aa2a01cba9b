// attention.cu -- chunked (split-KV) attention in the canonical order, one query row per z-block.
//
// Replaces flash_attn_func of OptFlashAttention2 (decode: q [B,1,16,64] vs the KV cache; prefill:
// causal 257x257) and the eager einsum/softmax/einsum attention of
// /root/reference/MeshAnything/miche/michelangelo/models/modules/transformer_blocks.py:57-74,166-185.
//
// grid = (chunks, heads, rows); a CTA owns MA_ATTN_CHUNK = 256 key positions of one (row, head):
//   * K and V rows of the chunk are contiguous in the cache ([slot][head][T][64] fp16), so one
//     elected thread pulls each with a single bulk async copy (TMA 1-D, cp.async.bulk) that lands on
//     an mbarrier -- 2 x 32 KB in flight per CTA with no register cost;
//   * 8 warps = 32 groups of 8 lanes; position r of the chunk belongs to group-lane r % 32; a group
//     reads one 128-byte row per step (16 B per lane, conflict-free), dot = 8 fmaf per lane + xor
//     4,2,1 butterfly;  pass 1 scores + chunk max, pass 2 exp / P (rounded to fp16 like flash-attn)
//     / PV;
//   * the chunk result (max, sum, o[64]) goes to a scratch slot; the last CTA of a (row, head) to
//     arrive (atomic counter) merges the chunks in ascending order and writes the fp16 output.
#include "canon.cuh"
#include "internal.h"

namespace ma {

constexpr int ATT_THREADS = 256;
constexpr int PART = 66;  // o[64], max, sum
constexpr int ATT_MERGE_BLOCK = 2 * MA_ATTN_CHUNK * HD * 2 / (PART * 4);  // chunk partials that fit over the K / V tiles

struct AttnSmem {
  __half k[MA_ATTN_CHUNK * HD];
  __half v[MA_ATTN_CHUNK * HD];
  float s[MA_ATTN_CHUNK];
  float red[8][65];
  float wmax[8];
  uint64_t bar[2];
  int last;
};

struct AttnArgs {
  const __half* q;
  int ldq;
  const __half* K;
  const __half* V;
  long T;
  int H;
  int rows_per_slot;
  const int* slots;
  const int* nkeys;
  float scale;
  __half* out;
  int ldo;
  float* part;
  int* counters;
  int max_chunks;
  int decode_prefetch;  // 1: rows [0, n-1) of the cache are older than the previous kernel (PDL prologue may load them)
};

__global__ void __launch_bounds__(ATT_THREADS) attention_kernel(AttnArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  AttnSmem& sm = *reinterpret_cast<AttnSmem*>(smem_raw);
  const int c = blockIdx.x, h = blockIdx.y, m = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, grp = lane >> 3, li = lane & 7;

  if (!a.decode_prefetch) pdl_wait();  // everything this kernel reads may come from the previous kernel
  // never more keys than this launch has chunks for: a frozen cache slot (continuous batching) keeps an old, possibly
  // larger position than the bucket the grid was sized from; its output is discarded anyway (ADVICE r01)
  const int n = min(a.nkeys[m], a.max_chunks * MA_ATTN_CHUNK);
  if (c * MA_ATTN_CHUNK >= n) return;
  const int len = min(MA_ATTN_CHUNK, n - c * MA_ATTN_CHUNK);
  const int nch = (n + MA_ATTN_CHUNK - 1) / MA_ATTN_CHUNK;
  const int slot = a.slots ? a.slots[m] : m / a.rows_per_slot;
  const long base = (((long)slot * a.H + h) * a.T + (long)c * MA_ATTN_CHUNK) * HD;

  // rows that may be fetched before the grid dependency resolves
  const int len_early = a.decode_prefetch ? max(0, min(len, (n - 1) - c * MA_ATTN_CHUNK)) : 0;
  if (tid == 0) {
    mbar_init(&sm.bar[0], 1);
    mbar_init(&sm.bar[1], 1);
    mbar_fence_init();
    if (len_early > 0) {
      mbar_expect_tx(&sm.bar[0], 2u * len_early * HD * 2);
      bulk_g2s(sm.k, a.K + base, len_early * HD * 2, &sm.bar[0]);
      bulk_g2s(sm.v, a.V + base, len_early * HD * 2, &sm.bar[0]);
    }
  }
  if (a.decode_prefetch) pdl_wait();
  pdl_trigger();
  if (tid == 0) {
    const int rest = len - len_early;
    if (rest > 0) {
      mbar_expect_tx(&sm.bar[1], 2u * rest * HD * 2);
      bulk_g2s(sm.k + len_early * HD, a.K + base + (long)len_early * HD, rest * HD * 2, &sm.bar[1]);
      bulk_g2s(sm.v + len_early * HD, a.V + base + (long)len_early * HD, rest * HD * 2, &sm.bar[1]);
    }
  }
  float qf[8];
  {
    uint4 u = *reinterpret_cast<const uint4*>(a.q + (long)m * a.ldq + h * HD + 8 * li);
    unpack8(u, qf);
  }
  __syncthreads();  // barrier inits visible to all waiters
  if (len_early > 0) mbar_wait(&sm.bar[0], 0);
  if (len - len_early > 0) mbar_wait(&sm.bar[1], 0);

  // ---- pass 1: scores and chunk max
  float lmax = -INFINITY;
#pragma unroll
  for (int rho = 0; rho < MA_ATTN_CHUNK / 32; rho++) {
    const int r = 32 * rho + 4 * warp + grp;
    const int rr = min(r, len - 1);
    uint4 u = *reinterpret_cast<const uint4*>(sm.k + rr * HD + 8 * li);
    float kf[8];
    unpack8(u, kf);
    float p = 0.0f;
#pragma unroll
    for (int j = 0; j < 8; j++) p = ffma(qf[j], kf[j], p);
    p = fadd(p, __shfl_xor_sync(0xffffffffu, p, 4));
    p = fadd(p, __shfl_xor_sync(0xffffffffu, p, 2));
    p = fadd(p, __shfl_xor_sync(0xffffffffu, p, 1));
    const float s = fmul(p, a.scale);
    if (r < len) {
      if (li == 0) sm.s[r] = s;
      lmax = fmaxf(lmax, s);
    }
  }
  lmax = warp_max(lmax);
  if (lane == 0) sm.wmax[warp] = lmax;
  __syncthreads();
  float cmax = sm.wmax[0];
#pragma unroll
  for (int w = 1; w < 8; w++) cmax = fmaxf(cmax, sm.wmax[w]);

  // ---- pass 2: p = exp(s - max), l += p, o += fp16(p) * v   (sequential over this group-lane's rounds)
  float l = 0.0f, o[8];
#pragma unroll
  for (int j = 0; j < 8; j++) o[j] = 0.0f;
#pragma unroll
  for (int rho = 0; rho < MA_ATTN_CHUNK / 32; rho++) {
    const int r = 32 * rho + 4 * warp + grp;
    if (r < len) {
      const float e = ma_exp(fsub(sm.s[r], cmax));
      l = fadd(l, e);
      uint4 u = *reinterpret_cast<const uint4*>(sm.v + r * HD + 8 * li);
      const float pf = __half2float(__float2half_rn(e));
      float vf[8];
      unpack8(u, vf);
#pragma unroll
      for (int j = 0; j < 8; j++) o[j] = ffma(pf, vf[j], o[j]);
    }
  }
  // groups of the warp: (g0+g2)+(g1+g3)
  l = fadd(l, __shfl_xor_sync(0xffffffffu, l, 16));
  l = fadd(l, __shfl_xor_sync(0xffffffffu, l, 8));
#pragma unroll
  for (int j = 0; j < 8; j++) {
    o[j] = fadd(o[j], __shfl_xor_sync(0xffffffffu, o[j], 16));
    o[j] = fadd(o[j], __shfl_xor_sync(0xffffffffu, o[j], 8));
  }
  if (grp == 0) {
#pragma unroll
    for (int j = 0; j < 8; j++) sm.red[warp][8 * li + j] = o[j];
    if (li == 0) sm.red[warp][64] = l;
  }
  __syncthreads();
  float* part = a.part + (((long)m * a.H + h) * a.max_chunks) * PART;
  if (tid < 65) {
    float x[8];
#pragma unroll
    for (int w = 0; w < 8; w++) x[w] = sm.red[w][tid];
    const float r = fadd(fadd(fadd(x[0], x[1]), fadd(x[2], x[3])), fadd(fadd(x[4], x[5]), fadd(x[6], x[7])));
    if (nch == 1) {
      sm.red[0][tid] = r;  // single chunk: finish locally (same arithmetic as the merge below with w = exp(0) = 1)
    } else {
      part[c * PART + (tid < 64 ? tid : 65)] = r;
      if (tid == 64) part[c * PART + 64] = cmax;
    }
  }
  if (nch > 1) {
    __threadfence();
    __syncthreads();
    if (tid == 0) {
      int* cnt = a.counters + (long)m * a.H + h;
      const int prev = atomicAdd(cnt, 1);
      sm.last = (prev == nch - 1);
      if (sm.last) *cnt = 0;  // re-arm for the next launch
    }
    __syncthreads();
    if (!sm.last) return;
    __threadfence();
    // merge in ascending chunk order.  The partials are staged in shared memory (the K / V tiles are no longer needed)
    // by all threads with every load in flight, so the merge costs one L2 round trip instead of a chain of them.
    float* pst = reinterpret_cast<float*>(sm.k);
    const bool single = nch <= ATT_MERGE_BLOCK;
    float M = -INFINITY, L = 0.0f, O = 0.0f;
    if (!single && tid < 64)
      for (int cc = 0; cc < nch; cc++) M = fmaxf(M, __ldcg(part + cc * PART + 64));
    for (int c0 = 0; c0 < nch; c0 += ATT_MERGE_BLOCK) {
      const int nb = min(ATT_MERGE_BLOCK, nch - c0);
      for (int t = tid; t < nb * PART; t += ATT_THREADS) pst[t] = __ldcg(part + (long)c0 * PART + t);
      __syncthreads();
      if (tid < 64) {
        if (single)
          for (int cc = 0; cc < nb; cc++) M = fmaxf(M, pst[cc * PART + 64]);
        for (int cc = 0; cc < nb; cc++) {
          const float w = ma_exp(fsub(pst[cc * PART + 64], M));
          L = ffma(pst[cc * PART + 65], w, L);
          O = ffma(pst[cc * PART + tid], w, O);
        }
      }
      __syncthreads();
    }
    if (tid < 64) a.out[(long)m * a.ldo + h * HD + tid] = __float2half_rn(__fdiv_rn(O, L));
  } else {
    __syncthreads();
    if (tid < 64) {
      // merge of a single chunk: w = ma_exp(0) = 1 -> L = fma(l,1,0) = l, O = fma(o,1,0) = o
      const float L = sm.red[0][64], O = sm.red[0][tid];
      a.out[(long)m * a.ldo + h * HD + tid] = __float2half_rn(__fdiv_rn(O, L));
    }
  }
}

size_t attention_scratch_bytes(int M, int H, int max_keys) {
  const size_t chunks = (size_t)(max_keys + MA_ATTN_CHUNK - 1) / MA_ATTN_CHUNK;
  return (size_t)M * H * chunks * PART * sizeof(float) + (size_t)M * H * sizeof(int) + 256;
}

int launch_attention_ex(const __half* q, int ldq, const __half* K, const __half* V, long T, int H, int rows_per_slot,
                        const int* slots, const int* nkeys, int max_keys, int M, float scale, __half* out, int ldo,
                        void* scratch, int decode_prefetch, bool pdl, cudaStream_t st) {
  if (M <= 0) return 0;
  static bool attr_done = false;
  if (!attr_done) {
    cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(AttnSmem));
    attr_done = true;
  }
  const int chunks = (max_keys + MA_ATTN_CHUNK - 1) / MA_ATTN_CHUNK;
  AttnArgs a;
  a.q = q; a.ldq = ldq; a.K = K; a.V = V; a.T = T; a.H = H;
  a.rows_per_slot = rows_per_slot > 0 ? rows_per_slot : 1;
  a.slots = slots; a.nkeys = nkeys; a.scale = scale; a.out = out; a.ldo = ldo;
  // scratch layout: counters first (must be zero on first use; every launch leaves them zero again), then the chunk
  // partials.  The split depends on M: a scratch area that serves launches with DIFFERENT M must be zeroed between
  // them (partials of one layout land on the counters of the other) -- api.cu keeps one area per M instead.
  a.counters = reinterpret_cast<int*>(scratch);
  size_t coff = ((size_t)M * H * sizeof(int) + 255) & ~(size_t)255;
  a.part = reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) + coff);
  a.max_chunks = chunks;
  a.decode_prefetch = decode_prefetch;
  dim3 grid(chunks, H, M);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(ATT_THREADS);
  cfg.dynamicSmemBytes = sizeof(AttnSmem);
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaLaunchKernelEx(&cfg, attention_kernel, a);
  count_launch();
  return check_launch("attention_kernel") ? 0 : 1;
}

int launch_attention(const __half* q, int ldq, const __half* K, const __half* V, long T, int H, int rows_per_slot,
                     const int* slots, const int* nkeys, int max_keys, int M, float scale, __half* out, int ldo,
                     void* scratch, cudaStream_t st) {
  return launch_attention_ex(q, ldq, K, V, T, H, rows_per_slot, slots, nkeys, max_keys, M, scale, out, ldo, scratch, 0,
                             false, st);
}

}  // namespace ma
