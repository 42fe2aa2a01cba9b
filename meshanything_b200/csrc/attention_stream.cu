// attention_stream.cu -- decode attention of a batch as ONE persistent, software-pipelined kernel.
//
// Same arithmetic as attention.cu (the canonical chunked attention that replaces flash_attn_func of OptFlashAttention2
// for q [B,1,16,64] against the KV cache, /root/reference/MeshAnything/models/shape_opt.py:205 -> transformers'
// OPTDecoderLayer attention) -- bit for bit: same chunks of MA_ATTN_CHUNK keys, same lane chains, same butterflies,
// same ascending merge.  What changes is how the bytes move.  attention_kernel gives every (row, head, chunk) its own
// CTA that loads 64 KB, waits for all of it, computes and exits.
// Here persistent CTAs (two per SM for a batch, one per SM for a single row: see the launcher) each walk their share
// of the work; a work item is a SEGMENT = a few consecutive chunks of one (row, head):
//   * warp 0 is the producer: the K rows and the V rows of a chunk are two 32 KB half-stages of a ring of 3 (batch) or
//     4 (single row) slots (cp.async.bulk onto mbarriers); the K slot is handed back right after the score pass, the
//     V slot after the P.V pass, so the next chunk's rows are in flight while this one is being computed -- HBM never
//     idles between chunks and no CTA launch / drain sits between two loads;
//   * 8 consumer warps; the score butterfly is lane-transposed: the 8 lanes of a row group hold partial dots of the
//     group's 8 rows, and an xor-4,2,1 exchange that halves the rows each level leaves lane li with the finished score
//     of row li (7 shuffles for 8 rows, one exp per row) -- the same additions in the same tree as the plain xor
//     butterfly;
//   * the k / v rows of the CURRENT token are taken straight from the qkv buffer by the lanes that own that key row and
//     written to the cache from there (kv_append_kernel folded in: one launch less per layer);
//   * chunk partials go to scratch with plain stores; a SEGMENT pays one fence + one atomic ticket (attention_kernel:
//     one per chunk -- a serialised ~2 us that a persistent CTA cannot hide behind other CTAs); the segment that
//     completes a (row, head) stages all partials in shared memory with 256 loads in flight together and runs the
//     ascending canonical merge from there.
#include "canon.cuh"
#include "internal.h"

namespace ma {

// Ring of 32 KB half-stages (the K or the V rows of one chunk): 3 slots for a batch (two CTAs per SM), 4 for a single
// row (one CTA per SM: two whole chunks fetched before the grid dependency resolves, see the launcher)
constexpr int AS_SLOTS_BATCH = 3;
constexpr int AS_SLOTS_ROW = 4;
constexpr int AS_TEAM = 256;                                 // consumer threads
constexpr int AS_THREADS = 32 + AS_TEAM;                     // warp 0 = producer
constexpr int AS_PART = 66;                                  // o[64], max, sum (layout of attention.cu)
constexpr int AS_MERGE_BLOCK = 29;                           // chunks staged per merge round

template <int SLOTS>
struct AttnStreamSmem {
  __half ring[SLOTS][MA_ATTN_CHUNK * HD];   // K0, V0, K1, V1, ... of this CTA's chunks, in this order
  float red[8][65];
  float pst[AS_MERGE_BLOCK * AS_PART];
  float wgt[64];
  float mst[64];
  float wmax[8];
  uint64_t full[SLOTS], empty[SLOTS];
  int last;
};
// H100: 233472 B of shared memory per SM, 1024 B reserved per CTA
static_assert(2 * (sizeof(AttnStreamSmem<AS_SLOTS_BATCH>) + 1024) <= 233472, "two CTAs of the batch geometry per SM");
// the single-row CTA next to the batch-1 out_proj CTA (8 weight rows of 1024, 18704 B) and fc1 CTA (32 rows, 67904 B)
// of decode_fast.cu on 132 SMs; more than half the SM, so never two on one SM
static_assert(sizeof(AttnStreamSmem<AS_SLOTS_ROW>) + 1024 + (18704 + 1024) + (67904 + 1024) <= 233472 &&
                  2 * (sizeof(AttnStreamSmem<AS_SLOTS_ROW>) + 1024) > 233472,
              "one CTA of the single-row geometry per SM, co-resident with the out_proj and fc1 GEMV CTAs");

struct AttnStreamArgs {
  const __half* q;      // [M][ldq]: q | k | v of the current token (ld = 3072)
  int ldq;
  __half* K;            // cache of this layer, [slot][head][T][64]
  __half* V;
  long T;
  const int* nkeys;     // keys per row INCLUDING the current token
  __half* out;          // [M][ldo]
  int ldo;
  float* part;
  int* counters;
  int M, max_chunks;
  int cps, nseg;        // chunks per segment, segments per (row, head)
  float scale;
};

__device__ __forceinline__ void team_bar() { asm volatile("bar.sync 1, %0;" ::"n"(AS_TEAM) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// Work item w = (row m, head h, segment g): chunks [g * cps, min((g + 1) * cps, chunks of row m)) -- g fastest.
struct AsItem {
  int m, h, c0, c1, n, nk, nch;
};
__device__ __forceinline__ int as_row(const AttnStreamArgs& a, int w) { return w / (a.nseg * NHEAD); }
// nkeys[m] of the row of item w, kept in (row, nk) across the items of a CTA: it is read from L2 because both roles read
// it before the grid dependency resolves (the first item's; see the consumers) and must see one value
__device__ __forceinline__ int as_nkeys(const AttnStreamArgs& a, int w, int& row, int& nk) {
  const int m = as_row(a, w);
  if (m != row) {
    row = m;
    nk = __ldcg(a.nkeys + m);
  }
  return nk;
}
__device__ __forceinline__ bool as_item(const AttnStreamArgs& a, int w, int nk, AsItem& it) {
  const int g = w % a.nseg, h = (w / a.nseg) % NHEAD;
  it.m = as_row(a, w);
  it.h = h;
  it.nk = nk;
  // never more keys than this launch has chunks for: a frozen cache slot (continuous batching) keeps an old, possibly
  // larger position than the bucket the launch was sized from; its output is discarded anyway
  it.n = min(it.nk, a.max_chunks * MA_ATTN_CHUNK);
  it.nch = (it.n + MA_ATTN_CHUNK - 1) / MA_ATTN_CHUNK;
  it.c0 = g * a.cps;
  it.c1 = min(it.nch, it.c0 + a.cps);
  return it.c0 < it.c1;
}

template <int SLOTS>
__global__ void __launch_bounds__(AS_THREADS, 2) attention_stream_kernel(AttnStreamArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  AttnStreamSmem<SLOTS>& sm = *reinterpret_cast<AttnStreamSmem<SLOTS>*>(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nitems = a.nseg * NHEAD * a.M;

  if (tid == 0) {
    for (int s = 0; s < SLOTS; s++) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.empty[s], 1);
    }
    mbar_fence_init();
  }
  __syncthreads();

  // Items of this CTA: w = blockIdx.x, + gridDim.x, ...  Producer and consumers walk the same items and chunks, so both
  // count the same sequence of half-stages u = 0 (K), 1 (V), 2 (K of the next chunk), ... ; half-stage u lives in
  // ring slot u % SLOTS and completes phase u / SLOTS of that slot's barriers.
  if (warp == 0) {
    // ---------------------------------------------------------------- producer
    // It only ever reads cache rows written by earlier steps (and nkeys, written by an earlier step's kernel), so it
    // does not wait for the grid dependency: under programmatic dependent launch its first loads overlap the tail of
    // the previous kernel.
    if (lane != 0) return;
    int u = 0, row = -1, nk = 0;
    for (int w = blockIdx.x; w < nitems; w += gridDim.x) {
      AsItem it;
      if (!as_item(a, w, as_nkeys(a, w, row, nk), it)) continue;
      for (int c = it.c0; c < it.c1; c++) {
        const int len = min(MA_ATTN_CHUNK, it.n - c * MA_ATTN_CHUNK);
        // rows older than the current token (the current one comes from the qkv buffer, not from the cache)
        const int old = (it.nk == it.n) ? min(len, (it.n - 1) - c * MA_ATTN_CHUNK) : len;
        const long base = (((long)it.m * NHEAD + it.h) * a.T + (long)c * MA_ATTN_CHUNK) * HD;
#pragma unroll
        for (int kv = 0; kv < 2; kv++, u++) {
          const int s = u % SLOTS;
          if (u >= SLOTS) mbar_wait(&sm.empty[s], ((u / SLOTS) & 1) ^ 1);
          if (old > 0) {
            mbar_expect_tx(&sm.full[s], (uint32_t)old * HD * 2);
            // a single row (the batch-1 step) reads each cache row once per step: evict_first keeps the up to 30 MB of a
            // layer's cache from pushing the step's other data out of L2
            if (SLOTS == AS_SLOTS_ROW)
              bulk_g2s_evict_first(sm.ring[s], (kv ? a.V : a.K) + base, (uint32_t)old * HD * 2, &sm.full[s]);
            else
              bulk_g2s(sm.ring[s], (kv ? a.V : a.K) + base, (uint32_t)old * HD * 2, &sm.full[s]);
          } else {
            mbar_arrive(&sm.full[s]);   // only the current token in this chunk: nothing to load
          }
        }
      }
    }
    return;
  }

  // ---------------------------------------------------------------- consumers (8 warps)
  const int wt = warp - 1, tl = tid - 32;
  const int grp = lane >> 3, li = lane & 7;
  // nkeys of the first item before the wait, as the producer reads it: after the wait the q load is then the only L2
  // round trip ahead of the first score pass (at a single row every item of the CTA has this row)
  int row = -1, nk = 0;
  if (blockIdx.x < nitems) as_nkeys(a, blockIdx.x, row, nk);
  pdl_wait();      // q / k / v of the current token come from the previous kernel
  pdl_trigger();
  int u = 0;
  for (int w = blockIdx.x; w < nitems; w += gridDim.x) {
    AsItem it;
    if (!as_item(a, w, as_nkeys(a, w, row, nk), it)) continue;
    const int m = it.m, h = it.h, nch = it.nch;
    const __half* qrow = a.q + (long)m * a.ldq + h * HD + 8 * li;
    const uint4 qp = *reinterpret_cast<const uint4*>(qrow);
    float* part = a.part + (((long)m * NHEAD + h) * a.max_chunks) * AS_PART;

    for (int c = it.c0; c < it.c1; c++, u += 2) {
      const int sk = u % SLOTS, sv = (u + 1) % SLOTS;
      const int len = min(MA_ATTN_CHUNK, it.n - c * MA_ATTN_CHUNK);
      const int cur = (it.nk == it.n) ? (it.n - 1) - c * MA_ATTN_CHUNK : -1;   // row of the current token in this chunk
      uint4 kcur = make_uint4(0, 0, 0, 0), vcur = kcur;
      const bool own_cur = cur >= 0 && cur < MA_ATTN_CHUNK && (4 * wt + grp) == (cur & 31);
      if (own_cur) {
        kcur = *reinterpret_cast<const uint4*>(qrow + HID);
        vcur = *reinterpret_cast<const uint4*>(qrow + 2 * HID);
        const long dst = (((long)m * NHEAD + h) * a.T + (long)c * MA_ATTN_CHUNK + cur) * HD + 8 * li;
        *reinterpret_cast<uint4*>(a.K + dst) = kcur;   // kv_append: later steps read it from the cache
        *reinterpret_cast<uint4*>(a.V + dst) = vcur;
      }
      const int rho_c = own_cur ? (cur >> 5) : -1;
      const __half* ks = sm.ring[sk];
      const __half* vs = sm.ring[sv];
      mbar_wait(&sm.full[sk], (u / SLOTS) & 1);

      // scores: partial dot of this lane's 8 dimensions for its group's 8 rows, then the transposing butterfly: lane
      // li ends up with the finished xor-4,2,1 sum of row rho = li
      float pr[8];
#pragma unroll
      for (int rho = 0; rho < 8; rho++) {
        const int r = 32 * rho + 4 * wt + grp;
        uint4 x = *reinterpret_cast<const uint4*>(ks + r * HD + 8 * li);   // rows >= len: stale bytes, masked below
        if (rho == rho_c) x = kcur;
        pr[rho] = dot8(qp, x, 0.0f);
      }
#pragma unroll
      for (int sft = 4; sft >= 1; sft >>= 1) {
        const bool up = (li & sft) != 0;
#pragma unroll
        for (int t = 0; t < sft; t++) {
          const float mine = up ? pr[t + sft] : pr[t];
          const float other = up ? pr[t] : pr[t + sft];
          pr[t] = fadd(mine, __shfl_xor_sync(0xffffffffu, other, sft));
        }
      }
      const float s_own = fmul(pr[0], a.scale);
      const bool own_valid = 32 * li + 4 * wt + grp < len;
      const float lmax = warp_max(own_valid ? s_own : -INFINITY);
      if (lane == 0) sm.wmax[wt] = lmax;   // readers of the previous chunk's maxima are past that chunk's last barrier
      team_bar();                          // every thread is past its reads of the K half-stage
      if (tl == 0) mbar_arrive(&sm.empty[sk]);
      float cmax = sm.wmax[0];
#pragma unroll
      for (int w2 = 1; w2 < 8; w2++) cmax = fmaxf(cmax, sm.wmax[w2]);
      const float e_own = own_valid ? ma_exp(fsub(s_own, cmax)) : 0.0f;
      float l = 0.0f, o[8];
#pragma unroll
      for (int t = 0; t < 8; t++) o[t] = 0.0f;
      mbar_wait(&sm.full[sv], ((u + 1) / SLOTS) & 1);
#pragma unroll
      for (int rho = 0; rho < 8; rho++) {
        const int r = 32 * rho + 4 * wt + grp;
        const float e = __shfl_sync(0xffffffffu, e_own, (lane & 24) | rho);   // from the lane that owns row rho
        if (r < len) {
          l = fadd(l, e);
          uint4 x = *reinterpret_cast<const uint4*>(vs + r * HD + 8 * li);
          if (rho == rho_c) x = vcur;
          pv8(__float2half_rn(e), x, o);
        }
      }
      l = fadd(l, __shfl_xor_sync(0xffffffffu, l, 16));
      l = fadd(l, __shfl_xor_sync(0xffffffffu, l, 8));
#pragma unroll
      for (int t = 0; t < 8; t++) {
        o[t] = fadd(o[t], __shfl_xor_sync(0xffffffffu, o[t], 16));
        o[t] = fadd(o[t], __shfl_xor_sync(0xffffffffu, o[t], 8));
      }
      if (grp == 0) {
#pragma unroll
        for (int t = 0; t < 8; t++) sm.red[wt][8 * li + t] = o[t];
        if (li == 0) sm.red[wt][64] = l;
      }
      team_bar();   // every thread is past its reads of the V half-stage; red complete
      if (tl == 0) mbar_arrive(&sm.empty[sv]);
      if (tl < 65) {
        float x[8];
#pragma unroll
        for (int w2 = 0; w2 < 8; w2++) x[w2] = sm.red[w2][tl];
        const float rsum = fadd(fadd(fadd(x[0], x[1]), fadd(x[2], x[3])), fadd(fadd(x[4], x[5]), fadd(x[6], x[7])));
        if (nch == 1) {
          sm.pst[tl] = rsum;   // single chunk: finished below without the scratch area
        } else {
          part[c * AS_PART + (tl < 64 ? tl : 65)] = rsum;
          if (tl == 64) part[c * AS_PART + 64] = cmax;
        }
      }
      // (red is rewritten only after the next chunk's first barrier, which these 65 threads reach after their reads)
    }

    if (nch == 1) {
      // the merge with w = exp(0) = 1 -> L = fma(l, 1, 0) = l, O = fma(o, 1, 0) = o
      team_bar();
      if (tl < 64) a.out[(long)m * a.ldo + h * HD + tl] = __float2half_rn(__fdiv_rn(sm.pst[tl], sm.pst[64]));
      team_bar();   // pst is free again
      continue;
    }
    // this segment's partials are written; the segment that completes the (row, head) merges all of them
    __threadfence();
    team_bar();
    const int nseg_row = (nch + a.cps - 1) / a.cps;
    if (nseg_row > 1) {
      if (tl == 0) {
        int* cnt = a.counters + (long)m * NHEAD + h;
        const int prev = atomicAdd(cnt, 1);
        const int last = (prev == nseg_row - 1);
        if (last) *cnt = 0;   // re-arm for the next launch
        sm.last = last;
      }
      team_bar();
      const int last = sm.last;
      team_bar();             // sm.last may be rewritten by the next item
      if (!last) continue;
      __threadfence();
    }
    // merge of the chunks of (m, h) in ascending order; partials staged through shared memory in blocks
    const bool single = nch <= AS_MERGE_BLOCK;
    if (!single) {
      for (int t = tl; t < nch; t += AS_TEAM) sm.mst[t] = __ldcg(part + t * AS_PART + 64);
      team_bar();
      float Mx = -INFINITY;
      for (int cc = 0; cc < nch; cc++) Mx = fmaxf(Mx, sm.mst[cc]);
      for (int t = tl; t < nch; t += AS_TEAM) sm.wgt[t] = ma_exp(fsub(sm.mst[t], Mx));
    }
    float Lsum = 0.0f, O = 0.0f;
    for (int c0 = 0; c0 < nch; c0 += AS_MERGE_BLOCK) {
      const int nb = min(AS_MERGE_BLOCK, nch - c0), nw = nb * AS_PART;
      for (int t = tl; t < nw; t += AS_TEAM) sm.pst[t] = __ldcg(part + (long)c0 * AS_PART + t);
      team_bar();
      if (single) {
        float Mx = -INFINITY;
        for (int cc = 0; cc < nch; cc++) Mx = fmaxf(Mx, sm.pst[cc * AS_PART + 64]);
        for (int t = tl; t < nch; t += AS_TEAM) sm.wgt[t] = ma_exp(fsub(sm.pst[t * AS_PART + 64], Mx));
        team_bar();
      }
      if (tl < 64) {
        for (int cc = 0; cc < nb; cc++) {
          const float wc = sm.wgt[c0 + cc];
          Lsum = ffma(sm.pst[cc * AS_PART + 65], wc, Lsum);
          O = ffma(sm.pst[cc * AS_PART + tl], wc, O);
        }
      }
      team_bar();
    }
    if (tl < 64) a.out[(long)m * a.ldo + h * HD + tl] = __float2half_rn(__fdiv_rn(O, Lsum));
  }
}

static int g_as_sms = 0;

// Decode attention for M rows (row m = cache slot m, one query each) + append of the current k / v to the cache.
// scratch: the layout of launch_attention_ex (counters, then partials), sized by attention_scratch_bytes.
//
// Geometry from M.  A batch (M > 1) runs two CTAs per SM with a 3-slot ring: the attention of B rows is a large share
// of the step and owns the SM.  A single row (the batch-1 decode step) runs ONE CTA per SM with a 4-slot ring
// (~139 KB): more than half the SM, so no SM gets two, and small enough that the per-phase GEMV kernels around it
// (decode_fast.cu) stay co-resident -- the qkv CTA (~52 KB) before it, then the out_proj (~19 KB) and fc1 (~67 KB)
// CTAs, which issue their weight bulk copies while the attention still streams the KV cache.  The producer fills the
// ring before the grid dependency resolves, i.e. while qkv computes: two whole chunks, which at up to 4 chunks per
// CTA (7459 keys) is half of the CTA's bytes.  Same consumers, same arithmetic, same bits.
int launch_attention_decode(const __half* qkv, int ldq, __half* K, __half* V, long T, const int* nkeys, int max_keys,
                            int M, float scale, __half* out, int ldo, void* scratch, bool pdl, cudaStream_t st) {
  if (M <= 0) return 0;
  if (!g_as_sms) {
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaFuncSetAttribute(attention_stream_kernel<AS_SLOTS_BATCH>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)sizeof(AttnStreamSmem<AS_SLOTS_BATCH>));
    cudaFuncSetAttribute(attention_stream_kernel<AS_SLOTS_ROW>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)sizeof(AttnStreamSmem<AS_SLOTS_ROW>));
    g_as_sms = sms > 0 ? sms : 132;
  }
  const bool row = M == 1;
  const int ctas = (row ? 1 : 2) * g_as_sms;
  const int chunks = (max_keys + MA_ATTN_CHUNK - 1) / MA_ATTN_CHUNK;
  AttnStreamArgs a;
  a.q = qkv; a.ldq = ldq; a.K = K; a.V = V; a.T = T; a.nkeys = nkeys; a.out = out; a.ldo = ldo;
  a.counters = reinterpret_cast<int*>(scratch);
  const size_t coff = ((size_t)M * NHEAD * sizeof(int) + 255) & ~(size_t)255;
  a.part = reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) + coff);
  a.M = M; a.max_chunks = chunks; a.scale = scale;
  // Segment length (chunks per work item): a segment pays one q load + one fence + one atomic ticket (~1 chunk's worth
  // of time, mostly hidden behind the ring's prefetch), a chunk none; items are dealt round-robin to the CTAs.  Take
  // the length that minimises the longest CTA's work, ceil(items / CTAs) * (cps + 1); ties go to the longer segment.
  {
    long best = -1;
    int best_cps = 1;
    for (int cps = 1; cps <= chunks; cps++) {
      const int nseg = (chunks + cps - 1) / cps;
      const long items = (long)nseg * NHEAD * M;
      const long cost = ((items + ctas - 1) / ctas) * (long)(min(cps, chunks) + 1);
      if (best < 0 || cost <= best) { best = cost; best_cps = cps; }
    }
    a.cps = best_cps;
    a.nseg = (chunks + a.cps - 1) / a.cps;
  }
  const long nitems = (long)a.nseg * NHEAD * M;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)min((long)ctas, nitems));
  cfg.blockDim = dim3(AS_THREADS);
  cfg.dynamicSmemBytes = row ? sizeof(AttnStreamSmem<AS_SLOTS_ROW>) : sizeof(AttnStreamSmem<AS_SLOTS_BATCH>);
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  if (row)
    cudaLaunchKernelEx(&cfg, attention_stream_kernel<AS_SLOTS_ROW>, a);
  else
    cudaLaunchKernelEx(&cfg, attention_stream_kernel<AS_SLOTS_BATCH>, a);
  count_launch();
  return check_launch("attention_stream_kernel") ? 0 : 1;
}

}  // namespace ma
