// decode_fast.cu -- batch-1 single-token decode step: 5 fused GEMV kernels per layer chained with
// programmatic dependent launch (PDL), plus lm_head + argmax + on-device bookkeeping.
//
// The step is HBM-bound (623.5 MB of fp16 weights per token, SURVEY.md 8d).  Design:
//   * every GEMV kernel runs one CTA per SM; a CTA owns a contiguous block of weight rows, which is
//     one contiguous byte range of the [N][K] matrix, so each warp pulls its rows with ONE bulk
//     async copy (cp.async.bulk, TMA 1-D) into shared memory, completion on its own mbarrier;
//   * that prefetch is issued BEFORE griddepcontrol.wait: with PDL the CTAs of kernel k+1 (and k+2..)
//     are already resident and streaming their weights while kernel k is still computing, so HBM
//     never idles across the 121 dependent phases of a token;
//   * each weight byte is read once per token, so the slab copies (and the attention's KV rows) carry the L2 evict_first
//     policy: 621 MB of weights and up to 30 MB of KV per layer stream through L2 without displacing the small data
//     that the next kernels read back (activations, residual stream, attention partials, the argmax candidates);
//   * activations never leave L2: residual add + LayerNorm are recomputed by every CTA in its
//     prologue (4 KB read), block 0 publishes the fp32 residual stream;
//   * dot products follow the canonical order (lane l owns k = 256g + 8l + j; butterfly), identical
//     to gemm_canon.cu and to the oracle, so batch-1 tokens equal batched tokens bit for bit;
//   * attention runs on attention_stream_kernel (M = 1: one CTA per SM, attention_stream.cu), which also appends the
//     current token's k / v to the cache; qkv writes q | k | v to one buffer.
// Kernels that read data produced two kernels earlier in their PDL prologue (the attention producer warp: nkeys, old KV
// rows) are only ever preceded by a kernel that triggers AFTER its own wait (qkv), so every earlier kernel has
// finished by the time they start.  Under MA_B200_NO_STREAM_ATTN=1 the attention is kv_append_kernel (launched in
// plain stream order) + attention_kernel, which fetches the old rows early for the same reason.
#include "canon.cuh"
#include "internal.h"

namespace ma {

int launch_attention_ex(const __half* q, int ldq, const __half* K, const __half* V, long T, int H, int rows_per_slot,
                        const int* slots, const int* nkeys, int max_keys, int M, float scale, __half* out, int ldo,
                        void* scratch, int decode_prefetch, bool pdl, cudaStream_t st);

constexpr int FG_THREADS = 256;
constexpr int FG_WARPS = 8;

enum { MODE_QKV = 0, MODE_OUT = 1, MODE_FC1 = 2, MODE_FC2 = 3, MODE_LM = 4 };

struct FastWs {  // device-resident scratch of the fast path (inside the decoder workspace)
  float hresA[HID];   // residual stream entering the layer (post-LN2 of the previous layer / embedding)
  float hresB[HID];   // post-LN1 residual stream
  __half qkv[QKV];    // q | k | v of the current token
  __half attn16[HID];
  __half y16[HID];
  __half f16[FFN];
  __half logits[8256];
  float cand_val[256];
  int cand_idx[256];
  int counter;
  int nkeys;
  alignas(256) unsigned char attn_scratch[256];  // really attention_scratch_bytes(...): see fast_workspace_bytes()
};

struct FastArgs {
  const __half* W;
  const __half* bias;
  int N, rows_per_cta;
  // prologue inputs
  const float* hres_in;
  const __half* y16_in;
  const float *gamma, *beta;
  const __half* x16_in;
  float* hres_out;
  int embed;  // MODE_QKV layer 0: the input is the token embedding
  const float *extra, *tok_pos, *cond, *pos_table;
  const __half* tok_table;
  SeqState s;
  // outputs
  __half* out16;
  // lm_head
  FastWs* ws;
  int do_argmax;
  int max_new, eos_id, pad_id;
  int32_t* out_ids;
  const int32_t* forced;
  __half* logits_out;
  int* all_done;
  int vocab;
};

template <int K>
struct alignas(128) FastSmemHdr {
  uint64_t bar[FG_WARPS];
  float red[8];
  float bval[FG_WARPS];
  int bidx[FG_WARPS];
  int last;
  alignas(16) __half xs[K];
};

template <int K, int MODE>
__global__ void __launch_bounds__(FG_THREADS) fast_gemv_kernel(FastArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  FastSmemHdr<K>& sh = *reinterpret_cast<FastSmemHdr<K>*>(smem_raw);
  __half* sw = reinterpret_cast<__half*>(smem_raw + sizeof(FastSmemHdr<K>));
  __half* sb = sw + (size_t)a.rows_per_cta * K;  // the bias of this CTA's rows
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (MODE != MODE_QKV) pdl_trigger();  // let the next kernel start streaming its weights right away

  // ---- rows of this CTA / this warp
  const int row0 = blockIdx.x * a.rows_per_cta;
  const int nrows = max(0, min(a.rows_per_cta, a.N - row0));
  const int base = nrows / FG_WARPS, rem = nrows % FG_WARPS;
  const int wr0 = warp * base + min(warp, rem);   // first row (relative to row0) of this warp
  const int wn = base + (warp < rem ? 1 : 0);

  // ---- weight prefetch (independent of every earlier kernel): one bulk copy per warp
  if (lane == 0) {
    mbar_init(&sh.bar[warp], 1);
    mbar_fence_init();
  }
  __syncwarp();
  if (lane == 0 && wn > 0) {
    mbar_expect_tx(&sh.bar[warp], (uint32_t)wn * K * 2);
    bulk_g2s_evict_first(sw + (size_t)wr0 * K, a.W + (size_t)(row0 + wr0) * K, (uint32_t)wn * K * 2, &sh.bar[warp]);
  }
  // the other step-independent operands (bias, LayerNorm gamma / beta, the condition embedding) are loaded here too:
  // read after the wait they would each add a DRAM round trip, queued behind the weight streams, to the token's chain
  if (a.bias)
    for (int i = tid; i < nrows; i += FG_THREADS) sb[i] = a.bias[row0 + i];
  float4 ln_g, ln_b, cond;
  if (MODE == MODE_QKV && a.embed) {
    cond = *reinterpret_cast<const float4*>(a.cond + HID + 4 * tid);
  } else if (MODE == MODE_QKV || MODE == MODE_FC1 || MODE == MODE_LM) {
    ln_g = *reinterpret_cast<const float4*>(a.gamma + 4 * tid);
    ln_b = *reinterpret_cast<const float4*>(a.beta + 4 * tid);
  }

  pdl_wait();  // everything below may read what earlier kernels wrote
  if (MODE == MODE_QKV) pdl_trigger();  // late trigger: the attention kernel prefetches dynamic data

  // ---- prologue: build the fp16 input vector in shared memory
  if (MODE == MODE_QKV || MODE == MODE_FC1 || MODE == MODE_LM) {
    float v[4];
    if (MODE == MODE_QKV && a.embed) {
      const int tok = a.s.tok[0], gen = a.s.gen[0], pos = a.s.pos[0];
      float4 X;
      int fidx;
      if (tok < 3) {
        X = *reinterpret_cast<const float4*>(a.extra + (long)tok * HID + 4 * tid);
        fidx = tok;
      } else {
        const uint2 u = *reinterpret_cast<const uint2*>(a.tok_table + (long)(tok - 3) * HID + 4 * tid);
        const __half2* h = reinterpret_cast<const __half2*>(&u);
        const float2 p0 = __half22float2(h[0]), p1 = __half22float2(h[1]);
        X = make_float4(p0.x, p0.y, p1.x, p1.y);
        int r = (gen - 2) % 9;
        if (r < 0) r += 9;
        fidx = r + 3;
      }
      const float4 F = *reinterpret_cast<const float4*>(a.tok_pos + (long)fidx * HID + 4 * tid);
      const float4 C = cond;
      const float4 P = *reinterpret_cast<const float4*>(a.pos_table + (long)(pos + 2) * HID + 4 * tid);
      v[0] = fadd(fadd(fadd(X.x, F.x), C.x), P.x);
      v[1] = fadd(fadd(fadd(X.y, F.y), C.y), P.y);
      v[2] = fadd(fadd(fadd(X.z, F.z), C.z), P.z);
      v[3] = fadd(fadd(fadd(X.w, F.w), C.w), P.w);
    } else {
      const float4 hv = *reinterpret_cast<const float4*>(a.hres_in + 4 * tid);
      const uint2 u = *reinterpret_cast<const uint2*>(a.y16_in + 4 * tid);
      const __half2* h = reinterpret_cast<const __half2*>(&u);
      const float2 p0 = __half22float2(h[0]), p1 = __half22float2(h[1]);
      v[0] = fadd(hv.x, p0.x); v[1] = fadd(hv.y, p0.y); v[2] = fadd(hv.z, p1.x); v[3] = fadd(hv.w, p1.y);
      layernorm4(v, ln_g, ln_b, MA_LN_EPS, HID, sh.red);
    }
    if (blockIdx.x == 0 && a.hres_out)
      *reinterpret_cast<float4*>(a.hres_out + 4 * tid) = make_float4(v[0], v[1], v[2], v[3]);
    __half2 h0 = __floats2half2_rn(v[0], v[1]), h1 = __floats2half2_rn(v[2], v[3]);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&h0);
    u.y = *reinterpret_cast<uint32_t*>(&h1);
    *reinterpret_cast<uint2*>(sh.xs + 4 * tid) = u;
  } else {
    // plain fp16 input (attention output / fc1 activations): K/8 16-byte pieces
    for (int i = tid; i < K / 8; i += FG_THREADS)
      *reinterpret_cast<uint4*>(sh.xs + 8 * i) = *reinterpret_cast<const uint4*>(a.x16_in + 8 * i);
  }
  __syncthreads();

  // ---- this lane's slice of x, packed fp16 (K/256 x 16 bytes)
  constexpr int G = K / 256;
  uint4 xp[G];
#pragma unroll
  for (int g = 0; g < G; g++) xp[g] = *reinterpret_cast<const uint4*>(sh.xs + 256 * g + 8 * lane);

  float bestv = -INFINITY;
  int besti = 0x7fffffff;

  if (wn > 0) mbar_wait(&sh.bar[warp], 0);
  constexpr int RB = (K == HID) ? 4 : 1;  // rows in flight per warp
  for (int r0 = 0; r0 < wn; r0 += RB) {
    float acc[RB];
#pragma unroll
    for (int i = 0; i < RB; i++) acc[i] = 0.0f;
#pragma unroll
    for (int g = 0; g < G; g++) {
      float xf[8];
      unpack8(xp[g], xf);
#pragma unroll
      for (int i = 0; i < RB; i++) {
        const int r = min(r0 + i, wn - 1);
        const uint4 u = *reinterpret_cast<const uint4*>(sw + (size_t)(wr0 + r) * K + 256 * g + 8 * lane);
        float wf[8];
        unpack8(u, wf);
#pragma unroll
        for (int j = 0; j < 8; j++) acc[i] = ffma(wf[j], xf[j], acc[i]);
      }
    }
#pragma unroll
    for (int i = 0; i < RB; i++) {
      const float sum = warp_sum(acc[i]);
      const int n = row0 + wr0 + r0 + i;
      if (r0 + i < wn && lane == 0) {
        const float bf = a.bias ? __half2float(sb[wr0 + r0 + i]) : 0.0f;
        __half h = __float2half_rn(fadd(sum, bf));
        if (MODE == MODE_FC1 && __half2float(h) < 0.0f) h = __float2half_rn(0.0f);
        a.out16[n] = h;
        if (MODE == MODE_LM) {
          const float v = __half2float(h);
          if (v > bestv || (v == bestv && n < besti)) { bestv = v; besti = n; }
        }
      }
    }
  }

  if (MODE == MODE_LM) {
    FastWs* ws = a.ws;
    const int gen = a.s.gen[0];
    if (a.logits_out) {
      // this CTA's slice of the step's logits (test hook); rows were written to out16 by lane 0 of each warp
      __syncthreads();
      for (int i = tid; i < nrows; i += FG_THREADS)
        a.logits_out[(long)gen * a.vocab + row0 + i] = a.out16[row0 + i];
    }
    if (!a.do_argmax) return;
    if (lane == 0) { sh.bval[warp] = bestv; sh.bidx[warp] = besti; }
    __syncthreads();
    if (tid == 0) {
      float bv = sh.bval[0];
      int bi = sh.bidx[0];
      for (int w = 1; w < FG_WARPS; w++)
        if (sh.bval[w] > bv || (sh.bval[w] == bv && sh.bidx[w] < bi)) { bv = sh.bval[w]; bi = sh.bidx[w]; }
      ws->cand_val[blockIdx.x] = bv;
      ws->cand_idx[blockIdx.x] = bi;
      __threadfence();
      const int prev = atomicAdd(&ws->counter, 1);
      sh.last = (prev == (int)gridDim.x - 1);
      if (sh.last) ws->counter = 0;
    }
    __syncthreads();
    if (!sh.last) return;
    __threadfence();
    // last CTA: reduce the per-CTA candidates, then do HF generate()'s bookkeeping on the device
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = tid; i < (int)gridDim.x; i += FG_THREADS) {
      const float v = __ldcg(&ws->cand_val[i]);
      const int ix = __ldcg(&ws->cand_idx[i]);
      if (v > bv || (v == bv && ix < bi)) { bv = v; bi = ix; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { sh.bval[warp] = bv; sh.bidx[warp] = bi; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < FG_WARPS; w++)
        if (sh.bval[w] > bv || (sh.bval[w] == bv && sh.bidx[w] < bi)) { bv = sh.bval[w]; bi = sh.bidx[w]; }
      int tok = bi;
      if (a.forced) tok = a.forced[gen];
      int fin = a.s.finished[0];
      if (fin) tok = a.pad_id;
      if (gen < a.max_new) a.out_ids[gen] = tok;
      if (!fin) a.s.lens[0] = gen + 1;
      if (!fin && tok == a.eos_id) fin = 1;
      a.s.finished[0] = fin;
      a.s.tok[0] = tok;
      a.s.gen[0] = gen + 1;
      const int np = a.s.pos[0] + 1;
      a.s.pos[0] = np;
      ws->nkeys = np + 1;
      if (a.all_done) *a.all_done = fin;
    }
  }
}

// ---- host side ---------------------------------------------------------------------------------
static int g_sms = 0;

size_t fast_workspace_bytes() {
  // attention scratch for one row, 16 heads, up to 18261 keys (the learned-position limit)
  return sizeof(FastWs) + attention_scratch_bytes(1, NHEAD, 18432) + 256;
}

template <int K, int MODE>
static int launch_fast(const FastArgs& a, int grid, bool pdl, cudaStream_t st) {
  const size_t smem = sizeof(FastSmemHdr<K>) + (size_t)a.rows_per_cta * K * 2 + (((size_t)a.rows_per_cta * 2 + 15) & ~(size_t)15);
  static size_t attr_set = 0;
  if (smem > attr_set) {
    cudaFuncSetAttribute(fast_gemv_kernel<K, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr_set = smem;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(FG_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaLaunchKernelEx(&cfg, fast_gemv_kernel<K, MODE>, a);
  count_launch();
  return check_launch("fast_gemv_kernel") ? 0 : 1;
}

int fast_step_enqueue(const ma_decoder_weights* w, SeqState s, int tmax, int max_keys, __half* kv, void* fast_ws,
                      const SampleArgs& sa, bool pdl, cudaStream_t st) {
  if (!g_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_sms <= 0 || g_sms > 256) g_sms = 132;
  }
  const int grid = g_sms;
  FastWs* ws = reinterpret_cast<FastWs*>(fast_ws);
  const long T = tmax;
  auto rpc = [&](int N) { return (N + grid - 1) / grid; };

  FastArgs base;
  memset(&base, 0, sizeof(base));
  base.s = s;
  base.ws = ws;
  base.extra = w->extra; base.tok_pos = w->tok_pos; base.cond = w->cond; base.pos_table = w->pos;
  base.tok_table = (const __half*)w->tok_table;
  base.vocab = w->vocab;

  for (int L = 0; L < w->n_layers; L++) {
    __half* kc = kv + ((size_t)(L * 2 + 0)) * NHEAD * T * HD;  // B = 1
    __half* vc = kv + ((size_t)(L * 2 + 1)) * NHEAD * T * HD;
    {  // qkv: input = embedding (layer 0) or LN2 of the previous layer
      FastArgs a = base;
      a.W = (const __half*)w->wqkv[L]; a.bias = (const __half*)w->bqkv[L]; a.N = QKV; a.rows_per_cta = rpc(QKV);
      a.embed = (L == 0);
      if (L > 0) { a.hres_in = ws->hresB; a.y16_in = ws->y16; a.gamma = w->ln2g[L - 1]; a.beta = w->ln2b[L - 1]; }
      a.hres_out = ws->hresA;
      a.out16 = ws->qkv;
      if (launch_fast<HID, MODE_QKV>(a, grid, pdl, st)) return 1;
    }
    if (!no_stream_attn()) {
      if (launch_attention_decode(ws->qkv, QKV, kc, vc, T, &ws->nkeys, max_keys, 1, 0.125f, ws->attn16, HID,
                                  ws->attn_scratch, pdl, st)) return 1;
    } else {
      if (launch_kv_append(ws->qkv, 1, 1, &ws->nkeys, kc, vc, T, st)) return 1;
      if (launch_attention_ex(ws->qkv, QKV, kc, vc, T, NHEAD, 1, nullptr, &ws->nkeys, max_keys, 1, 0.125f, ws->attn16,
                              HID, ws->attn_scratch, 1, pdl, st)) return 1;
    }
    {  // out_proj
      FastArgs a = base;
      a.W = (const __half*)w->wo[L]; a.bias = (const __half*)w->bo[L]; a.N = HID; a.rows_per_cta = rpc(HID);
      a.x16_in = ws->attn16; a.out16 = ws->y16;
      if (launch_fast<HID, MODE_OUT>(a, grid, pdl, st)) return 1;
    }
    {  // fc1: input = LN1(hresA + y16)
      FastArgs a = base;
      a.W = (const __half*)w->w1[L]; a.bias = (const __half*)w->b1[L]; a.N = FFN; a.rows_per_cta = rpc(FFN);
      a.hres_in = ws->hresA; a.y16_in = ws->y16; a.gamma = w->ln1g[L]; a.beta = w->ln1b[L];
      a.hres_out = ws->hresB; a.out16 = ws->f16;
      if (launch_fast<HID, MODE_FC1>(a, grid, pdl, st)) return 1;
    }
    {  // fc2
      FastArgs a = base;
      a.W = (const __half*)w->w2[L]; a.bias = (const __half*)w->b2[L]; a.N = HID; a.rows_per_cta = rpc(HID);
      a.x16_in = ws->f16; a.out16 = ws->y16;
      if (launch_fast<FFN, MODE_FC2>(a, grid, pdl, st)) return 1;
    }
  }
  {  // lm_head on LN2 of the last layer (+ greedy pick and bookkeeping)
    FastArgs a = base;
    const int L = w->n_layers - 1;
    a.W = (const __half*)w->lm_head; a.bias = nullptr; a.N = w->vocab; a.rows_per_cta = rpc(w->vocab);
    a.hres_in = ws->hresB; a.y16_in = ws->y16; a.gamma = w->ln2g[L]; a.beta = w->ln2b[L];
    a.out16 = sa.do_sample ? const_cast<__half*>(sa.logits) : ws->logits;
    a.do_argmax = !sa.do_sample;
    a.max_new = sa.max_new; a.eos_id = sa.eos_id; a.pad_id = sa.pad_id;
    a.out_ids = sa.out_ids; a.forced = sa.forced; a.logits_out = sa.logits_out; a.all_done = sa.all_done;
    if (launch_fast<HID, MODE_LM>(a, grid, pdl, st)) return 1;
  }
  if (sa.do_sample) {
    SampleArgs s2 = sa;
    s2.logits_out = nullptr;  // already written by the lm_head kernel
    s2.nkeys_next = &ws->nkeys;
    if (launch_sample(s2, st)) return 1;
  }
  return 0;
}

int* fast_nkeys_ptr(void* fast_ws) { return &reinterpret_cast<FastWs*>(fast_ws)->nkeys; }

}  // namespace ma
