// api.cu -- the C ABI of libmeshanything_b200.so (include/meshanything_b200.h) and the host side
// of generate(): prefill, then one CUDA graph launch per token.
#include <stdarg.h>
#include <stdlib.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <map>
#include <mutex>
#include <vector>

#include "canon.cuh"
#include "internal.h"

namespace ma {

static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches += (unsigned long long)n; }
bool check_launch(const char* what) {
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    cudaGetLastError();
    return false;
  }
  return true;
}

static inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// ---- workspace carve-up of the decoder ---------------------------------------------------------
constexpr int PREFILL_SEQS = 8;  // sequences prefilled per pass (rows = 257 * PREFILL_SEQS)

struct DecWs {
  float* hres;
  __half *x16, *qkv, *attn16, *y16, *f16, *logits, *lastx16;
  int* nkeys;
  SeqState s;
  int* all_done;
  void* attn_scratch;      // decode steps (M = B rows)
  size_t attn_scratch_bytes;
  void* attn_scratch_pre;  // prefill passes (M = 257 x sequences): its own area, because the layout (counters, then
  size_t attn_scratch_pre_bytes;  // partials) depends on M and a slot prefill may follow decode steps
  void* fast;
  void* tc_scratch;   // gemm_ws.cu: fp32 K-slice partials + tickets
  size_t total;
};

static DecWs carve(void* base, int B, int tmax, int vocab) {
  DecWs w;
  const size_t rows = (size_t)std::max(B, PREFIX * std::min(B, PREFILL_SEQS));
  size_t off = 0;
  auto take = [&](size_t bytes) {
    void* p = base ? (void*)((char*)base + off) : nullptr;
    off += align_up(bytes);
    return p;
  };
  w.hres = (float*)take(rows * HID * 4);
  w.x16 = (__half*)take(rows * HID * 2);
  w.qkv = (__half*)take(rows * QKV * 2);
  w.attn16 = (__half*)take(rows * HID * 2);
  w.y16 = (__half*)take(rows * HID * 2);
  w.f16 = (__half*)take(rows * FFN * 2);
  w.logits = (__half*)take((size_t)B * vocab * 2);
  w.lastx16 = (__half*)take((size_t)B * HID * 2);
  w.nkeys = (int*)take(rows * 4);
  w.s.pos = (int*)take((size_t)B * 4);
  w.s.gen = (int*)take((size_t)B * 4);
  w.s.tok = (int*)take((size_t)B * 4);
  w.s.finished = (int*)take((size_t)B * 4);
  w.s.lens = (int*)take((size_t)B * 4);
  w.s.sid = (int*)take((size_t)B * 4);
  w.all_done = (int*)take(256);
  w.attn_scratch_bytes = attention_scratch_bytes((int)B, NHEAD, tmax);
  w.attn_scratch = take(w.attn_scratch_bytes);
  w.attn_scratch_pre_bytes = attention_scratch_bytes(PREFIX * std::min(B, PREFILL_SEQS), NHEAD, PREFIX);
  w.attn_scratch_pre = take(w.attn_scratch_pre_bytes);
  w.fast = take(fast_workspace_bytes());
  w.tc_scratch = take(linear_ws_scratch_bytes());
  w.total = off;
  return w;
}

static inline __half* kv_layer(void* kv, int layer, int which, int B, long T) {
  return (__half*)kv + ((size_t)(layer * 2 + which) * B) * NHEAD * T * HD;
}

// MA_B200_NO_STREAM_ATTN=1: decode steps of a batch use kv_append_kernel + attention_kernel (one CTA per chunk) instead
// of attention_stream_kernel -- same bits, kept for A/B timing (tools/bench_batched.py)
static const bool g_no_stream_attn = [] {
  const char* e = getenv("MA_B200_NO_STREAM_ATTN");
  return e && e[0] == '1';
}();

static const bool g_no_pdl = [] {   // MA_B200_NO_PDL=1: plain stream order between the kernels of a batched decode step
  const char* e = getenv("MA_B200_NO_PDL");
  return e && e[0] == '1';
}();

// One pass of the 24 layers over M rows (general batched kernels).
// y = act(x W^T + b) for M rows of the decoder: the canonical kernel, or (tc) the tensor cores -- the weight-streaming
// wgmma GEMM for M <= 128 rows (decode steps), the tiled wgmma GEMM for the 257-row prefill passes
static int dec_linear(bool tc, const DecWs& ws, const void* W, const void* b, const __half* x, int ldx, __half* y, int ldy,
                      int M, int N, int K, int epi, cudaStream_t st, bool pdl = false) {
  if (tc) {
    // Up to 128 rows the weight-streaming kernel takes every matrix (it reads each weight once and splits K across
    // the SMs; lm_head, N = 8195, is not tileable at all); the tiled kernel keeps the 257-row prefill passes.
    // tools/bench_batched.py times the three kernels per decoder shape.
    const bool tiled_ok = M >= 64 && linear_tc_supported(M, N, K, ldx, ldy, x, W, y);
    const bool ws_ok = M <= 128 && linear_ws_supported(M, N, K, ldx, x, W);
    if (ws_ok && (linear_ws_mode() || !tiled_ok || K > 1024))
      return launch_linear_ws((const __half*)W, (const __half*)b, x, ldx, y, ldy, M, N, K, epi, ws.tc_scratch, st, pdl);
    if (tiled_ok) return launch_linear_tc((const __half*)W, (const __half*)b, x, ldx, y, ldy, M, N, K, epi, st);
  }
  return launch_linear((const __half*)W, (const __half*)b, x, ldx, y, ldy, M, N, K, epi, st);
}

static int run_layers(const ma_decoder_weights* w, const DecWs& ws, void* kv, int B, long T, int M, int rows_per_slot,
                      int slot0, int max_keys, cudaStream_t st, bool tc = false) {
  void* scratch = rows_per_slot > 1 ? ws.attn_scratch_pre : ws.attn_scratch;
  // Decode step of a batch on the tensor-core path: the kernels of a layer are programmatic dependents of each other --
  // a GEMM sends its first ring of WEIGHT tiles, the attention its first K / V rows, before the previous kernel has
  // finished (each waits with griddepcontrol.wait before it touches anything the previous kernel wrote)
  const bool pdl = tc && rows_per_slot == 1 && !g_no_pdl;
  for (int L = 0; L < w->n_layers; L++) {
    __half* kc = kv_layer(kv, L, 0, B, T) + (size_t)slot0 * NHEAD * T * HD;
    __half* vc = kv_layer(kv, L, 1, B, T) + (size_t)slot0 * NHEAD * T * HD;
    if (dec_linear(tc, ws, w->wqkv[L], w->bqkv[L], ws.x16, HID, ws.qkv, QKV, M, QKV, HID, MA_EPI_NONE, st, pdl)) return 1;
    if (rows_per_slot == 1 && !g_no_stream_attn) {
      // decode step of a batch: persistent pipelined kernel, k / v of the current token appended on the way
      if (launch_attention_decode(ws.qkv, QKV, kc, vc, T, ws.nkeys, max_keys, M, 0.125f, ws.attn16, HID, scratch, pdl,
                                  st)) return 1;
    } else {
      if (launch_kv_append(ws.qkv, M, rows_per_slot, ws.nkeys, kc, vc, T, st)) return 1;
      if (launch_attention(ws.qkv, QKV, kc, vc, T, NHEAD, rows_per_slot, nullptr, ws.nkeys, max_keys, M, 0.125f,
                           ws.attn16, HID, scratch, st)) return 1;
    }
    if (dec_linear(tc, ws, w->wo[L], w->bo[L], ws.attn16, HID, ws.y16, HID, M, HID, HID, MA_EPI_NONE, st, pdl)) return 1;
    if (launch_layernorm(ws.hres, ws.y16, w->ln1g[L], w->ln1b[L], MA_LN_EPS, M, HID, ws.hres, ws.x16, st, pdl)) return 1;
    if (dec_linear(tc, ws, w->w1[L], w->b1[L], ws.x16, HID, ws.f16, FFN, M, FFN, HID, MA_EPI_RELU, st, pdl)) return 1;
    if (dec_linear(tc, ws, w->w2[L], w->b2[L], ws.f16, FFN, ws.y16, HID, M, HID, FFN, MA_EPI_NONE, st, pdl)) return 1;
    if (launch_layernorm(ws.hres, ws.y16, w->ln2g[L], w->ln2b[L], MA_LN_EPS, M, HID, ws.hres, ws.x16, st, pdl)) return 1;
  }
  return 0;
}

// ---- per-step CUDA graphs ----------------------------------------------------------------------
struct GraphKey {
  const void *w, *kv, *ws, *out_ids, *forced, *logits_out;
  unsigned long long whash;
  // mode: generate (0) or slot (1) graphs; ws_mode: the gemm_ws reduction (linear_ws_mode()), which a graph bakes in
  int B, tmax, max_new, bucket, flags, do_sample, top_k, eos, pad, mode, ws_mode;
  float top_p;
  unsigned long long seed;
  bool operator<(const GraphKey& o) const { return memcmp(this, &o, sizeof(GraphKey)) < 0; }
};
static std::map<GraphKey, cudaGraphExec_t> g_graphs;
static std::map<cudaGraphExec_t, unsigned long long> g_graph_launches;  // kernels per launch of a graph
static cudaStream_t g_stream = nullptr;
static int* g_flag_host = nullptr;  // pinned
static cudaEvent_t g_ev_in = nullptr, g_ev_out = nullptr, g_ev_flag = nullptr;

static int g_device = -1;   // the library keeps one internal stream + graph cache: one device per process
static std::mutex g_mu;     // ma_decode_generate is serialised (graph cache, pinned flag, internal stream)

static int ensure_globals() {
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    set_error("cudaGetDevice: %s", cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  if (g_device >= 0 && dev != g_device) {
    set_error("ma_decode_generate was first used on device %d; this process now runs on device %d "
              "(one process per GPU)", g_device, dev);
    return 1;
  }
  if (!g_stream) {
    if (cudaStreamCreateWithFlags(&g_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaHostAlloc((void**)&g_flag_host, 64, cudaHostAllocDefault) != cudaSuccess ||
        cudaEventCreateWithFlags(&g_ev_in, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&g_ev_out, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&g_ev_flag, cudaEventDisableTiming) != cudaSuccess) {
      set_error("cannot create stream/events: %s", cudaGetErrorString(cudaGetLastError()));
      return 1;
    }
    g_device = dev;
  }
  return 0;
}


// One decode step of the whole batch on the general kernels (embed -> 24 layers -> lm_head -> pick).
static int enqueue_batched_step(const ma_decoder_weights* w, const DecWs& ws, void* kv, int B, long T, int max_keys,
                                const SampleArgs& sa, cudaStream_t s, bool tc) {
  if (launch_embed_tokens(w, ws.s, B, ws.hres, ws.x16, ws.nkeys, s)) return 1;
  if (run_layers(w, ws, kv, B, T, B, 1, 0, max_keys, s, tc)) return 1;
  if (dec_linear(tc, ws, w->lm_head, nullptr, ws.x16, HID, ws.logits, w->vocab, B, w->vocab, HID, MA_EPI_NONE, s,
                 tc && !g_no_pdl)) return 1;
  return launch_sample(sa, s);
}

// Tensor-core GEMMs in the decoder: batches only (one sequence is a GEMV, HBM-bound on the canonical kernels), and only
// where ids are not promised bit for bit: sampling (logits tolerance, BASELINE configs 3-5) or MA_GEN_TC
static inline bool use_tc(int B, int do_sample, int flags) { return B > 1 && (do_sample || (flags & MA_GEN_TC)); }

static unsigned long long weights_hash(const ma_decoder_weights* w) {
  unsigned long long h = 1469598103934665603ull;  // FNV-1a over the pointer table: graphs bake the pointers in
  const unsigned char* pb = (const unsigned char*)w;
  for (size_t q = 0; q < sizeof(ma_decoder_weights); q++) h = (h ^ pb[q]) * 1099511628211ull;
  return h;
}

// Launch `enqueue` through the per-step graph cache (captured on first use of `key`).
template <class F>
static int launch_cached_graph(const GraphKey& key, cudaStream_t st, F&& enqueue) {
  auto it = g_graphs.find(key);
  if (it == g_graphs.end()) {
    cudaGraph_t graph = nullptr;
    if (cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
      set_error("cudaStreamBeginCapture: %s", cudaGetErrorString(cudaGetLastError()));
      return 1;
    }
    const unsigned long long before = g_launches.load();
    int erc = enqueue(st);
    const unsigned long long per_step = g_launches.load() - before;
    cudaError_t ce = cudaStreamEndCapture(st, &graph);
    if (erc || ce != cudaSuccess || !graph) {
      if (!erc) set_error("cudaStreamEndCapture: %s", cudaGetErrorString(ce));
      cudaGetLastError();
      return 1;
    }
    cudaGraphExec_t exec = nullptr;
    ce = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce != cudaSuccess) {
      set_error("cudaGraphInstantiate: %s", cudaGetErrorString(ce));
      return 1;
    }
    if (g_graphs.size() > 64) {
      for (auto& kvp : g_graphs) cudaGraphExecDestroy(kvp.second);
      g_graphs.clear();
      g_graph_launches.clear();
    }
    it = g_graphs.emplace(key, exec).first;
    g_launches -= per_step;  // the capture itself launched nothing
    g_graph_launches[exec] = per_step;
  }
  if (cudaGraphLaunch(it->second, st) != cudaSuccess) {
    set_error("cudaGraphLaunch: %s", cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  g_launches += g_graph_launches[it->second];
  return 0;
}

static void fill_sample_args(SampleArgs& sa, const ma_decoder_weights* w, const DecWs& ws, int B, int max_new,
                             const ma_sampling* sampling, int eos_id, int pad_id, int32_t* out_ids) {
  memset(&sa, 0, sizeof(sa));
  sa.logits = ws.logits; sa.vocab = w->vocab; sa.B = B; sa.max_new = max_new; sa.eos_id = eos_id; sa.pad_id = pad_id;
  sa.do_sample = sampling ? sampling->do_sample : 0;
  sa.top_k = sampling ? sampling->top_k : 0;
  sa.top_p = sampling ? sampling->top_p : 1.0f;
  sa.seed = sampling ? sampling->seed : 0;
  sa.s = ws.s; sa.out_ids = out_ids;
}

static int check_decode_args(const char* who, const ma_decoder_weights* w, int B, int tmax, int max_new) {
  if (w->n_layers > MA_MAX_LAYERS || w->vocab > 8195 + 61) {
    set_error("%s: n_layers=%d / vocab=%d unsupported", who, w->n_layers, w->vocab);
    return 1;
  }
  if (B <= 0 || max_new <= 0 || PREFIX + max_new > tmax) {
    set_error("%s: B=%d, tmax=%d < 257 + max_new=%d", who, B, tmax, max_new);
    return 1;
  }
  if (PREFIX + max_new + 2 > w->npos) {
    // meshanything.py:97-98: 18259 learned positions (+2 offset rows)
    set_error("%s: sequence of %d exceeds %d learned positions", who, PREFIX + max_new, w->npos - 2);
    return 1;
  }
  return 0;
}

}  // namespace ma

using namespace ma;

extern "C" {

int ma_abi_version(void) { return MA_ABI_VERSION; }
const char* ma_last_error(void) { return g_err; }
unsigned long long ma_launch_count(void) { return g_launches.load(); }

int ma_linear_f16(const void* W, const void* bias, const void* x, int ldx, void* y, int ldy, int M, int N, int K,
                  int epilogue, void* stream) {
  return launch_linear((const __half*)W, (const __half*)bias, (const __half*)x, ldx, (__half*)y, ldy, M, N, K,
                       epilogue, (cudaStream_t)stream);
}

size_t ma_linear_ws_scratch_bytes(void) { return linear_ws_scratch_bytes(); }
void ma_linear_ws_set_mode(int cluster) { linear_ws_set_mode(cluster); }

int ma_linear_ws_f16(const void* W, const void* bias, const void* x, int ldx, void* y, int ldy, int M, int N, int K,
                     int epilogue, void* scratch, void* stream) {
  return launch_linear_ws((const __half*)W, (const __half*)bias, (const __half*)x, ldx, (__half*)y, ldy, M, N, K,
                          epilogue, scratch, (cudaStream_t)stream);
}

int ma_layernorm(const float* x, const void* res16, const float* gamma, const float* beta, float eps, int M, int W,
                 float* out32, void* out16, void* stream) {
  return launch_layernorm(x, (const __half*)res16, gamma, beta, eps, M, W, out32, (__half*)out16,
                          (cudaStream_t)stream);
}

size_t ma_attention_scratch_bytes(int M, int H, int max_keys) { return attention_scratch_bytes(M, H, max_keys); }

int ma_attention_f16(const void* q, int ldq, const void* K, const void* V, long T, int H, const int* slots,
                     const int* nkeys, int max_keys, int M, float scale, void* out, int ldo, void* scratch,
                     void* stream) {
  if (M > 65535) {
    set_error("ma_attention_f16: M=%d exceeds 65535 rows per call", M);
    return 1;
  }
  return launch_attention((const __half*)q, ldq, (const __half*)K, (const __half*)V, T, H, 1, slots, nkeys, max_keys, M,
                          scale, (__half*)out, ldo, scratch, (cudaStream_t)stream);
}

int ma_attention_decode_f16(const void* qkv, int ldq, void* K, void* V, long T, const int* nkeys, int max_keys, int M,
                            float scale, void* out, int ldo, void* scratch, void* stream) {
  if (!qkv || !K || !V || !nkeys || !out || !scratch || M < 1 || max_keys < 1 || max_keys > T || ldq < 3 * HID) {
    set_error("ma_attention_decode_f16: bad arguments (M=%d, max_keys=%d, T=%ld, ldq=%d)", M, max_keys, T, ldq);
    return 1;
  }
  return launch_attention_decode((const __half*)qkv, ldq, (__half*)K, (__half*)V, T, nkeys, max_keys, M, scale,
                                 (__half*)out, ldo, scratch, false, (cudaStream_t)stream);
}

int ma_sample_tokens(const void* logits, int B, int vocab, const ma_sampling* sampling, int32_t* out_tokens,
                     int32_t* out_support, void* stream) {
  if (!logits || !out_tokens || B < 1 || vocab < 1) {
    set_error("ma_sample_tokens: bad arguments");
    return 1;
  }
  SampleArgs sa;
  memset(&sa, 0, sizeof(sa));
  sa.logits = (const __half*)logits; sa.vocab = vocab; sa.B = B; sa.max_new = 1; sa.eos_id = -1; sa.pad_id = -1;
  sa.do_sample = sampling ? sampling->do_sample : 0;
  sa.top_k = sampling ? sampling->top_k : 0;
  sa.top_p = sampling ? sampling->top_p : 1.0f;
  sa.seed = sampling ? sampling->seed : 0;
  sa.first = 1; sa.token_out = out_tokens; sa.support_out = out_support;
  return launch_sample(sa, (cudaStream_t)stream);
}

size_t ma_kv_cache_bytes(int n_layers, int B, int tmax) {
  return (size_t)n_layers * 2 * B * NHEAD * (size_t)tmax * HD * sizeof(__half);
}

size_t ma_decoder_workspace_bytes(int B, int tmax) { return carve(nullptr, B, tmax, 8195 + 61).total; }

int ma_decode_generate(const ma_decoder_weights* w, const float* prefix, int B, int tmax, int max_new,
                       const ma_sampling* sampling, int eos_id, int pad_id, void* kv, void* ws_, int32_t* out_ids,
                       int32_t* out_lens, const int32_t* forced_ids, void* logits_out, int flags, void* stream) {
  if (!w || !prefix || !kv || !ws_ || !out_ids || B <= 0 || max_new <= 0) {
    set_error("ma_decode_generate: bad arguments");
    return 1;
  }
  if (check_decode_args("ma_decode_generate", w, B, tmax, max_new)) return 1;
  std::lock_guard<std::mutex> lock(g_mu);
  if (ensure_globals()) return 1;
  cudaStream_t user = (cudaStream_t)stream;
  cudaStream_t st = g_stream;  // graph capture is illegal on the legacy default stream: always run on our own
  cudaEventRecord(g_ev_in, user);
  cudaStreamWaitEvent(st, g_ev_in, 0);

  const long T = tmax;
  DecWs ws = carve(ws_, B, tmax, 8195 + 61);
  cudaMemsetAsync(ws.attn_scratch, 0, ws.attn_scratch_bytes, st);
  cudaMemsetAsync(ws.attn_scratch_pre, 0, ws.attn_scratch_pre_bytes, st);
  cudaMemsetAsync(ws.fast, 0, fast_workspace_bytes(), st);
  if (launch_fill_i32(out_ids, pad_id, (long)B * max_new, st)) return 1;

  SampleArgs sa;
  fill_sample_args(sa, w, ws, B, max_new, sampling, eos_id, pad_id, out_ids);
  sa.first = 1; sa.forced = forced_ids; sa.logits_out = (__half*)logits_out;
  sa.all_done = ws.all_done;

  const bool tc = use_tc(B, sa.do_sample, flags);
  if (tc) cudaMemsetAsync(ws.tc_scratch, 0, linear_ws_scratch_bytes(), st);   // tickets start at zero
  const bool fast = (B == 1) && !(flags & MA_GEN_NO_FAST);
  if (fast) sa.nkeys_next = fast_nkeys_ptr(ws.fast);

  // ---- prefill: 257 prefix rows per sequence, PREFILL_SEQS sequences per pass
  for (int b0 = 0; b0 < B; b0 += PREFILL_SEQS) {
    const int nb = std::min(PREFILL_SEQS, B - b0), M = nb * PREFIX;
    if (launch_embed_prefix(w, prefix + (size_t)b0 * PREFIX * HID, nb, ws.hres, ws.x16, ws.nkeys, st)) return 1;
    if (run_layers(w, ws, kv, B, T, M, PREFIX, b0, PREFIX, st, tc)) return 1;
    if (launch_gather_rows(ws.x16, HID, PREFIX - 1, PREFIX, nb, ws.lastx16 + (size_t)b0 * HID, st)) return 1;
  }
  if (dec_linear(tc, ws, w->lm_head, nullptr, ws.lastx16, HID, ws.logits, w->vocab, B, w->vocab, HID, MA_EPI_NONE, st))
    return 1;
  if (launch_sample(sa, st)) return 1;
  sa.first = 0;
  sa.nkeys_next = nullptr;

  // ---- decode: one step per generated token

  const bool use_graph = !(flags & MA_GEN_NO_GRAPH);
  const bool early = !(flags & MA_GEN_NO_EARLY_EXIT) && !forced_ids;
  const int CHECK_EVERY = 64;
  const unsigned long long whash = use_graph ? weights_hash(w) : 0;  // the struct is read at capture time
  bool flag_pending = false;
  int rc = 0;
  for (int i = 1; i < max_new && rc == 0; i++) {
    const int ctx = PREFIX + i;                          // keys visible to this step (all rows advance together)
    const int bucket = (ctx + 1023) / 1024;              // attention grid size class
    const int max_keys = std::min(tmax, bucket * 1024);
    auto enqueue = [&](cudaStream_t s) -> int {
      if (fast)
        return fast_step_enqueue(w, ws.s, tmax, max_keys, (__half*)kv, ws.fast, sa, !(flags & MA_GEN_NO_PDL), s);
      return enqueue_batched_step(w, ws, kv, B, T, max_keys, sa, s, tc);
    };
    if (!use_graph) {
      rc = enqueue(st);
    } else {
      GraphKey key;
      memset(&key, 0, sizeof(key));
      key.w = w; key.kv = kv; key.ws = ws_; key.out_ids = out_ids; key.forced = forced_ids; key.logits_out = logits_out;
      key.B = B; key.tmax = tmax; key.max_new = max_new; key.bucket = bucket; key.flags = flags;
      key.do_sample = sa.do_sample; key.top_k = sa.top_k; key.eos = eos_id; key.pad = pad_id; key.top_p = sa.top_p;
      key.seed = sa.do_sample ? sa.seed : 0;   // greedy graphs do not depend on the seed
      key.whash = whash;
      key.ws_mode = linear_ws_mode();
      if (launch_cached_graph(key, st, enqueue)) return 1;
    }
    if (early && (i % CHECK_EVERY) == 0) {
      // lagged, non-blocking early-exit poll: look at the flag copied CHECK_EVERY steps ago
      if (flag_pending && cudaEventQuery(g_ev_flag) == cudaSuccess) {
        if (*g_flag_host == 1) break;
        flag_pending = false;
      }
      if (!flag_pending) {
        cudaMemcpyAsync(g_flag_host, ws.all_done, sizeof(int), cudaMemcpyDeviceToHost, st);
        cudaEventRecord(g_ev_flag, st);
        flag_pending = true;
      }
    }
  }
  if (rc) return rc;
  if (out_lens) cudaMemcpyAsync(out_lens, ws.s.lens, sizeof(int) * B, cudaMemcpyDeviceToDevice, st);
  cudaEventRecord(g_ev_out, st);
  cudaStreamWaitEvent(user, g_ev_out, 0);
  return check_launch("ma_decode_generate") ? 0 : 1;
}


// ---- continuous batching (SURVEY.md section 8(f)2): B cache slots, each running its own sequence ------------------
// The host scheduler (meshanything_b200/scheduler.py) refills a slot as soon as its sequence has finished instead of
// padding it until the longest sequence of the batch ends (HF generate semantics, a10).  Rows never interact and the
// kernels are batch-invariant, so every sequence gets bit-identical ids to a solo ma_decode_generate.

static int slots_enter(void* stream, cudaStream_t* st) {
  if (ensure_globals()) return 1;
  cudaEventRecord(g_ev_in, (cudaStream_t)stream);
  cudaStreamWaitEvent(g_stream, g_ev_in, 0);
  *st = g_stream;
  return 0;
}
static int slots_leave(void* stream, const char* who) {
  cudaEventRecord(g_ev_out, g_stream);
  cudaStreamWaitEvent((cudaStream_t)stream, g_ev_out, 0);
  return check_launch(who) ? 0 : 1;
}

int ma_decode_slots_init(int B, int tmax, int pad_id, void* ws_, void* stream) {
  if (!ws_ || B <= 0 || tmax < PREFIX + 1) {
    set_error("ma_decode_slots_init: bad arguments");
    return 1;
  }
  std::lock_guard<std::mutex> lock(g_mu);
  cudaStream_t st;
  if (slots_enter(stream, &st)) return 1;
  DecWs ws = carve(ws_, B, tmax, 8195 + 61);
  cudaMemsetAsync(ws.attn_scratch, 0, ws.attn_scratch_bytes, st);
  cudaMemsetAsync(ws.attn_scratch_pre, 0, ws.attn_scratch_pre_bytes, st);
  cudaMemsetAsync(ws.tc_scratch, 0, linear_ws_scratch_bytes(), st);
  // every slot starts free: finished, nothing generated, a valid (pad) token at a valid position
  if (launch_fill_i32(ws.s.pos, PREFIX, B, st) || launch_fill_i32(ws.s.gen, 0, B, st) ||
      launch_fill_i32(ws.s.tok, pad_id, B, st) || launch_fill_i32(ws.s.finished, 1, B, st) ||
      launch_fill_i32(ws.s.lens, 0, B, st) || launch_fill_i32(ws.s.sid, 0, B, st)) return 1;
  return slots_leave(stream, "ma_decode_slots_init");
}

int ma_decode_slot_stream(int slot, int B, int tmax, int stream_id, void* ws_, void* stream) {
  if (!ws_ || slot < 0 || slot >= B) {
    set_error("ma_decode_slot_stream: bad arguments (slot %d of %d)", slot, B);
    return 1;
  }
  std::lock_guard<std::mutex> lock(g_mu);
  cudaStream_t st;
  if (slots_enter(stream, &st)) return 1;
  DecWs ws = carve(ws_, B, tmax, 8195 + 61);
  if (launch_fill_i32(ws.s.sid + slot, stream_id, 1, st)) return 1;
  return slots_leave(stream, "ma_decode_slot_stream");
}

int ma_decode_slots_seek(int B, int tmax, int pos, int gen, int tok, void* ws_, void* stream) {
  if (!ws_ || B <= 0 || pos < PREFIX || pos >= tmax || gen < 1) {
    set_error("ma_decode_slots_seek: bad arguments (pos %d of tmax %d)", pos, tmax);
    return 1;
  }
  std::lock_guard<std::mutex> lock(g_mu);
  cudaStream_t st;
  if (slots_enter(stream, &st)) return 1;
  DecWs ws = carve(ws_, B, tmax, 8195 + 61);
  if (launch_fill_i32(ws.s.pos, pos, B, st) || launch_fill_i32(ws.s.gen, gen, B, st) ||
      launch_fill_i32(ws.s.tok, tok, B, st) || launch_fill_i32(ws.s.finished, 0, B, st) ||
      launch_fill_i32(ws.s.lens, gen, B, st)) return 1;
  return slots_leave(stream, "ma_decode_slots_seek");
}

int ma_decode_slot_prefill(const ma_decoder_weights* w, const float* prefix, int slot, int B, int tmax, int max_new,
                           const ma_sampling* sampling, int eos_id, int pad_id, void* kv, void* ws_, int32_t* out_ids,
                           void* stream) {
  if (!w || !prefix || !kv || !ws_ || !out_ids || slot < 0 || slot >= B) {
    set_error("ma_decode_slot_prefill: bad arguments (slot %d of %d)", slot, B);
    return 1;
  }
  if (check_decode_args("ma_decode_slot_prefill", w, B, tmax, max_new)) return 1;
  std::lock_guard<std::mutex> lock(g_mu);
  cudaStream_t st;
  if (slots_enter(stream, &st)) return 1;
  const long T = tmax;
  DecWs ws = carve(ws_, B, tmax, 8195 + 61);
  if (launch_fill_i32(out_ids + (size_t)slot * max_new, pad_id, max_new, st)) return 1;
  if (launch_embed_prefix(w, prefix, 1, ws.hres, ws.x16, ws.nkeys, st)) return 1;
  const bool tc = use_tc(B, sampling ? sampling->do_sample : 0, 0);
  if (run_layers(w, ws, kv, B, T, PREFIX, PREFIX, slot, PREFIX, st, tc)) return 1;
  __half* last = ws.lastx16 + (size_t)slot * HID;
  if (launch_gather_rows(ws.x16, HID, PREFIX - 1, PREFIX, 1, last, st)) return 1;
  if (dec_linear(tc, ws, w->lm_head, nullptr, last, HID, ws.logits + (size_t)slot * w->vocab, w->vocab, 1, w->vocab, HID,
                 MA_EPI_NONE, st)) return 1;
  SampleArgs sa;
  fill_sample_args(sa, w, ws, B, max_new, sampling, eos_id, pad_id, out_ids);
  sa.first = 1; sa.row0 = slot; sa.nrows = 1; sa.slots = 1;
  if (launch_sample(sa, st)) return 1;
  return slots_leave(stream, "ma_decode_slot_prefill");
}

int ma_decode_slots_step(const ma_decoder_weights* w, int B, int tmax, int max_new, int n_steps, int max_ctx,
                         const ma_sampling* sampling, int eos_id, int pad_id, void* kv, void* ws_, int32_t* out_ids,
                         int flags, void* stream) {
  if (!w || !kv || !ws_ || !out_ids || n_steps < 0 || max_ctx < PREFIX + 1) {
    set_error("ma_decode_slots_step: bad arguments");
    return 1;
  }
  if (check_decode_args("ma_decode_slots_step", w, B, tmax, max_new)) return 1;
  std::lock_guard<std::mutex> lock(g_mu);
  cudaStream_t st;
  if (slots_enter(stream, &st)) return 1;
  const long T = tmax;
  DecWs ws = carve(ws_, B, tmax, 8195 + 61);
  SampleArgs sa;
  fill_sample_args(sa, w, ws, B, max_new, sampling, eos_id, pad_id, out_ids);
  sa.slots = 1;
  const bool use_graph = !(flags & MA_GEN_NO_GRAPH);
  const unsigned long long whash = use_graph ? weights_hash(w) : 0;
  for (int i = 0; i < n_steps; i++) {
    const int ctx = std::min(tmax, max_ctx + i);   // upper bound of the keys any live slot sees at this step
    const int bucket = (ctx + 1023) / 1024;
    const int max_keys = std::min(tmax, bucket * 1024);
    auto enqueue = [&](cudaStream_t s) -> int {
      return enqueue_batched_step(w, ws, kv, B, T, max_keys, sa, s, use_tc(B, sa.do_sample, flags));
    };
    if (!use_graph) {
      if (enqueue(st)) return 1;
    } else {
      GraphKey key;
      memset(&key, 0, sizeof(key));
      key.w = w; key.kv = kv; key.ws = ws_; key.out_ids = out_ids;
      key.B = B; key.tmax = tmax; key.max_new = max_new; key.bucket = bucket; key.flags = flags; key.mode = 1;
      key.do_sample = sa.do_sample; key.top_k = sa.top_k; key.eos = eos_id; key.pad = pad_id; key.top_p = sa.top_p;
      key.seed = sa.do_sample ? sa.seed : 0;   // greedy graphs do not depend on the seed
      key.whash = whash;
      key.ws_mode = linear_ws_mode();
      if (launch_cached_graph(key, st, enqueue)) return 1;
    }
  }
  return slots_leave(stream, "ma_decode_slots_step");
}

int ma_decode_slots_poll(int B, int tmax, void* ws_, int32_t* finished_host, int32_t* lens_host, void* stream) {
  if (!ws_ || !finished_host || !lens_host || B <= 0) {
    set_error("ma_decode_slots_poll: bad arguments");
    return 1;
  }
  std::lock_guard<std::mutex> lock(g_mu);
  cudaStream_t st;
  if (slots_enter(stream, &st)) return 1;
  DecWs ws = carve(ws_, B, tmax, 8195 + 61);
  cudaMemcpyAsync(finished_host, ws.s.finished, sizeof(int) * B, cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(lens_host, ws.s.lens, sizeof(int) * B, cudaMemcpyDeviceToHost, st);
  if (cudaStreamSynchronize(st) != cudaSuccess) {
    set_error("ma_decode_slots_poll: %s", cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  return slots_leave(stream, "ma_decode_slots_poll");
}


int ma_decode_persistent_supported(void) { return 0; }

}  // extern "C"
