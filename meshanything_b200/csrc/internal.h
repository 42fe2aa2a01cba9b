// internal.h -- host-side launch helpers shared by the translation units of libmeshanything_b200.so
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/meshanything_b200.h"

namespace ma {

constexpr int HID = 1024;
constexpr int NHEAD = 16;
constexpr int HD = 64;
constexpr int FFN = 4096;
constexpr int PREFIX = 257;
constexpr int QKV = 3 * HID;

// per-sequence generation state, device resident (arrays of length B inside the workspace)
struct SeqState {
  int* pos;       // cached positions (absolute index of the next token)
  int* gen;       // tokens generated so far
  int* tok;       // last generated token (input of the next step)
  int* finished;  // eos seen
  int* lens;      // tokens up to and including eos (or gen)
  int* sid;       // continuous batching: Philox stream of the sequence in this slot (its index in the queue), so that
                  // two shapes that pass through the same slot do not draw the same uniforms
};

void set_error(const char* fmt, ...);
void count_launch(int n = 1);
bool check_launch(const char* what);

// gemm_canon.cu
int launch_linear(const __half* W, const __half* bias, const __half* x, int ldx, __half* y, int ldy, int M, int N,
                  int K, int epi, cudaStream_t st);

// gemm_tc.cu (wgmma + TMA; tolerance-checked stages only)
// attention_tc.cu (wgmma flash attention for the tolerance-compared stages)
bool attention_tc_supported(int ldq, int ldo, long T, long Tpad, int nkeys, const void* q, const void* K, const void* Vt,
                            const void* out);
int launch_attention_tc(const __half* q, int ldq, const __half* K, const __half* Vt, long T, long Tpad, int H,
                        int rows_per_slot, int n_slots, int nkeys, float scale, __half* out, int ldo, cudaStream_t st);
int launch_scatter_heads_t(const __half* src, int ld, int col0, int head_stride, int H, int n, long Tpad, int n_slots,
                           __half* dst, cudaStream_t st);

bool linear_tc_supported(int M, int N, int K, int ldx, int ldy, const void* x, const void* W, const void* y);
int launch_linear_tc(const __half* W, const __half* bias, const __half* x, int ldx, __half* y, int ldy, int M, int N,
                     int K, int epi, cudaStream_t st);

// gemm_ws.cu (wgmma weight-streaming GEMM for M <= 128 rows: batched decode steps under a tolerance)
size_t linear_ws_scratch_bytes();
void linear_ws_set_mode(int cluster);
int linear_ws_mode();   // 1: K slices reduced over distributed shared memory (default), 0: L2 + tickets
bool linear_ws_supported(int M, int N, int K, int ldx, const void* x, const void* W);
int launch_linear_ws(const __half* W, const __half* bias, const __half* x, int ldx, __half* y, int ldy, int M, int N,
                     int K, int epi, void* scratch, cudaStream_t st, bool pdl = false);

// attention.cu
size_t attention_scratch_bytes(int M, int H, int max_keys);
// decode attention of M cache slots (one query row each) + append of the current k / v (attention_stream.cu)
int launch_attention_decode(const __half* qkv, int ldq, __half* K, __half* V, long T, const int* nkeys, int max_keys,
                            int M, float scale, __half* out, int ldo, void* scratch, bool pdl, cudaStream_t st);
int launch_attention(const __half* q, int ldq, const __half* K, const __half* V, long T, int H, int rows_per_slot,
                     const int* slots, const int* nkeys, int max_keys, int M, float scale, __half* out, int ldo,
                     void* scratch, cudaStream_t st);
// api.cu: MA_B200_NO_STREAM_ATTN=1 -- decode attention on kv_append_kernel + attention_kernel instead
bool no_stream_attn();

// elementwise.cu
int launch_layernorm(const float* x, const __half* res16, const float* gamma, const float* beta, float eps, int M,
                     int W, float* out32, __half* out16, cudaStream_t st, bool pdl = false);
int launch_embed_prefix(const ma_decoder_weights* w, const float* prefix, int B, float* hres, __half* x16, int* nkeys,
                        cudaStream_t st);
int launch_embed_tokens(const ma_decoder_weights* w, SeqState s, int B, float* hres, __half* x16, int* nkeys,
                        cudaStream_t st);
int launch_kv_append(const __half* qkv, int M, int rows_per_slot, const int* nkeys, __half* kc, __half* vc, long T,
                     cudaStream_t st);
int launch_gather_rows(const __half* src, int ld, int row0, int stride, int B, __half* dst, cudaStream_t st);
struct SampleArgs {
  const __half* logits;  // [B][vocab]
  int vocab, B, max_new, eos_id, pad_id;
  int do_sample, top_k;
  float top_p;
  unsigned long long seed;
  SeqState s;
  int first;             // 1: this is the pick after the prefill (initialises the state)
  int32_t* out_ids;      // [B][max_new]
  const int32_t* forced; // [B][max_new] or null
  __half* logits_out;    // [max_new][B][vocab] or null
  int* all_done;         // device flag: 1 when every row finished
  int* nkeys_next;       // optional [B]: keys visible to the next step (pos + 1), for the batch-1 fast path
  int32_t* support_out;  // test hook [B][256]: token ids that survive top-k/top-p (descending), -1 padded
  int32_t* token_out;    // test hook [B]: the picked token
  int row0, nrows;       // rows [row0, row0 + nrows) are processed (nrows = 0: all B rows)
  int slots;             // 1: continuous batching -- finished rows are frozen (no state advance, no output write)
                         //    and a row also finishes when it reaches max_new tokens
};
int launch_sample(const SampleArgs& a, cudaStream_t st);
int launch_fill_i32(int32_t* p, int v, long n, cudaStream_t st);

// decode_fast.cu (batch-1 fused GEMV path)
int* fast_nkeys_ptr(void* fast_ws);
size_t fast_workspace_bytes();
// max_keys: the attention grid covers this many keys; no step of the launch may see more
int fast_step_enqueue(const ma_decoder_weights* w, SeqState s, int tmax, int max_keys, __half* kv, void* fast_ws,
                      const SampleArgs& sa, bool pdl, cudaStream_t st);

}  // namespace ma
