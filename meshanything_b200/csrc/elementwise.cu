// elementwise.cu -- embeddings, residual + LayerNorm, KV append, token pick and bookkeeping.
#include "canon.cuh"
#include "internal.h"

namespace ma {

// ---------------------------------------------------------------- residual + LayerNorm
// One CTA per row, blockDim = W/4, thread t owns elements 4t..4t+3 (canonical block sum).
__global__ void layernorm_kernel(const float* __restrict__ x, const __half* __restrict__ res16,
                                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int W,
                                 float* __restrict__ out32, __half* __restrict__ out16) {
  __shared__ float red[8];
  const long row = blockIdx.x;
  const int t = threadIdx.x;
  pdl_trigger();   // the next kernel (a GEMM: weight tiles first) may start its prologue now
  pdl_wait();      // no-op unless launched as a programmatic dependent; x / res16 come from the previous kernel
  float v[4];
  if (x) {
    const float4 xv = *reinterpret_cast<const float4*>(x + row * W + 4 * t);
    v[0] = xv.x; v[1] = xv.y; v[2] = xv.z; v[3] = xv.w;
  } else {
    v[0] = v[1] = v[2] = v[3] = 0.0f;
  }
  if (res16) {
    const uint2 u = *reinterpret_cast<const uint2*>(res16 + row * W + 4 * t);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
    const float2 a = __half22float2(h[0]), b = __half22float2(h[1]);
    if (x) {
      v[0] = fadd(v[0], a.x); v[1] = fadd(v[1], a.y); v[2] = fadd(v[2], b.x); v[3] = fadd(v[3], b.y);
    } else {
      v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
    }
  }
  layernorm4(v, *reinterpret_cast<const float4*>(gamma + 4 * t), *reinterpret_cast<const float4*>(beta + 4 * t), eps, W,
             red);
  if (out32) *reinterpret_cast<float4*>(out32 + row * W + 4 * t) = make_float4(v[0], v[1], v[2], v[3]);
  if (out16) {
    __half2 h0 = __floats2half2_rn(v[0], v[1]), h1 = __floats2half2_rn(v[2], v[3]);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&h0);
    u.y = *reinterpret_cast<uint32_t*>(&h1);
    *reinterpret_cast<uint2*>(out16 + row * W + 4 * t) = u;
  }
}

int launch_layernorm(const float* x, const __half* res16, const float* gamma, const float* beta, float eps, int M,
                     int W, float* out32, __half* out16, cudaStream_t st, bool pdl) {
  if (M <= 0) return 0;
  if (W % 128 != 0 || W > 1024 || (!x && !res16)) {
    set_error("ma_layernorm: unsupported width %d or no input", W);
    return 1;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(M);
  cfg.blockDim = dim3(W / 4);
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaLaunchKernelEx(&cfg, layernorm_kernel, x, res16, gamma, beta, eps, W, out32, out16);
  count_launch();
  return check_launch("layernorm_kernel") ? 0 : 1;
}

// ---------------------------------------------------------------- embeddings
__device__ __forceinline__ void store_row4(float* hres, __half* x16, long row, int t, const float* v) {
  *reinterpret_cast<float4*>(hres + row * HID + 4 * t) = make_float4(v[0], v[1], v[2], v[3]);
  __half2 h0 = __floats2half2_rn(v[0], v[1]), h1 = __floats2half2_rn(v[2], v[3]);
  uint2 u;
  u.x = *reinterpret_cast<uint32_t*>(&h0);
  u.y = *reinterpret_cast<uint32_t*>(&h1);
  *reinterpret_cast<uint2*>(x16 + row * HID + 4 * t) = u;
}

// step 0 of generate(): hidden = (prefix + cond_embed[0]) + embed_positions[s + 2]
// (shape_opt.py:331-337,359-364; OPTLearnedPositionalEmbedding offset 2)
__global__ void embed_prefix_kernel(const float* __restrict__ prefix, const float* __restrict__ cond,
                                    const float* __restrict__ pos, float* __restrict__ hres, __half* __restrict__ x16,
                                    int* __restrict__ nkeys) {
  const long row = blockIdx.x;
  const int s = (int)(row % PREFIX), t = threadIdx.x;
  const float4 p = *reinterpret_cast<const float4*>(prefix + row * HID + 4 * t);
  const float4 c = *reinterpret_cast<const float4*>(cond + 4 * t);
  const float4 e = *reinterpret_cast<const float4*>(pos + (long)(s + 2) * HID + 4 * t);
  float v[4] = {fadd(fadd(p.x, c.x), e.x), fadd(fadd(p.y, c.y), e.y), fadd(fadd(p.z, c.z), e.z),
                fadd(fadd(p.w, c.w), e.w)};
  store_row4(hres, x16, row, t, v);
  if (t == 0) nkeys[row] = s + 1;
}

int launch_embed_prefix(const ma_decoder_weights* w, const float* prefix, int B, float* hres, __half* x16, int* nkeys,
                        cudaStream_t st) {
  embed_prefix_kernel<<<B * PREFIX, HID / 4, 0, st>>>(prefix, w->cond, w->pos, hres, x16, nkeys);
  count_launch();
  return check_launch("embed_prefix_kernel") ? 0 : 1;
}

// Input embedding of one generated token (shape_opt.py:318-328,237-245,448-460):
//   hidden = (((X + F) + C) + P),  X = extra_embeds[id] or fp16 tok_table[id-3],
//   F = token_embed_positions[id or (gen-2) mod 9 + 3], C = cond_embed[1], P = embed_positions[pos+2]
__device__ __forceinline__ void token_embedding4(const ma_decoder_weights& w, int tok, int gen, int pos, int t,
                                                 float* v) {
  float4 X;
  int fidx;
  if (tok < 3) {
    X = *reinterpret_cast<const float4*>(w.extra + (long)tok * HID + 4 * t);
    fidx = tok;
  } else {
    const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const __half*>(w.tok_table) +
                                                    (long)(tok - 3) * HID + 4 * t);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
    const float2 a = __half22float2(h[0]), b = __half22float2(h[1]);
    X = make_float4(a.x, a.y, b.x, b.y);
    int r = (gen - 2) % 9;
    if (r < 0) r += 9;  // torch remainder is floored
    fidx = r + 3;
  }
  const float4 F = *reinterpret_cast<const float4*>(w.tok_pos + (long)fidx * HID + 4 * t);
  const float4 C = *reinterpret_cast<const float4*>(w.cond + HID + 4 * t);
  const float4 P = *reinterpret_cast<const float4*>(w.pos + (long)(pos + 2) * HID + 4 * t);
  v[0] = fadd(fadd(fadd(X.x, F.x), C.x), P.x);
  v[1] = fadd(fadd(fadd(X.y, F.y), C.y), P.y);
  v[2] = fadd(fadd(fadd(X.z, F.z), C.z), P.z);
  v[3] = fadd(fadd(fadd(X.w, F.w), C.w), P.w);
}

__global__ void embed_tokens_kernel(ma_decoder_weights w, SeqState s, float* __restrict__ hres,
                                    __half* __restrict__ x16, int* __restrict__ nkeys) {
  const int b = blockIdx.x, t = threadIdx.x;
  const int tok = s.tok[b], gen = s.gen[b], pos = s.pos[b];
  float v[4];
  token_embedding4(w, tok, gen, pos, t, v);
  store_row4(hres, x16, b, t, v);
  if (t == 0) nkeys[b] = pos + 1;
}

int launch_embed_tokens(const ma_decoder_weights* w, SeqState s, int B, float* hres, __half* x16, int* nkeys,
                        cudaStream_t st) {
  embed_tokens_kernel<<<B, HID / 4, 0, st>>>(*w, s, hres, x16, nkeys);
  count_launch();
  return check_launch("embed_tokens_kernel") ? 0 : 1;
}

// ---------------------------------------------------------------- KV append (no torch.cat: SURVEY 2.2 G3)
// qkv [M][3072]: k = cols 1024..2047, v = cols 2048..3071 ; cache [slot][head][T][64]
__global__ void kv_append_kernel(const __half* __restrict__ qkv, int rows_per_slot, const int* __restrict__ nkeys,
                                 __half* __restrict__ kc, __half* __restrict__ vc, long T) {
  const long m = blockIdx.x;
  const int slot = (int)(m / rows_per_slot), pos = nkeys[m] - 1;
  const int t = threadIdx.x;  // 256 threads: 0..127 K, 128..255 V ; each moves 16 bytes
  const int which = t >> 7, e = (t & 127) * 8, head = e >> 6, d = e & 63;
  const uint4 u = *reinterpret_cast<const uint4*>(qkv + m * QKV + HID * (1 + which) + e);
  __half* dst = (which ? vc : kc) + (((long)slot * NHEAD + head) * T + pos) * HD + d;
  *reinterpret_cast<uint4*>(dst) = u;
}

int launch_kv_append(const __half* qkv, int M, int rows_per_slot, const int* nkeys, __half* kc, __half* vc, long T,
                     cudaStream_t st) {
  kv_append_kernel<<<M, 256, 0, st>>>(qkv, rows_per_slot, nkeys, kc, vc, T);
  count_launch();
  return check_launch("kv_append_kernel") ? 0 : 1;
}

// dst[b][0..1023] = src[(row0 + b*stride)][0..1023]
__global__ void gather_rows_kernel(const __half* __restrict__ src, int ld, int row0, int stride,
                                   __half* __restrict__ dst) {
  const int b = blockIdx.x, t = threadIdx.x;  // 128 threads x 16 bytes
  *reinterpret_cast<uint4*>(dst + (long)b * HID + 8 * t) =
      *reinterpret_cast<const uint4*>(src + (long)(row0 + (long)b * stride) * ld + 8 * t);
}
int launch_gather_rows(const __half* src, int ld, int row0, int stride, int B, __half* dst, cudaStream_t st) {
  gather_rows_kernel<<<B, 128, 0, st>>>(src, ld, row0, stride, dst);
  count_launch();
  return check_launch("gather_rows_kernel") ? 0 : 1;
}

__global__ void fill_i32_kernel(int32_t* p, int v, long n) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
int launch_fill_i32(int32_t* p, int v, long n, cudaStream_t st) {
  if (n <= 0) return 0;
  fill_i32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p, v, n);
  count_launch();
  return check_launch("fill_i32_kernel") ? 0 : 1;
}

// ---------------------------------------------------------------- token pick + bookkeeping
// Philox4x32-10 keyed by (seed, row, step): one uniform in [0,1) per pick.
__device__ __forceinline__ uint32_t mulhilo(uint32_t a, uint32_t b, uint32_t* hi) {
  const unsigned long long p = (unsigned long long)a * b;
  *hi = (uint32_t)(p >> 32);
  return (uint32_t)p;
}
__device__ float philox_uniform(unsigned long long seed, uint32_t row, uint32_t step) {
  uint32_t c0 = step, c1 = row, c2 = 0x4d455348u, c3 = 0x414e5954u;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int i = 0; i < 10; i++) {
    uint32_t hi0, hi1;
    const uint32_t lo0 = mulhilo(0xD2511F53u, c0, &hi0), lo1 = mulhilo(0xCD9E8D57u, c2, &hi1);
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return (float)(c0 >> 8) * (1.0f / 16777216.0f);
}

// (value, index) order used by the greedy pick: larger value first, lower index on ties
__device__ __forceinline__ bool better(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

constexpr int SAMPLE_THREADS = 256;
constexpr int KEEP_MAX = 256;  // capacity of the kept set (top_k plus ties at the threshold)

// order-preserving 16-bit key of an fp16 value: larger value <=> larger key (-0 < +0, irrelevant here)
__device__ __forceinline__ unsigned key16(__half h) {
  const unsigned u = __half_as_ushort(h);
  return (u & 0x8000u) ? (~u & 0xffffu) : (u | 0x8000u);
}

// One CTA per row.  Greedy: argmax of the fp16 logits (HF 4.39.3 _greedy_search keeps fp16), lowest index on ties.
// Sampling = HF _sample with TopKLogitsWarper(top_k) then TopPLogitsWarper(top_p) (logits_process.py):
//   1. keep every logit >= the k-th largest VALUE (ties at the threshold are kept, as `scores < kth` removes
//      only strictly smaller ones): exact k-th value by a two-level radix select on the 16-bit keys;
//   2. softmax over the kept set; in ascending order drop tokens while the cumulative probability is <= 1 - top_p,
//      always keeping the largest;
//   3. inverse-CDF draw over the survivors (descending value, higher index first) with one Philox uniform.
__global__ void __launch_bounds__(SAMPLE_THREADS) sample_kernel(SampleArgs a) {
  __shared__ float sv[SAMPLE_THREADS];
  __shared__ int si[SAMPLE_THREADS];
  __shared__ int hist[256];
  __shared__ float keepv[KEEP_MAX], sortv[KEEP_MAX];
  __shared__ int keepi[KEEP_MAX], sorti[KEEP_MAX];
  __shared__ int s_bin, s_above;
  extern __shared__ unsigned short keys[];  // [vocab] order-preserving keys of the row (sampling only)
  const int b = blockIdx.x + a.row0, tid = threadIdx.x;
  const __half* lg = a.logits + (long)b * a.vocab;
  const int gen = a.first ? 0 : a.s.gen[b];
  if (a.slots && !a.first && a.s.finished[b]) return;  // frozen slot (uniform per CTA): nothing to pick or advance

  if (a.logits_out) {
    __half* dst = a.logits_out + ((long)gen * a.B + b) * a.vocab;
    for (int i = tid; i < a.vocab; i += SAMPLE_THREADS) dst[i] = lg[i];
  }

  int n_keep = 1;
  if (!a.do_sample) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = tid; i < a.vocab; i += SAMPLE_THREADS) {
      const float v = __half2float(lg[i]);
      if (better(v, i, bv, bi)) { bv = v; bi = i; }
    }
    sv[tid] = bv; si[tid] = bi;
    __syncthreads();
    for (int s = SAMPLE_THREADS / 2; s > 0; s >>= 1) {
      if (tid < s && better(sv[tid + s], si[tid + s], sv[tid], si[tid])) { sv[tid] = sv[tid + s]; si[tid] = si[tid + s]; }
      __syncthreads();
    }
    if (tid == 0) { sortv[0] = sv[0]; sorti[0] = si[0]; }
    __syncthreads();
  } else {
    const int k = min(a.top_k, a.vocab);
    // stage the row's keys once (coalesced); every later pass reads shared memory
    for (int i = tid; i < a.vocab; i += SAMPLE_THREADS) keys[i] = (unsigned short)key16(lg[i]);
    // ---- level 1: histogram of the high byte
    hist[tid] = 0;
    __syncthreads();
    for (int i = tid; i < a.vocab; i += SAMPLE_THREADS) atomicAdd(&hist[keys[i] >> 8], 1);
    __syncthreads();
    if (tid == 0) {
      int above = 0, bin = 255;
      for (; bin > 0; bin--) {
        if (above + hist[bin] >= k) break;
        above += hist[bin];
      }
      s_bin = bin; s_above = above;
    }
    __syncthreads();
    const int b1 = s_bin, above1 = s_above;
    // ---- level 2: low byte inside that bin
    hist[tid] = 0;
    __syncthreads();
    for (int i = tid; i < a.vocab; i += SAMPLE_THREADS) {
      const unsigned kk = keys[i];
      if ((int)(kk >> 8) == b1) atomicAdd(&hist[kk & 255], 1);
    }
    __syncthreads();
    if (tid == 0) {
      int above = above1, bin = 255;
      for (; bin > 0; bin--) {
        if (above + hist[bin] >= k) break;
        above += hist[bin];
      }
      s_bin = (b1 << 8) | bin;   // key of the k-th largest value
    }
    __syncthreads();
    const unsigned kth = (unsigned)s_bin;
    // ---- ordered compaction (deterministic): strictly greater first, then the ties at the threshold by index.
    // Thread t owns the contiguous ids [t*per, (t+1)*per); block-wide exclusive scans give the slots.
    const int per = (a.vocab + SAMPLE_THREADS - 1) / SAMPLE_THREADS;
    const int lo = tid * per, hi = min(a.vocab, lo + per);
    int ngt = 0, neq = 0;
    for (int i = lo; i < hi; i++) {
      const unsigned kk = keys[i];
      ngt += kk > kth;
      neq += kk == kth;
    }
    si[tid] = ngt; hist[tid] = neq;
    __syncthreads();
    for (int d = 1; d < SAMPLE_THREADS; d <<= 1) {
      const int x = tid >= d ? si[tid - d] : 0, y = tid >= d ? hist[tid - d] : 0;
      __syncthreads();
      si[tid] += x; hist[tid] += y;
      __syncthreads();
    }
    const int tot_gt = si[SAMPLE_THREADS - 1], tot_eq = hist[SAMPLE_THREADS - 1];
    int sg = si[tid] - ngt, se = tot_gt + hist[tid] - neq;
    for (int i = lo; i < hi; i++) {
      const unsigned kk = keys[i];
      if (kk > kth) { keepv[sg] = __half2float(lg[i]); keepi[sg] = i; sg++; }
      else if (kk == kth) {
        if (se < KEEP_MAX) { keepv[se] = __half2float(lg[i]); keepi[se] = i; }
        se++;
      }
    }
    __syncthreads();
    n_keep = min(tot_gt + tot_eq, KEEP_MAX);  // > KEEP_MAX only if > 128 logits tie at the threshold: lowest ids kept
    // ---- rank sort: descending value, ties by descending index.  TopPLogitsWarper removes a prefix of an
    // (unstable) ascending torch.sort, so WHICH of several equal logits it drops is undefined in the reference;
    // here the lowest ids among equals go first.  The number kept and every non-tied member are HF's.
    if (tid < n_keep) {
      const float v = keepv[tid];
      const int ix = keepi[tid];
      int rank = 0;
      for (int j = 0; j < n_keep; j++) rank += (keepv[j] > v || (keepv[j] == v && keepi[j] > ix)) ? 1 : 0;
      sortv[rank] = v; sorti[rank] = ix;
    }
    __syncthreads();
  }

  if (a.support_out) {  // test hook: the kept set after top-k / top-p is written below by thread 0
    for (int i = tid; i < KEEP_MAX; i += SAMPLE_THREADS) a.support_out[(long)b * KEEP_MAX + i] = -1;
    __syncthreads();
  }

  if (tid == 0) {
    int tok = sorti[0];
    if (a.do_sample) {
      const int K = n_keep;
      // softmax over the kept set (descending order), fp32
      float sum = 0.0f;
      for (int j = 0; j < K; j++) { keepv[j] = ma_exp(fsub(sortv[j], sortv[0])); sum = fadd(sum, keepv[j]); }
      for (int j = 0; j < K; j++) keepv[j] = __fdiv_rn(keepv[j], sum);
      // top-p: ascending cumulative probability <= 1 - top_p is removed (keep >= 1 token)
      int keep = K;
      float cum = 0.0f;
      const float thr = fsub(1.0f, a.top_p);
      for (int j = K - 1; j >= 1; j--) {
        cum = fadd(cum, keepv[j]);
        if (cum <= thr) keep = j; else break;
      }
      if (a.support_out)
        for (int j = 0; j < keep; j++) a.support_out[(long)b * KEEP_MAX + j] = sorti[j];
      float ksum = 0.0f;
      for (int j = 0; j < keep; j++) ksum = fadd(ksum, keepv[j]);
      // stream = the row, or (continuous batching) the queue index of the sequence that occupies the slot
      const uint32_t stream = (a.slots && a.s.sid) ? (uint32_t)a.s.sid[b] : (uint32_t)b;
      const float u = fmul(philox_uniform(a.seed, stream, (uint32_t)gen), ksum);
      float acc = 0.0f;
      tok = sorti[keep - 1];
      for (int j = 0; j < keep; j++) {
        acc = fadd(acc, keepv[j]);
        if (u < acc) { tok = sorti[j]; break; }
      }
    }
    if (a.forced) tok = a.forced[(long)b * a.max_new + gen];
    int fin = a.first ? 0 : a.s.finished[b];
    if (fin) tok = a.pad_id;  // HF: next_tokens * unfinished + pad * (1 - unfinished)
    if (a.out_ids && gen < a.max_new) a.out_ids[(long)b * a.max_new + gen] = tok;
    if (a.s.lens) {
      if (!fin) a.s.lens[b] = gen + 1;
      if (!fin && (tok == a.eos_id || (a.slots && gen + 1 >= a.max_new))) fin = 1;
      a.s.finished[b] = fin;
      a.s.tok[b] = tok;
      a.s.gen[b] = gen + 1;
      const int np = a.first ? PREFIX : a.s.pos[b] + 1;
      a.s.pos[b] = np;
      if (a.nkeys_next) a.nkeys_next[b] = np + 1;
    }
    if (a.token_out) a.token_out[b] = tok;
    si[0] = fin;
  }
  __syncthreads();
  // all_done: every row finished.  Rows are handled by different CTAs: each clears the flag if unfinished.
  if (tid == 0 && a.all_done && !si[0]) *a.all_done = 0;
}

__global__ void set_flag_kernel(int* f, int v) { *f = v; }

int launch_sample(const SampleArgs& a, cudaStream_t st) {
  if (a.do_sample && (a.top_k < 1 || a.top_k > KEEP_MAX / 2)) {
    set_error("sampling needs 1 <= top_k <= %d", KEEP_MAX / 2);
    return 1;
  }
  if (a.all_done) {
    set_flag_kernel<<<1, 1, 0, st>>>(a.all_done, 1);
    count_launch();
  }
  const size_t dyn = a.do_sample ? (size_t)a.vocab * sizeof(unsigned short) : 0;
  if (dyn > 32 * 1024) {
    set_error("sampling supports vocab <= 16384 (got %d)", a.vocab);
    return 1;
  }
  sample_kernel<<<a.nrows > 0 ? a.nrows : a.B, SAMPLE_THREADS, dyn, st>>>(a);
  count_launch();
  return check_launch("sample_kernel") ? 0 : 1;
}

}  // namespace ma
