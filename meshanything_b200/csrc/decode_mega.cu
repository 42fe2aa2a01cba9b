// decode_mega.cu -- batch-1 greedy decode as ONE persistent kernel: one CTA per SM runs every phase
// of every layer of up to `n_steps` tokens.
//
// Why: a token is 24 x (qkv, attention, out_proj, fc1, fc2) + lm_head = 121 dependent phases that
// together must stream 623.5 MB of weights (+ the KV cache) from HBM in ~100 us.  As separate
// kernels (decode_fast.cu) every phase pays a launch boundary (4.8 us measured even with PDL); with
// grid-wide barriers between phases it still pays barrier + dependent load (2.5 us measured).  Here
//   * each CTA owns a fixed, even-sized block of rows of every weight matrix (contiguous bytes), staged
//     through four shared-memory buffers (qkv 44 KB, out_proj 16 KB, fc1 56 KB, fc2 64 KB) refilled by
//     one bulk async copy (TMA 1-D, mbarrier completion) as soon as the phase that read them ends:
//     the weights of layer L+1 are in flight while layer L computes, so HBM streams continuously;
//   * the K/V rows an SM needs for attention are prefetched into registers before the qkv phase;
//   * there is NO grid barrier: every activation vector is exchanged through L2 as 8-byte words
//     {2 x fp16 (or one fp32), 32-bit epoch}; 8-byte stores are single-copy atomic, so a consumer
//     that sees the epoch sees the data (the NCCL "LL" protocol) -- one L2 round trip per hand-off;
//   * the residual stream lives in shared memory; every CTA recomputes the LayerNorms redundantly.
// Arithmetic is the canonical order of DESIGN.md section 3: results are bit-identical to
// gemm_canon.cu / attention.cu / decode_fast.cu and to the CPU oracle.
// Two re-partitionings of this kernel (thread-block clusters + DSMEM; 16 groups of 9 CTAs with split-K out_proj / fc2
// and a reducer tier: git 6b2d32b) were slower than this row split, because every extra stage of the dependent chain
// costs a fixed hand-off in situ whatever its width (measured on the earlier 148-SM target).  What it keeps: the lane-transposed
// attention scores, the merge by every CTA at short contexts (one hand-off less), bounded waits that
// surface as an error (lens = -1) instead of a silently wrong mesh, and the post-mortem record of the first time-out.
#include "canon.cuh"
#include "internal.h"

namespace ma {

constexpr int MG_THREADS = 512;  // 16 warps: one or two weight rows per warp in every GEMV phase, two attention teams
constexpr int MG_WARPS = 16;
constexpr int TEAM = 256;        // threads of one attention team (8 warps = 32 group-lanes, the canonical structure)
constexpr int PARTF = 66;      // o[64], max, sum
constexpr int MAX_CHUNKS = 72;  // 18432 keys

struct MegaWs {
  uint2 qkv_w[QKV / 2];   // flagged words: {half2, epoch}
  uint2 attn_w[HID / 2];
  uint2 ya_w[HID / 2];    // out_proj output
  uint2 yb_w[HID / 2];    // fc2 output
  uint2 f_w[FFN / 2];
  uint2 cand_w[256 * 2];  // {value bits, epoch}, {index, epoch}
  int error;              // != 0: a poll timed out (the first CTA that gave up, + 1)
  int pad_[3];
  unsigned long long trace[1280];
  unsigned long long trace_cta[160 * 8];   // per-CTA stamps of one (step, layer): skew analysis
  ma_decoder_weights w;   // device copy of the weight table
  alignas(256) uint2 part_w[NHEAD * MAX_CHUNKS * PARTF];  // {fp32 bits, epoch}
  alignas(256) __half bias_cta[MA_MAX_LAYERS * 160 * 128];  // [layer][cta][128]: this CTA's biases (see BIAS_*)
};

// layout of one CTA's 128 packed biases of a layer
constexpr int BIAS_QKV = 0, BIAS_OUT = 32, BIAS_FC1 = 48, BIAS_FC2 = 112;

struct MegaArgs {
  MegaWs* ws;
  SeqState s;
  __half* kv;  // [layer][kv][head][T][64]   (batch 1)
  long T;
  int n_steps, step_base, max_new, eos_id, pad_id;
  int rows_qkv, rows_out, rows_fc1, rows_fc2, rows_lm;  // rows per CTA of each matrix (even)
  int32_t* out_ids;
  const int32_t* forced;
  __half* logits_out;
  int* all_done;
  int* nkeys_next;
  int trace;
  int fault;   // test hook: CTA `fault - 1` withholds its out_proj rows from the third token on
};

__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// ---- flagged-word exchange -------------------------------------------------------------------------
__device__ __forceinline__ void ll_store(uint2* p, uint32_t data, uint32_t ep) {
  asm volatile("st.volatile.global.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(data), "r"(ep) : "memory");
}
__device__ __forceinline__ uint4 ll_load2(const uint2* p) {  // two words
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint2 ll_load1(const uint2* p) {
  uint2 v;
  asm volatile("ld.volatile.global.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
  return v;
}
__constant__ unsigned c_spin_limit = 1u << 24;  // polls before a wait gives up (~ seconds): never hang the GPU
#define SPIN_LIMIT c_spin_limit
// one unsuccessful poll: true when the wait must be abandoned (somebody already failed, or this wait ran out of polls;
// the first CTA to give up leaves its number + 1 in the error word)
__device__ __forceinline__ bool poll_giveup(int* err, unsigned& spins) {
  if ((++spins & 1023u) == 0) {
    if (*reinterpret_cast<volatile int*>(err)) return true;
    if (spins > SPIN_LIMIT) {
      atomicCAS(err, 0, 1 + (int)blockIdx.x);
      return true;
    }
  }
  return false;
}
// spin until both words carry epoch `ep`; returns the two data halves
__device__ __forceinline__ uint2 ll_wait2(const uint2* p, uint32_t ep, int* err) {
  uint4 v = ll_load2(p);
  unsigned spins = 0;
  while (v.y != ep || v.w != ep) {
    if (poll_giveup(err, spins)) break;
    v = ll_load2(p);
  }
  return make_uint2(v.x, v.z);
}
__device__ __forceinline__ uint32_t ll_wait1(const uint2* p, uint32_t ep, int* err) {
  uint2 v = ll_load1(p);
  unsigned spins = 0;
  while (v.y != ep) {
    if (poll_giveup(err, spins)) break;
    v = ll_load1(p);
  }
  return v.x;
}
// wait for N consecutive 16-byte units (2 words each) starting at p with stride `stride` units: all loads are
// issued before any flag is checked, and only the units that are not there yet are polled again
template <int N>
__device__ __forceinline__ void ll_wait_units(const uint2* p, int stride, uint32_t ep, uint2* out, int* err) {
  uint4 v[N];
#pragma unroll
  for (int i = 0; i < N; i++) v[i] = ll_load2(p + 2 * i * stride);
  unsigned spins = 0;
  for (;;) {
    bool ok = true;
#pragma unroll
    for (int i = 0; i < N; i++) {
      if (v[i].y != ep || v[i].w != ep) {
        ok = false;
        v[i] = ll_load2(p + 2 * i * stride);
      }
    }
    if (ok) break;
    if (poll_giveup(err, spins)) break;
  }
#pragma unroll
  for (int i = 0; i < N; i++) out[i] = make_uint2(v[i].x, v[i].z);
}
// gather a flagged fp16 vector of `nhalf` elements (1024 or 4096) into shared memory
__device__ __forceinline__ void store_x4(float* dst, uint2 d) {  // 4 fp16 -> 4 fp32 (exact)
  const __half2* hh = reinterpret_cast<const __half2*>(&d);
  const float2 p0 = __half22float2(hh[0]), p1 = __half22float2(hh[1]);
  *reinterpret_cast<float4*>(dst) = make_float4(p0.x, p0.y, p1.x, p1.y);
}
__device__ __forceinline__ void ll_gather(const uint2* src, int nhalf, uint32_t ep, __half* dst, int* err) {
  const int tid = threadIdx.x;
  if (nhalf == FFN) {  // 1024 units: two per thread, both in flight
    uint2 d[2];
    ll_wait_units<2>(src + 2 * tid, MG_THREADS, ep, d, err);
    *reinterpret_cast<uint2*>(dst + 4 * tid) = d[0];
    *reinterpret_cast<uint2*>(dst + 4 * (tid + MG_THREADS)) = d[1];
  } else {
    for (int u = tid; u < nhalf / 4; u += MG_THREADS) {
      const uint2 d = ll_wait2(src + 2 * u, ep, err);
      *reinterpret_cast<uint2*>(dst + 4 * u) = d;
    }
  }
}

// ---- shared memory layout ---------------------------------------------------------------------------
struct alignas(128) MegaSmem {
  uint64_t bar[4];  // full barriers of buffers D (qkv), C (out), A (fc1), B (fc2)
  uint64_t lnbar[2];   // ln1 / ln2 parameter regions
  uint64_t bbar[2];    // packed-bias double buffer
  alignas(16) float ln1[2 * HID];   // gamma | beta of self_attn_layer_norm of the current layer
  alignas(16) float ln2[2 * HID];   // gamma | beta of final_layer_norm
  alignas(16) __half bias[2][128];
  ma_decoder_weights wtab;          // pointer table (kept on chip: every access would be an HBM miss)
  int errflag;
  float red[2][8];   // LayerNorm: warp sums of the mean pass / of the variance pass
  float wmax[2][8];
  float ared[2][8][65];
  float bval[MG_WARPS];
  int bidx[MG_WARPS];
  float cstage[2 * 2 * MAX_CHUNKS];  // per team: {max, sum} of the chunks of one head during the merge
  alignas(16) __half stage16[64];    // fp16 results of this CTA's rows of the current GEMV phase
  alignas(16) float hres[HID];  // residual stream
  alignas(16) __half xs[FFN];   // fp16 input vector of the current GEMV (fp32 would double the shared-memory
                                // traffic, which bounds the GEMV phases: every warp re-reads x)
};

__device__ __forceinline__ uint4 ldcg16(const void* p) { return __ldcg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// LayerNorm of 1024 values by the first 256 threads (thread t owns 4t..4t+3: the canonical block sum); the other
// threads only take part in the barriers.  Returns the normalised values in v (threads < 256).
// Only warps 0-7 take part (named barrier 3); the other warps go straight to the caller's __syncthreads.
__device__ __forceinline__ void layernorm_1024(float* v, const float* gamma, const float* beta, float (*red)[8], int tid) {
  if (tid >= 256) return;
  const int warp = tid >> 5, lane = tid & 31;
  const float inv = __fdiv_rn(1.0f, 1024.0f);
  float p = fadd(fadd(v[0], v[1]), fadd(v[2], v[3]));
  p = warp_sum(p);
  if (lane == 0) red[0][warp] = p;
  asm volatile("bar.sync 3, 256;" ::: "memory");
  const float mean = fmul(warp_tree(red[0], 8), inv);
  const float d0 = fsub(v[0], mean), d1 = fsub(v[1], mean), d2 = fsub(v[2], mean), d3 = fsub(v[3], mean);
  float q = fadd(fadd(fmul(d0, d0), fmul(d1, d1)), fadd(fmul(d2, d2), fmul(d3, d3)));
  q = warp_sum(q);
  if (lane == 0) red[1][warp] = q;
  asm volatile("bar.sync 3, 256;" ::: "memory");
  const float var = fmul(warp_tree(red[1], 8), inv);
  const float rstd = __fdiv_rn(1.0f, __fsqrt_rn(fadd(var, MA_LN_EPS)));
  const float4 g = *reinterpret_cast<const float4*>(gamma + 4 * tid);
  const float4 b = *reinterpret_cast<const float4*>(beta + 4 * tid);
  v[0] = ffma(fmul(d0, rstd), g.x, b.x);
  v[1] = ffma(fmul(d1, rstd), g.y, b.y);
  v[2] = ffma(fmul(d2, rstd), g.z, b.z);
  v[3] = ffma(fmul(d3, rstd), g.w, b.w);
}

__device__ __forceinline__ void team_sync(int team) { asm volatile("bar.sync %0, %1;" ::"r"(1 + team), "r"(TEAM) : "memory"); }

// Rows of this CTA held in shared memory `sw` ([nrows][K]): warp w computes rows w, w+16, w+32, w+48 (those
// that exist) together; lane 0 writes fp16(dot + bias) (ReLU optional) to stage[row].  The caller synchronises and
// emits the rows pairwise.  `bias` is this CTA's slice (shared memory) or null.
__device__ __forceinline__ void load_x8(const float* p, float* xf) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  xf[0] = a.x; xf[1] = a.y; xf[2] = a.z; xf[3] = a.w; xf[4] = b.x; xf[5] = b.y; xf[6] = b.z; xf[7] = b.w;
}

template <int K, bool RELU>
__device__ __forceinline__ void gemv_stage(const __half* sw, int nrows, const __half* bias, const __half* xs, int warp,
                                           int lane, __half* stage) {
  constexpr int G = K / 256;
  if (warp >= nrows) return;
  const __half* w[4];
  bool has[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int r = warp + MG_WARPS * i;
    has[i] = r < nrows;
    w[i] = sw + (size_t)(has[i] ? r : warp) * K + 8 * lane;
  }
  float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
  if (!has[1]) {  // one row (out_proj, fc2, the tail warps of qkv / fc1)
#pragma unroll 4
    for (int g = 0; g < G; g++) {
      float xf[8], f[8];
      unpack8(*reinterpret_cast<const uint4*>(xs + 256 * g + 8 * lane), xf);
      unpack8(*reinterpret_cast<const uint4*>(w[0] + 256 * g), f);
#pragma unroll
      for (int j = 0; j < 8; j++) acc[0] = ffma(f[j], xf[j], acc[0]);
    }
  } else if (!has[2]) {  // two rows (qkv, fc1)
#pragma unroll 4
    for (int g = 0; g < G; g++) {
      float xf[8], f0[8], f1[8];
      unpack8(*reinterpret_cast<const uint4*>(xs + 256 * g + 8 * lane), xf);
      unpack8(*reinterpret_cast<const uint4*>(w[0] + 256 * g), f0);
      unpack8(*reinterpret_cast<const uint4*>(w[1] + 256 * g), f1);
#pragma unroll
      for (int j = 0; j < 8; j++) {
        acc[0] = ffma(f0[j], xf[j], acc[0]);
        acc[1] = ffma(f1[j], xf[j], acc[1]);
      }
    }
  } else {  // three or four rows (lm_head)
#pragma unroll 2
    for (int g = 0; g < G; g++) {
      float xf[8], f[4][8];
      unpack8(*reinterpret_cast<const uint4*>(xs + 256 * g + 8 * lane), xf);
#pragma unroll
      for (int i = 0; i < 4; i++) unpack8(*reinterpret_cast<const uint4*>(w[i] + 256 * g), f[i]);
#pragma unroll
      for (int j = 0; j < 8; j++) {
#pragma unroll
        for (int i = 0; i < 4; i++) acc[i] = ffma(f[i][j], xf[j], acc[i]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    if (i == 0 || has[1]) acc[i] = warp_sum(acc[i]);
  }
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < 4; i++) {
      if (has[i]) {
        const int r = warp + MG_WARPS * i;
        __half h = __float2half_rn(fadd(acc[i], bias ? __half2float(bias[r]) : 0.0f));
        if (RELU && __half2float(h) < 0.0f) h = __float2half_rn(0.0f);
        stage[r] = h;
      }
    }
  }
}

__device__ __forceinline__ uint32_t pack2(__half a, __half b) {
  return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}

// refill a weight buffer with rows [row0, row0+nrows) of W[N][K] (one bulk copy, thread 0 only)
__device__ __forceinline__ void refill(__half* dst, const void* W, int row0, int nrows, int K, uint64_t* bar) {
  fence_proxy_async();
  if (nrows > 0) {
    const uint32_t bytes = (uint32_t)nrows * K * 2;
    mbar_expect_tx(bar, bytes);
    bulk_g2s(dst, reinterpret_cast<const __half*>(W) + (size_t)row0 * K, bytes, bar);
  } else {
    mbar_expect_tx(bar, 0);  // plain arrival so that the phase still completes
  }
}

// LayerNorm gamma|beta (2 x 4 KB) and this CTA's 256 bytes of packed biases: small bulk copies issued one layer ahead
__device__ __forceinline__ void fill_ln(float* dst, const float* g, const float* b, uint64_t* bar) {
  fence_proxy_async();
  mbar_expect_tx(bar, 2u * HID * 4);
  bulk_g2s(dst, g, HID * 4, bar);
  bulk_g2s(dst + HID, b, HID * 4, bar);
}
__device__ __forceinline__ void fill_bias(__half* dst, const __half* src, uint64_t* bar) {
  fence_proxy_async();
  mbar_expect_tx(bar, 256);
  bulk_g2s(dst, src, 256, bar);
}

__global__ void __launch_bounds__(MG_THREADS, 1) decode_mega_kernel(MegaArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  MegaSmem& sm = *reinterpret_cast<MegaSmem*>(smem_raw);
  __half* bufD = reinterpret_cast<__half*>(smem_raw + sizeof(MegaSmem));  // qkv rows
  __half* bufC = bufD + (size_t)a.rows_qkv * HID;                         // out_proj rows
  __half* bufA = bufC + (size_t)a.rows_out * HID;                         // fc1 rows
  __half* bufB = bufA + (size_t)a.rows_fc1 * HID;                         // fc2 rows (K = 4096)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int team = warp >> 3, wt = warp & 7, tl = tid & (TEAM - 1);       // attention team / warp and thread in it
  const int grp = lane >> 3, li = lane & 7;
  MegaWs* ws = a.ws;
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&ws->w);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&sm.wtab);
    for (int i = tid; i < (int)(sizeof(ma_decoder_weights) / 4); i += MG_THREADS) dst[i] = src[i];
  }
  if (tid == 0) sm.errflag = *reinterpret_cast<volatile int*>(&ws->error);
  __syncthreads();
  if (sm.errflag) return;   // an earlier launch of this generate timed out: nothing more is emitted (CTA-uniform)
  const ma_decoder_weights& W = sm.wtab;
  const int NL = W.n_layers;
  const long T = a.T;
  int* err = &ws->error;

  const int cta = blockIdx.x, ncta = gridDim.x;
  const int row0_qkv = cta * a.rows_qkv, n_qkv = max(0, min(a.rows_qkv, QKV - row0_qkv));
  const int row0_out = cta * a.rows_out, n_out = max(0, min(a.rows_out, HID - row0_out));
  const int row0_fc1 = cta * a.rows_fc1, n_fc1 = max(0, min(a.rows_fc1, FFN - row0_fc1));
  const int row0_fc2 = cta * a.rows_fc2, n_fc2 = max(0, min(a.rows_fc2, HID - row0_fc2));
  const int row0_lm = cta * a.rows_lm, n_lm = max(0, min(a.rows_lm, W.vocab - row0_lm));
  // lm rows are staged in D|C|A (contiguous); sub-ranges refilled when each buffer becomes free
  const int lmD = min(n_lm, a.rows_qkv), lmC = max(0, min(n_lm, a.rows_qkv + a.rows_out) - a.rows_qkv),
            lmA = max(0, n_lm - a.rows_qkv - a.rows_out);

  uint32_t parD = 0, parC = 0, parA = 0, parB = 0, parL1 = 0, parL2 = 0, parB0 = 0, parB1 = 0;
  int lc = 0;  // layer instances processed by this launch
  if (tid == 0) {
    for (int i = 0; i < 4; i++) mbar_init(&sm.bar[i], 1);
    for (int i = 0; i < 2; i++) { mbar_init(&sm.lnbar[i], 1); mbar_init(&sm.bbar[i], 1); }
    mbar_fence_init();
    fill_ln(sm.ln1, W.ln1g[0], W.ln1b[0], &sm.lnbar[0]);
    fill_ln(sm.ln2, W.ln2g[0], W.ln2b[0], &sm.lnbar[1]);
    fill_bias(sm.bias[0], ws->bias_cta + ((size_t)0 * 160 + cta) * 128, &sm.bbar[0]);
    fill_bias(sm.bias[1], ws->bias_cta + ((size_t)(NL > 1 ? 1 : 0) * 160 + cta) * 128, &sm.bbar[1]);
    refill(bufD, W.wqkv[0], row0_qkv, n_qkv, HID, &sm.bar[0]);
    refill(bufC, W.wo[0], row0_out, n_out, HID, &sm.bar[1]);
    refill(bufA, W.w1[0], row0_fc1, n_fc1, HID, &sm.bar[2]);
    refill(bufB, W.w2[0], row0_fc2, n_fc2, FFN, &sm.bar[3]);
  }
  __syncthreads();

  // generation state, identical in every CTA
  int pos = a.s.pos[0], gen = a.s.gen[0], tok = a.s.tok[0], fin = a.s.finished[0];
  unsigned long long* tr = (a.trace && cta == 0 && tid == 0) ? ws->trace : nullptr;
  int tri = 0;
#define STAMP() do { if (tr && tri < 1270) tr[tri++] = gtimer(); } while (0)
  // every CTA stamps phase k of (second traced step, layer NL/2)
#define CSTAMP(k) do { if (a.trace && tid == 0 && step == 1 && L == NL / 2) ws->trace_cta[cta * 8 + (k)] = gtimer(); } while (0)

  // xs <- fp16(v) and hres <- v for the 1024-wide vector owned 4 per thread by the first 256 threads
  auto publish_x = [&](const float* v, bool keep_hres) {
    if (tid < 256) {
      if (keep_hres) *reinterpret_cast<float4*>(sm.hres + 4 * tid) = make_float4(v[0], v[1], v[2], v[3]);
      __half2 h0 = __floats2half2_rn(v[0], v[1]), h1 = __floats2half2_rn(v[2], v[3]);
      uint2 u;
      u.x = *reinterpret_cast<uint32_t*>(&h0);
      u.y = *reinterpret_cast<uint32_t*>(&h1);
      *reinterpret_cast<uint2*>(sm.xs + 4 * tid) = u;
    }
  };
  // v <- hres + float(flagged vector words of this thread)
  auto residual_in = [&](const uint2* words, uint32_t ep, float* v) {
    if (tid < 256) {
      const float4 hv = *reinterpret_cast<const float4*>(sm.hres + 4 * tid);
      const uint2 d = ll_wait2(words + 2 * tid, ep, err);
      const __half2* hh = reinterpret_cast<const __half2*>(&d);
      const float2 p0 = __half22float2(hh[0]), p1 = __half22float2(hh[1]);
      v[0] = fadd(hv.x, p0.x); v[1] = fadd(hv.y, p0.y); v[2] = fadd(hv.z, p1.x); v[3] = fadd(hv.w, p1.y);
    } else {
      v[0] = v[1] = v[2] = v[3] = 0.0f;
    }
  };

  for (int step = 0; step < a.n_steps; step++) {
    if (gen >= a.max_new || fin) break;  // uniform across the grid
    const int nkeys = pos + 1;
    const int nch = (nkeys + MA_ATTN_CHUNK - 1) / MA_ATTN_CHUNK;
    const int nitems = nch * NHEAD;
    const uint32_t ep0 = (uint32_t)(a.step_base + step) * (uint32_t)NL + 1u;  // epoch of layer 0 of this step
    STAMP();

    for (int L = 0; L < NL; L++) {
      const uint32_t ep = ep0 + (uint32_t)L;
      const int bsel = lc & 1;            // layer instances alternate between the two bias buffers
      const __half* lb = sm.bias[bsel];   // this layer's packed biases (waited for below)
      __half* kc = a.kv + ((size_t)(L * 2 + 0)) * NHEAD * T * HD;
      __half* vc = a.kv + ((size_t)(L * 2 + 1)) * NHEAD * T * HD;

      // ---------------- K/V prefetch into registers: first attention item of this team (rows < pos are old)
      uint4 kreg[8], vreg[8];
      // attention items are dealt from the LAST CTA downwards (those CTAs own no out_proj / fc2 / qkv rows), first to
      // the teams 0 of all CTAs, then to the teams 1
      int item = team * ncta + (ncta - 1 - cta);
      if (item < nitems) {
        const int c = item >> 4, h = item & 15;
        const long base = ((long)h * T + (long)c * MA_ATTN_CHUNK) * HD;
#pragma unroll
        for (int rho = 0; rho < 8; rho++) {
          const int r = 32 * rho + 4 * wt + grp;
          if (c * MA_ATTN_CHUNK + r < pos) {
            kreg[rho] = ldcg16(kc + base + (long)r * HD + 8 * li);
            vreg[rho] = ldcg16(vc + base + (long)r * HD + 8 * li);
          }
        }
      }

      // ---------------- qkv phase: input = token embedding (layer 0) or LN2(hres + fc2 output) of the previous layer
      {
        float v[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        if (L == 0) {
          if (tid < 256) {
            float4 X;
            int fidx;
            if (tok < 3) {
              X = *reinterpret_cast<const float4*>(W.extra + (long)tok * HID + 4 * tid);
              fidx = tok;
            } else {
              const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const __half*>(W.tok_table) +
                                                              (long)(tok - 3) * HID + 4 * tid);
              const __half2* hh = reinterpret_cast<const __half2*>(&u);
              const float2 p0 = __half22float2(hh[0]), p1 = __half22float2(hh[1]);
              X = make_float4(p0.x, p0.y, p1.x, p1.y);
              int r = (gen - 2) % 9;
              if (r < 0) r += 9;
              fidx = r + 3;
            }
            const float4 F = *reinterpret_cast<const float4*>(W.tok_pos + (long)fidx * HID + 4 * tid);
            const float4 C = *reinterpret_cast<const float4*>(W.cond + HID + 4 * tid);
            const float4 P = *reinterpret_cast<const float4*>(W.pos + (long)(pos + 2) * HID + 4 * tid);
            v[0] = fadd(fadd(fadd(X.x, F.x), C.x), P.x);
            v[1] = fadd(fadd(fadd(X.y, F.y), C.y), P.y);
            v[2] = fadd(fadd(fadd(X.z, F.z), C.z), P.z);
            v[3] = fadd(fadd(fadd(X.w, F.w), C.w), P.w);
          }
        } else {
          residual_in(ws->yb_w, ep - 1, v);  // fc2 output of layer L-1
          mbar_wait(&sm.lnbar[1], parL2);
          parL2 ^= 1;
          layernorm_1024(v, sm.ln2, sm.ln2 + HID, sm.red, tid);
        }
        publish_x(v, true);
      }
      __syncthreads();   // xs complete; every thread has read its gamma/beta
      if (L > 0 && tid == 0) fill_ln(sm.ln2, W.ln2g[L], W.ln2b[L], &sm.lnbar[1]);
      STAMP();
      CSTAMP(0);
      mbar_wait(&sm.bbar[bsel], bsel ? parB1 : parB0);
      if (bsel) parB1 ^= 1; else parB0 ^= 1;
      mbar_wait(&sm.bar[0], parD);
      parD ^= 1;
      STAMP();
      gemv_stage<HID, false>(bufD, n_qkv, lb + BIAS_QKV, sm.xs, warp, lane, sm.stage16);
      STAMP();
      __syncthreads();
      STAMP();
      if (tid < (n_qkv >> 1)) {
        const int n = row0_qkv + 2 * tid;
        const uint32_t d = *reinterpret_cast<const uint32_t*>(sm.stage16 + 2 * tid);
        ll_store(ws->qkv_w + (n >> 1), d, ep);
        if (n >= HID) {  // k / v of the current token also go to the cache for later steps
          const int e = (n - HID) & (HID - 1), head = e >> 6, dd = e & 63;
          __half* c = (n < 2 * HID) ? kc : vc;
          *reinterpret_cast<uint32_t*>(c + ((long)head * T + pos) * HD + dd) = d;
        }
      }
      if (tid == 0) {
        if (L + 1 < NL) refill(bufD, W.wqkv[L + 1], row0_qkv, n_qkv, HID, &sm.bar[0]);
        else refill(bufD, W.lm_head, row0_lm, lmD, HID, &sm.bar[0]);
      }
      STAMP();
      CSTAMP(1);
      // (attention-phase stamps: after the item loop, after the merge)

      // ---------------- attention phase: items (chunk c, head h) = slot, slot + 2*ncta, ... of this team
      for (int it = 0; item < nitems; item += 2 * ncta, it++) {
        const int c = item >> 4, h = item & 15;
        const int len = min(MA_ATTN_CHUNK, nkeys - c * MA_ATTN_CHUNK);
        const long base = ((long)h * T + (long)c * MA_ATTN_CHUNK) * HD;
        const int cur = pos - c * MA_ATTN_CHUNK;  // row of the current token inside this chunk (if 0 <= cur < 256)
#pragma unroll
        for (int rho = 0; rho < 8; rho++) {
          const int r = 32 * rho + 4 * wt + grp;
          if (r < len && it > 0 && r != cur) {  // later items were not prefetched
            kreg[rho] = ldcg16(kc + base + (long)r * HD + 8 * li);
            vreg[rho] = ldcg16(vc + base + (long)r * HD + 8 * li);
          }
        }
        // q of this head and, for the chunk that holds it, k / v of the current token: flagged words
        float qf[8];
        {
          uint2 d[2];
          ll_wait_units<2>(ws->qkv_w + (h * HD + 8 * li) / 2, 1, ep, d, err);
          unpack8(make_uint4(d[0].x, d[0].y, d[1].x, d[1].y), qf);
        }
        if (cur >= 0 && cur < MA_ATTN_CHUNK) {
          const int rho_c = cur >> 5, gl_c = cur & 31;
          if (4 * wt + grp == gl_c) {
            uint2 kk[2], vv[2];
            ll_wait_units<2>(ws->qkv_w + (HID + h * HD + 8 * li) / 2, 1, ep, kk, err);
            ll_wait_units<2>(ws->qkv_w + (2 * HID + h * HD + 8 * li) / 2, 1, ep, vv, err);
            const uint2 k0 = kk[0], k1 = kk[1], v0 = vv[0], v1 = vv[1];
#pragma unroll
            for (int rho = 0; rho < 8; rho++)
              if (rho == rho_c) {
                kreg[rho] = make_uint4(k0.x, k0.y, k1.x, k1.y);
                vreg[rho] = make_uint4(v0.x, v0.y, v1.x, v1.y);
              }
          }
        }
        // Scores of this lane group's 8 rows (rho = 0..7).  Every lane holds the partial dot of ITS 8 dimensions for
        // each row; the canonical xor-4,2,1 sum over the 8 lanes is taken with the transposing butterfly (7 shuffles
        // instead of 24): lane li ends up with the finished score of row rho = li -- the same additions in the same
        // tree as the plain butterfly.  exp is then evaluated once per row (by its owner lane) instead of 8 times.
        float pr[8];
#pragma unroll
        for (int rho = 0; rho < 8; rho++) {
          float kf[8];
          unpack8(kreg[rho], kf);
          float p = 0.0f;
#pragma unroll
          for (int j = 0; j < 8; j++) p = ffma(qf[j], kf[j], p);
          pr[rho] = p;
        }
#pragma unroll
        for (int sft = 4; sft >= 1; sft >>= 1) {
          const bool up = (li & sft) != 0;
#pragma unroll
          for (int i = 0; i < sft; i++) {
            const float mine = up ? pr[i + sft] : pr[i];
            const float other = up ? pr[i] : pr[i + sft];
            pr[i] = fadd(mine, __shfl_xor_sync(0xffffffffu, other, sft));
          }
        }
        const float s_own = fmul(pr[0], 0.125f);                 // score of row rho = li of this lane group
        const bool own_valid = 32 * li + 4 * wt + grp < len;
        float lmax = own_valid ? s_own : -INFINITY;
        lmax = warp_max(lmax);
        team_sync(team);  // previous users of wmax / ared of this team are done
        if (lane == 0) sm.wmax[team][wt] = lmax;
        team_sync(team);
        float cmax = sm.wmax[team][0];
#pragma unroll
        for (int w2 = 1; w2 < 8; w2++) cmax = fmaxf(cmax, sm.wmax[team][w2]);
        const float e_own = own_valid ? ma_exp(fsub(s_own, cmax)) : 0.0f;
        float l = 0.0f, o[8];
#pragma unroll
        for (int j = 0; j < 8; j++) o[j] = 0.0f;
#pragma unroll
        for (int rho = 0; rho < 8; rho++) {
          const int r = 32 * rho + 4 * wt + grp;
          const float e = __shfl_sync(0xffffffffu, e_own, (lane & 24) | rho);   // from the lane that owns row rho
          if (r < len) {
            l = fadd(l, e);
            const float pf = __half2float(__float2half_rn(e));
            float vf[8];
            unpack8(vreg[rho], vf);
#pragma unroll
            for (int j = 0; j < 8; j++) o[j] = ffma(pf, vf[j], o[j]);
          }
        }
        l = fadd(l, __shfl_xor_sync(0xffffffffu, l, 16));
        l = fadd(l, __shfl_xor_sync(0xffffffffu, l, 8));
#pragma unroll
        for (int j = 0; j < 8; j++) {
          o[j] = fadd(o[j], __shfl_xor_sync(0xffffffffu, o[j], 16));
          o[j] = fadd(o[j], __shfl_xor_sync(0xffffffffu, o[j], 8));
        }
        if (grp == 0) {
#pragma unroll
          for (int j = 0; j < 8; j++) sm.ared[team][wt][8 * li + j] = o[j];
          if (li == 0) sm.ared[team][wt][64] = l;
        }
        team_sync(team);
        if (tl < 65) {
          float x[8];
#pragma unroll
          for (int w2 = 0; w2 < 8; w2++) x[w2] = sm.ared[team][w2][tl];
          const float rsum = fadd(fadd(fadd(x[0], x[1]), fadd(x[2], x[3])), fadd(fadd(x[4], x[5]), fadd(x[6], x[7])));
          uint2* part = ws->part_w + ((long)h * MAX_CHUNKS + c) * PARTF;
          ll_store(part + (tl < 64 ? tl : 65), __float_as_uint(rsum), ep);
          if (tl == 64) ll_store(part + 64, __float_as_uint(cmax), ep);
        }
      }
      // the same items of the next layer instance: start pulling their K/V rows into L2 now (first items are also
      // prefetched into registers at the top of the layer; the later rounds of long contexts then hit L2, not HBM)
      if (tl == 0) {
        const int Ln = (L + 1 < NL) ? L + 1 : 0;
        const __half* kn = a.kv + ((size_t)(Ln * 2 + 0)) * NHEAD * T * HD;
        const __half* vn = a.kv + ((size_t)(Ln * 2 + 1)) * NHEAD * T * HD;
        for (int it2 = team * ncta + (ncta - 1 - cta); it2 < nitems; it2 += 2 * ncta) {
          const int c2 = it2 >> 4, h2 = it2 & 15;
          const uint32_t bytes = (uint32_t)min(MA_ATTN_CHUNK, nkeys - c2 * MA_ATTN_CHUNK) * HD * 2;
          const long off = ((long)h2 * T + (long)c2 * MA_ATTN_CHUNK) * HD;
          asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(kn + off), "r"(bytes) : "memory");
          asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(vn + off), "r"(bytes) : "memory");
        }
      }
      STAMP();
      CSTAMP(2);
      // merge of the chunks of head h by team 0 of the CTA that owns item (chunk 0, head h): ascending order
      if (team == 0 && ncta - 1 - cta < NHEAD) {   // the team that owns item (chunk 0, head h)
        const int h = ncta - 1 - cta;
        const uint2* part = ws->part_w + (long)h * MAX_CHUNKS * PARTF;
        // All 66 words of every chunk are staged in shared memory by the 256 threads of the team with their polls in
        // flight together (blocks of up to 31 chunks = the 8 KB of xs, idle during attention).  The chunk weights
        // exp(m_c - M) are computed once per chunk; then 64 threads run the ascending fma chain of the canonical merge.
        float* ost = reinterpret_cast<float*>(sm.xs);          // [chunk][66]
        float* wgt = sm.cstage + team * 2 * MAX_CHUNKS;         // [chunk]
        float* mst = wgt + MAX_CHUNKS;                          // [chunk] maxima (needed before any weight)
        const bool single = nch <= 31;   // one staging round also brings the maxima: no separate round for them
        team_sync(team);
        if (!single) {
          for (int i = tl; i < nch; i += TEAM) mst[i] = __uint_as_float(ll_wait1(part + (long)i * PARTF + 64, ep, err));
          team_sync(team);
          float M = -INFINITY;
          for (int cc = 0; cc < nch; cc++) M = fmaxf(M, mst[cc]);
          for (int i = tl; i < nch; i += TEAM) wgt[i] = ma_exp(fsub(mst[i], M));
        }
        float Lsum = 0.0f, O = 0.0f;
        for (int c0 = 0; c0 < nch; c0 += 31) {
          const int nb = min(31, nch - c0), nw = nb * PARTF;
          {
            uint2 w[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
              const int i = tl + TEAM * k;
              if (i < nw) w[k] = ll_load1(part + (long)c0 * PARTF + i);
            }
            unsigned spins = 0;
            for (;;) {
              bool ok = true;
#pragma unroll
              for (int k = 0; k < 8; k++) {
                const int i = tl + TEAM * k;
                if (i < nw && w[k].y != ep) {
                  ok = false;
                  w[k] = ll_load1(part + (long)c0 * PARTF + i);
                }
              }
              if (ok) break;
              if (poll_giveup(err, spins)) break;
            }
#pragma unroll
            for (int k = 0; k < 8; k++) {
              const int i = tl + TEAM * k;
              if (i < nw) ost[i] = __uint_as_float(w[k].x);
            }
          }
          team_sync(team);
          if (single) {
            float M = -INFINITY;
            for (int cc = 0; cc < nch; cc++) M = fmaxf(M, ost[cc * PARTF + 64]);
            for (int i = tl; i < nch; i += TEAM) wgt[i] = ma_exp(fsub(ost[i * PARTF + 64], M));
            team_sync(team);
          }
          if (tl < 64) {
            for (int cc = 0; cc < nb; cc++) {
              const float wc = wgt[c0 + cc];
              Lsum = ffma(ost[cc * PARTF + 65], wc, Lsum);
              O = ffma(ost[cc * PARTF + tl], wc, O);
            }
          }
          team_sync(team);
        }
        if (tl < 64) {
          const __half r = __float2half_rn(__fdiv_rn(O, Lsum));
          const __half r2 = __shfl_down_sync(0xffffffffu, r, 1);
          if ((tl & 1) == 0) ll_store(ws->attn_w + (h * HD + tl) / 2, pack2(r, r2), ep);
        }
      }
      STAMP();
      CSTAMP(3);

      // ---------------- out_proj phase
      if (n_out > 0) {
        ll_gather(ws->attn_w, HID, ep, sm.xs, err);
        __syncthreads();
        mbar_wait(&sm.bar[1], parC);
        gemv_stage<HID, false>(bufC, n_out, lb + BIAS_OUT, sm.xs, warp, lane, sm.stage16);
        __syncthreads();
        const bool withhold = a.fault && cta == a.fault - 1 && a.step_base + step >= 2;
        if (tid < (n_out >> 1) && !withhold)
          ll_store(ws->ya_w + ((row0_out + 2 * tid) >> 1), *reinterpret_cast<const uint32_t*>(sm.stage16 + 2 * tid), ep);
      } else {
        __syncthreads();
        mbar_wait(&sm.bar[1], parC);
      }
      parC ^= 1;
      if (tid == 0) {
        if (L + 1 < NL) refill(bufC, W.wo[L + 1], row0_out, n_out, HID, &sm.bar[1]);
        else refill(bufC, W.lm_head, row0_lm + a.rows_qkv, lmC, HID, &sm.bar[1]);
      }
      STAMP();
      CSTAMP(4);

      // ---------------- fc1 phase: input = LN1(hres + out_proj)
      {
        float v[4];
        residual_in(ws->ya_w, ep, v);
        mbar_wait(&sm.lnbar[0], parL1);
        parL1 ^= 1;
        layernorm_1024(v, sm.ln1, sm.ln1 + HID, sm.red, tid);
        publish_x(v, true);
      }
      __syncthreads();
      if (tid == 0) fill_ln(sm.ln1, W.ln1g[(L + 1) % NL], W.ln1b[(L + 1) % NL], &sm.lnbar[0]);
      mbar_wait(&sm.bar[2], parA);
      parA ^= 1;
      gemv_stage<HID, true>(bufA, n_fc1, lb + BIAS_FC1, sm.xs, warp, lane, sm.stage16);
      __syncthreads();
      if (tid < (n_fc1 >> 1))
        ll_store(ws->f_w + ((row0_fc1 + 2 * tid) >> 1), *reinterpret_cast<const uint32_t*>(sm.stage16 + 2 * tid), ep);
      if (tid == 0) {
        if (L + 1 < NL) refill(bufA, W.w1[L + 1], row0_fc1, n_fc1, HID, &sm.bar[2]);
        else refill(bufA, W.lm_head, row0_lm + a.rows_qkv + a.rows_out, lmA, HID, &sm.bar[2]);
      }
      STAMP();
      CSTAMP(5);

      // ---------------- fc2 phase
      if (n_fc2 > 0) {
        ll_gather(ws->f_w, FFN, ep, sm.xs, err);
        __syncthreads();
        mbar_wait(&sm.bar[3], parB);
        gemv_stage<FFN, false>(bufB, n_fc2, lb + BIAS_FC2, sm.xs, warp, lane, sm.stage16);
        __syncthreads();
        if (tid < (n_fc2 >> 1))
          ll_store(ws->yb_w + ((row0_fc2 + 2 * tid) >> 1), *reinterpret_cast<const uint32_t*>(sm.stage16 + 2 * tid), ep);
      } else {
        __syncthreads();
        mbar_wait(&sm.bar[3], parB);
      }
      parB ^= 1;
      if (tid == 0) {
        refill(bufB, W.w2[(L + 1 < NL) ? L + 1 : 0], row0_fc2, n_fc2, FFN, &sm.bar[3]);
        // the bias buffer of this layer is free: refill it for the layer instance that uses it next (L + 2)
        fill_bias(sm.bias[bsel], ws->bias_cta + ((size_t)((L + 2) % NL) * 160 + cta) * 128, &sm.bbar[bsel]);
      }
      lc++;
      STAMP();
      CSTAMP(6);
    }

    // ---------------- lm_head on LN2 of the last layer + greedy pick
    const uint32_t epc = (uint32_t)(a.step_base + step) + 1u;
    {
      float v[4];
      residual_in(ws->yb_w, ep0 + (uint32_t)NL - 1u, v);
      mbar_wait(&sm.lnbar[1], parL2);
      parL2 ^= 1;
      layernorm_1024(v, sm.ln2, sm.ln2 + HID, sm.red, tid);
      publish_x(v, false);
    }
    __syncthreads();
    if (tid == 0) fill_ln(sm.ln2, W.ln2g[0], W.ln2b[0], &sm.lnbar[1]);
    mbar_wait(&sm.bar[0], parD);
    mbar_wait(&sm.bar[1], parC);
    mbar_wait(&sm.bar[2], parA);
    parD ^= 1; parC ^= 1; parA ^= 1;
    gemv_stage<HID, false>(bufD, n_lm, nullptr, sm.xs, warp, lane, sm.stage16);
    __syncthreads();
    float bestv = -INFINITY;
    int besti = 0x7fffffff;
    if (tid < n_lm) {
      const __half hv = sm.stage16[tid];
      if (a.logits_out) a.logits_out[(long)gen * W.vocab + row0_lm + tid] = hv;
      bestv = __half2float(hv);
      besti = row0_lm + tid;
    }
    if (warp < 2) {  // rows_lm <= 64: the candidates live in the first two warps
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bestv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
        if (ov > bestv || (ov == bestv && oi < besti)) { bestv = ov; besti = oi; }
      }
      if (lane == 0) { sm.bval[warp] = bestv; sm.bidx[warp] = besti; }
    }
    __syncthreads();
    if (tid == 0) {
      float bv = sm.bval[0];
      int bi = sm.bidx[0];
      if (sm.bval[1] > bv || (sm.bval[1] == bv && sm.bidx[1] < bi)) { bv = sm.bval[1]; bi = sm.bidx[1]; }
      __threadfence();  // publish this step's KV-cache rows before the step's final hand-off
      ll_store(ws->cand_w + 2 * cta, __float_as_uint(bv), epc);
      ll_store(ws->cand_w + 2 * cta + 1, (uint32_t)bi, epc);
      // weights of the next token's first layer
      refill(bufD, W.wqkv[0], row0_qkv, n_qkv, HID, &sm.bar[0]);
      refill(bufC, W.wo[0], row0_out, n_out, HID, &sm.bar[1]);
      refill(bufA, W.w1[0], row0_fc1, n_fc1, HID, &sm.bar[2]);
    }
    {
      float bv = -INFINITY;
      int bi = 0x7fffffff;
      if (tid < ncta) {
        const uint2 d = ll_wait2(ws->cand_w + 2 * tid, epc, err);
        bv = __uint_as_float(d.x);
        bi = (int)d.y;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
      }
      __syncthreads();
      if (lane == 0) { sm.bval[warp] = bv; sm.bidx[warp] = bi; }
      if (tid == 0) sm.errflag = *reinterpret_cast<volatile int*>(&ws->error);   // one reader: CTA-uniform decision
      __syncthreads();
      bv = sm.bval[0];
      bi = sm.bidx[0];
      for (int w2 = 1; w2 < MG_WARPS; w2++)
        if (sm.bval[w2] > bv || (sm.bval[w2] == bv && sm.bidx[w2] < bi)) { bv = sm.bval[w2]; bi = sm.bidx[w2]; }
      if (sm.errflag) break;   // a wait of this step failed somewhere: emit nothing more
      int ntok = bi;
      if (a.forced) ntok = a.forced[gen];
      if (fin) ntok = a.pad_id;
      if (cta == 0 && tid == 0) {
        if (gen < a.max_new) a.out_ids[gen] = ntok;
        if (!fin) a.s.lens[0] = gen + 1;
      }
      if (!fin && ntok == a.eos_id) fin = 1;
      tok = ntok;
      gen += 1;
      pos += 1;
      __syncthreads();
    }
    STAMP();
  }

  // every buffer has a refill in flight here: drain them before the shared memory is released
  mbar_wait(&sm.bar[0], parD);
  mbar_wait(&sm.bar[1], parC);
  mbar_wait(&sm.bar[2], parA);
  mbar_wait(&sm.bar[3], parB);
  mbar_wait(&sm.lnbar[0], parL1);
  mbar_wait(&sm.lnbar[1], parL2);
  mbar_wait(&sm.bbar[0], parB0);
  mbar_wait(&sm.bbar[1], parB1);
  if (cta == 0 && tid == 0) {
    const int e = *reinterpret_cast<volatile int*>(&ws->error);
    a.s.pos[0] = pos; a.s.gen[0] = gen; a.s.tok[0] = tok; a.s.finished[0] = e ? 1 : fin;
    if (e) a.s.lens[0] = -1;   // surfaced by the callers of ma_decode_generate (out_lens): no silently wrong mesh
    if (a.nkeys_next) *a.nkeys_next = pos + 1;
    if (a.all_done) *a.all_done = e ? 1 : fin;
  }
}

// ---- host side -----------------------------------------------------------------------------------
static int g_mega_sms = 0;
size_t mega_workspace_bytes() { return sizeof(MegaWs) + 256; }

static int mega_sms() {
  if (!g_mega_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_mega_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_mega_sms <= 0 || g_mega_sms > 160) g_mega_sms = 132;
  }
  return g_mega_sms;
}
static inline int mega_rpc(int N) { return (((N + mega_sms() - 1) / mega_sms()) + 1) & ~1; }  // even rows per CTA

// bias_cta[L][cta][128] <- the biases of the rows CTA `cta` owns in layer L
__global__ void mega_pack_bias_kernel(MegaWs* ws, int rq, int ro, int r1, int r2) {
  const int L = blockIdx.y, cta = blockIdx.x, t = threadIdx.x;  // 128 threads
  const ma_decoder_weights& W = ws->w;
  __half v = __float2half_rn(0.0f);
  if (t < BIAS_OUT) {
    const int n = cta * rq + t;
    if (t < rq && n < QKV) v = reinterpret_cast<const __half*>(W.bqkv[L])[n];
  } else if (t < BIAS_FC1) {
    const int i = t - BIAS_OUT, n = cta * ro + i;
    if (i < ro && n < HID) v = reinterpret_cast<const __half*>(W.bo[L])[n];
  } else if (t < BIAS_FC2) {
    const int i = t - BIAS_FC1, n = cta * r1 + i;
    if (i < r1 && n < FFN) v = reinterpret_cast<const __half*>(W.b1[L])[n];
  } else {
    const int i = t - BIAS_FC2, n = cta * r2 + i;
    if (i < r2 && n < HID) v = reinterpret_cast<const __half*>(W.b2[L])[n];
  }
  ws->bias_cta[((size_t)L * 160 + cta) * 128 + t] = v;
}

int mega_prepare(const ma_decoder_weights* w, void* mega_ws, cudaStream_t st) {
  MegaWs* ws = reinterpret_cast<MegaWs*>(mega_ws);
  if (cudaMemsetAsync(ws, 0, offsetof(MegaWs, bias_cta), st) != cudaSuccess) return 1;  // all epochs 0
  if (cudaMemcpyAsync(&ws->w, w, sizeof(ma_decoder_weights), cudaMemcpyHostToDevice, st) != cudaSuccess) return 1;
  const int rq = mega_rpc(QKV), ro = mega_rpc(HID), r1 = mega_rpc(FFN), r2 = mega_rpc(HID);
  if (rq > 32 || ro > 16 || r1 > 64 || r2 > 16) {
    set_error("mega: rows per CTA out of range");
    return 1;
  }
  mega_pack_bias_kernel<<<dim3(160, w->n_layers), 128, 0, st>>>(ws, rq, ro, r1, r2);
  count_launch();
  return check_launch("mega_pack_bias_kernel") ? 0 : 1;
}

static int g_mega_fault = 0;
void mega_set_debug(unsigned long long timeout_ns, int fault) {
  if (timeout_ns) {
    // a poll of a word that is not there yet takes ~0.4 us (one L2 round trip)
    const unsigned long long polls = timeout_ns / 400ull + 2048ull;
    const unsigned v = polls > 0xffffffffull ? 0xffffffffu : (unsigned)polls;
    cudaMemcpyToSymbol(c_spin_limit, &v, sizeof(v));
  }
  g_mega_fault = fault;
}
bool mega_fits(int tmax) { return tmax <= MAX_CHUNKS * MA_ATTN_CHUNK; }
// Can the persistent kernel run on this device?  (every CTA must own fc1 and lm_head rows, the last 16 CTAs no
// out_proj rows, and a CTA's rows must fit its shared memory: at least 147 SMs.  An H100 with 132 SMs does not
// qualify, and batch-1 greedy decoding runs on the per-phase kernels of decode_fast.cu there.)
int mega_supported() {
  static int ok = -1;
  if (ok < 0) {
    const int sms = mega_sms(), r1 = mega_rpc(FFN), ro = mega_rpc(HID);
    const int grid = (FFN + r1 - 1) / r1;
    ok = (grid <= sms && grid >= NHEAD && grid - NHEAD >= (HID + ro - 1) / ro && mega_rpc(QKV) <= 32 && ro <= 16 && r1 <= 64) ? 1 : 0;
    if (!ok) set_error("mega: unsupported SM count %d", sms);
  }
  return ok;
}
int mega_error_flag_offset() { return (int)offsetof(MegaWs, error); }
int mega_trace_offset() { return (int)offsetof(MegaWs, trace); }
int mega_trace_cta_offset() { return (int)offsetof(MegaWs, trace_cta); }

int mega_enqueue(const ma_decoder_weights* w, SeqState s, int tmax, __half* kv, void* mega_ws, const SampleArgs& sa,
                 int n_steps, int step_base, int trace, cudaStream_t st) {
  if (tmax > MAX_CHUNKS * MA_ATTN_CHUNK) {
    set_error("mega: tmax=%d exceeds %d keys", tmax, MAX_CHUNKS * MA_ATTN_CHUNK);
    return 1;
  }
  const int sms = mega_sms();
  auto rpc = [&](int N) { return mega_rpc(N); };
  MegaArgs a;
  memset(&a, 0, sizeof(a));
  a.ws = reinterpret_cast<MegaWs*>(mega_ws);
  a.s = s;
  a.kv = kv;
  a.T = tmax;
  a.n_steps = n_steps;
  a.step_base = step_base;
  a.max_new = sa.max_new; a.eos_id = sa.eos_id; a.pad_id = sa.pad_id;
  a.rows_qkv = rpc(QKV); a.rows_out = rpc(HID); a.rows_fc1 = rpc(FFN); a.rows_fc2 = rpc(HID); a.rows_lm = rpc(w->vocab);
  a.out_ids = sa.out_ids; a.forced = sa.forced; a.logits_out = sa.logits_out; a.all_done = sa.all_done;
  a.nkeys_next = sa.nkeys_next;
  a.trace = trace;
  a.fault = g_mega_fault;
  if (a.rows_lm > a.rows_qkv + a.rows_out + a.rows_fc1 || a.rows_lm > 64 || a.rows_fc1 > 64) {
    set_error("mega: rows per CTA out of range (lm %d, fc1 %d)", a.rows_lm, a.rows_fc1);
    return 1;
  }
  // Every CTA must produce fc1 and lm_head rows (they are what orders buffer reuse), so the grid is the
  // number of CTAs that own fc1 rows; CTAs beyond the rows of a smaller matrix idle in that phase only.
  const int grid = (FFN + a.rows_fc1 - 1) / a.rows_fc1;
  if (grid > sms || (w->vocab + a.rows_lm - 1) / a.rows_lm != grid || grid < NHEAD) {
    set_error("mega: unsupported SM count %d (grid %d)", sms, grid);
    return 1;
  }
  // the merging teams (last 16 CTAs) stage partials in xs while the other team may run ahead: those CTAs must not
  // own out_proj / fc2 rows (whose phases write xs from all threads)
  if (grid - NHEAD < (HID + a.rows_out - 1) / a.rows_out) {
    set_error("mega: the last %d CTAs must not own out_proj rows (grid %d)", NHEAD, grid);
    return 1;
  }
  const size_t smem = sizeof(MegaSmem) + ((size_t)(a.rows_qkv + a.rows_out + a.rows_fc1) * HID + (size_t)a.rows_fc2 * FFN) * 2;
  static size_t attr_set = 0;
  if (smem > attr_set) {
    if (cudaFuncSetAttribute(decode_mega_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
      set_error("mega: cannot get %zu bytes of shared memory", smem);
      cudaGetLastError();
      return 1;
    }
    attr_set = smem;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(MG_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative;  // all CTAs co-resident (they wait on each other's data)
  at[0].val.cooperative = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, decode_mega_kernel, a);
  count_launch();
  return check_launch("decode_mega_kernel") ? 0 : 1;
}

}  // namespace ma
