/*
 * decoder_oracle.c -- CPU ORACLE (test infrastructure, NOT a product path).
 *
 * Plain-C restatement of the ShapeOPT-350M decoder of MeshAnything as the reference executes it
 * under `torch.autocast('cuda', fp16)`:
 *
 *   ShapeOPTDecoder.forward        /root/reference/MeshAnything/models/shape_opt.py:248-438
 *   ShapeOPTDecoder.embed_with_vae /root/reference/MeshAnything/models/shape_opt.py:237-245
 *   OPTFacePositionalEmbedding     /root/reference/MeshAnything/models/shape_opt.py:440-460
 *   ShapeOPT.forward (lm_head)     /root/reference/MeshAnything/models/shape_opt.py:143-155
 *   OPTLearnedPositionalEmbedding / OPTDecoderLayer (post-LN, ReLU) -- transformers==4.39.3
 *     (requirements.txt:9; not vendored).  Same math in the installed 5.5.0:
 *     site-packages/transformers/models/opt/modeling_opt.py:43-71,184-254.
 *   flash_attn_func: softmax(q k^T / sqrt(64)) v, fp16 in/out, fp32 accumulate, P rounded to fp16
 *     before the PV product (flash-attn, unpinned dependency, README.md:75).
 *
 * Rounding points (autocast): Linear inputs/weights/biases are fp16, Linear outputs are rounded to
 * fp16 once after (fp32 accumulator + bias); LayerNorm, residual adds and embeddings are fp32.
 *
 * The reference leaves the fp32 accumulation ORDER to cuBLAS / flash-attn.  This oracle fixes one
 * ("canonical order", DESIGN.md section 3) that is emulated here with scalar loops over virtual
 * lanes; the CUDA kernels must reproduce it bit for bit.  Parity of this restatement with the
 * reference is UNPINNED by the reference (it ships no tests or golden vectors); it is pinned by
 * tests/test_oracle.py against fp32 logits of transformers' own OPTDecoderLayer stack + the reference's own
 * embedding functions (tests/golden/decoder_hf_fp32.npz, decoder_hf_fp32_deep.npz: 24 layers x 320 positions)
 * and, on the GPU box, by tests/test_gpu_hf.py (HF OPTDecoderLayer x 24 under fp16 autocast).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this library.
 */
#include <math.h>
#ifdef _OPENMP
#include <omp.h>
#endif
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#if defined(__F16C__) && defined(__AVX2__) && defined(__FMA__)
#include <immintrin.h>
#define ORC_SIMD 1
#endif

#include "../include/ma_canon_constants.h"

typedef _Float16 h16;

#define HID 1024
#define NHEAD 16
#define HD 64
#define FFN 4096
#define PREFIX 257

/* ------------------------------------------------------------------ canonical scalar pieces */

static inline float ma_exp(float x) {
  if (x < MA_EXP_FLUSH) return 0.0f;
  float y = x * MA_LOG2E;
  float n = rintf(y);
  float f = y - n;
  float p = MA_EXP2_C6;
  p = fmaf(p, f, MA_EXP2_C5);
  p = fmaf(p, f, MA_EXP2_C4);
  p = fmaf(p, f, MA_EXP2_C3);
  p = fmaf(p, f, MA_EXP2_C2);
  p = fmaf(p, f, MA_EXP2_C1);
  p = fmaf(p, f, MA_EXP2_C0);
  int32_t bits;
  memcpy(&bits, &p, 4);
  bits += ((int32_t)n) << 23;
  memcpy(&p, &bits, 4);
  return p;
}

/* lane-0 value of the xor-16,8,4,2,1 butterfly over 32 lane partials */
static inline float butterfly32(const float *a) {
  float s1[16], s2[8], s3[4], s4[2];
  for (int i = 0; i < 16; i++) s1[i] = a[i] + a[i + 16];
  for (int i = 0; i < 8; i++) s2[i] = s1[i] + s1[i + 8];
  for (int i = 0; i < 4; i++) s3[i] = s2[i] + s2[i + 4];
  for (int i = 0; i < 2; i++) s4[i] = s3[i] + s3[i + 2];
  return s4[0] + s4[1];
}

/* Lane-transposed layout: element k = 256 g + 8 l + j  ->  index (g*8 + j)*32 + l. */
static void transpose_row_h16(const h16 *src, h16 *dst, int K) {
  for (int g = 0; g < K / 256; g++)
    for (int l = 0; l < 32; l++)
      for (int j = 0; j < 8; j++) dst[(g * 8 + j) * 32 + l] = src[256 * g + 8 * l + j];
}
static void transpose_x_f32(const h16 *src, float *dst, int K) {
  for (int g = 0; g < K / 256; g++)
    for (int l = 0; l < 32; l++)
      for (int j = 0; j < 8; j++) dst[(g * 8 + j) * 32 + l] = (float)src[256 * g + 8 * l + j];
}

/* canonical dot: lane l accumulates k = 256g+8l+j sequentially (g major, j minor) with fmaf from 0,
 * then the butterfly.  wT / xT are lane-transposed. */
static inline float dot_canon_T(const h16 *wT, const float *xT, int K) {
  float a[32];
#ifdef ORC_SIMD
  __m256 a0 = _mm256_setzero_ps(), a1 = a0, a2 = a0, a3 = a0;
  for (int q = 0; q < K / 32; q++) {
    const h16 *w = wT + q * 32;
    const float *x = xT + q * 32;
    a0 = _mm256_fmadd_ps(_mm256_cvtph_ps(_mm_loadu_si128((const __m128i *)(w))), _mm256_loadu_ps(x), a0);
    a1 = _mm256_fmadd_ps(_mm256_cvtph_ps(_mm_loadu_si128((const __m128i *)(w + 8))), _mm256_loadu_ps(x + 8), a1);
    a2 = _mm256_fmadd_ps(_mm256_cvtph_ps(_mm_loadu_si128((const __m128i *)(w + 16))), _mm256_loadu_ps(x + 16), a2);
    a3 = _mm256_fmadd_ps(_mm256_cvtph_ps(_mm_loadu_si128((const __m128i *)(w + 24))), _mm256_loadu_ps(x + 24), a3);
  }
  _mm256_storeu_ps(a, a0);
  _mm256_storeu_ps(a + 8, a1);
  _mm256_storeu_ps(a + 16, a2);
  _mm256_storeu_ps(a + 24, a3);
#else
  for (int l = 0; l < 32; l++) a[l] = 0.0f;
  for (int q = 0; q < K / 32; q++)
    for (int l = 0; l < 32; l++) a[l] = fmaf((float)wT[q * 32 + l], xT[q * 32 + l], a[l]);
#endif
  return butterfly32(a);
}

/* pairwise left-to-right tree over n warp sums (n = 8: ((0+1)+(2+3))+((4+5)+(6+7)); n = 6: ((0+1)+(2+3))+(4+5)) */
static float warp_tree(const float *s, int n) {
  float buf[16];
  for (int i = 0; i < n; i++) buf[i] = s[i];
  while (n > 1) {
    int m = 0;
    for (int i = 0; i + 1 < n; i += 2) buf[m++] = buf[i] + buf[i + 1];
    if (n & 1) buf[m++] = buf[n - 1];
    n = m;
  }
  return buf[0];
}

/* canonical block sum over W = 4*T elements: thread t owns 4t..4t+3 -> (x0+x1)+(x2+x3); warp butterfly; warp tree */
static float block_sum(const float *v, int W) {
  int T = W / 4, nw = T / 32;
  float ws[16];
  for (int w = 0; w < nw; w++) {
    float a[32];
    for (int l = 0; l < 32; l++) {
      const float *p = v + 4 * (32 * w + l);
      a[l] = (p[0] + p[1]) + (p[2] + p[3]);
    }
    ws[w] = butterfly32(a);
  }
  return warp_tree(ws, nw);
}

/* y = LN(x) * gamma + beta, fp32, width W (multiple of 128) */
static void layernorm_canon(const float *x, const float *gamma, const float *beta, float eps, float *y, int W) {
  float tmp[4096];
  float mean = block_sum(x, W) * (1.0f / (float)W);
  for (int i = 0; i < W; i++) {
    float d = x[i] - mean;
    tmp[i] = d * d;
  }
  float var = block_sum(tmp, W) * (1.0f / (float)W);
  float rstd = 1.0f / sqrtf(var + eps);
  for (int i = 0; i < W; i++) {
    float d = x[i] - mean;
    y[i] = fmaf(d * rstd, gamma[i], beta[i]);
  }
}

/* one head, one query, keys [0,n): K/V rows are HD contiguous fp16 with row stride `stride` elements */
static void attention_head_canon(const h16 *q, const h16 *Kc, const h16 *Vc, long stride, int n, h16 *out) {
  int nch = (n + MA_ATTN_CHUNK - 1) / MA_ATTN_CHUNK;
  float *pm = (float *)malloc(sizeof(float) * nch * 66);
  float qf[HD];
  for (int d = 0; d < HD; d++) qf[d] = (float)q[d];
  for (int c = 0; c < nch; c++) {
    int len = n - c * MA_ATTN_CHUNK;
    if (len > MA_ATTN_CHUNK) len = MA_ATTN_CHUNK;
    float s[MA_ATTN_CHUNK];
    float m = -INFINITY;
    for (int r = 0; r < len; r++) {
      const h16 *k = Kc + (long)(c * MA_ATTN_CHUNK + r) * stride;
      float p[8];
      for (int i = 0; i < 8; i++) {
        float a = 0.0f;
        for (int j = 0; j < 8; j++) a = fmaf(qf[8 * i + j], (float)k[8 * i + j], a);
        p[i] = a;
      }
      float u0 = p[0] + p[4], u1 = p[1] + p[5], u2 = p[2] + p[6], u3 = p[3] + p[7];
      float v0 = u0 + u2, v1 = u1 + u3;
      s[r] = (v0 + v1) * 0.125f;
      if (s[r] > m) m = s[r];
    }
    /* 32 group-lanes: position r -> gl = r % 32, sequential over rounds */
    static _Thread_local float acc[32][65];
    for (int gl = 0; gl < 32; gl++)
      for (int d = 0; d < 65; d++) acc[gl][d] = 0.0f;
    for (int r = 0; r < len; r++) {
      int gl = r & 31;
      const h16 *v = Vc + (long)(c * MA_ATTN_CHUNK + r) * stride;
      float e = ma_exp(s[r] - m);
      acc[gl][64] = acc[gl][64] + e;
      float pf = (float)(h16)e;
      for (int d = 0; d < HD; d++) acc[gl][d] = fmaf(pf, (float)v[d], acc[gl][d]);
    }
    float *o = pm + c * 66;
    o[64] = m;
    for (int d = 0; d < 65; d++) {
      float xw[8];
      for (int w = 0; w < 8; w++)
        xw[w] = (acc[4 * w + 0][d] + acc[4 * w + 2][d]) + (acc[4 * w + 1][d] + acc[4 * w + 3][d]);
      float r = ((xw[0] + xw[1]) + (xw[2] + xw[3])) + ((xw[4] + xw[5]) + (xw[6] + xw[7]));
      if (d < 64) o[d] = r; else o[65] = r;
    }
  }
  float M = -INFINITY;
  for (int c = 0; c < nch; c++) if (pm[c * 66 + 64] > M) M = pm[c * 66 + 64];
  float L = 0.0f, O[HD];
  for (int d = 0; d < HD; d++) O[d] = 0.0f;
  for (int c = 0; c < nch; c++) {
    float w = ma_exp(pm[c * 66 + 64] - M);
    L = fmaf(pm[c * 66 + 65], w, L);
    for (int d = 0; d < HD; d++) O[d] = fmaf(pm[c * 66 + d], w, O[d]);
  }
  for (int d = 0; d < HD; d++) out[d] = (h16)(O[d] / L);
  free(pm);
}

/* ------------------------------------------------------------------ unit-level entry points */

/* y[M][N] = fp16(dot(W[n], x[m]) + b[n]) (+relu); W [N][K], x [M][K], b [N] or NULL, all fp16 */
void orc_linear(const uint16_t *W_, const uint16_t *b_, const uint16_t *x_, int M, int N, int K, int relu,
                uint16_t *y_) {
  const h16 *W = (const h16 *)W_, *b = (const h16 *)b_, *x = (const h16 *)x_;
  h16 *y = (h16 *)y_;
  float *xT = (float *)malloc(sizeof(float) * (size_t)M * K);
  for (int m = 0; m < M; m++) transpose_x_f32(x + (size_t)m * K, xT + (size_t)m * K, K);
#pragma omp parallel
  {
    h16 *wT = (h16 *)malloc(sizeof(h16) * K);
#pragma omp for schedule(static)
    for (int n = 0; n < N; n++) {
      transpose_row_h16(W + (size_t)n * K, wT, K);
      float bf = b ? (float)b[n] : 0.0f;
      for (int m = 0; m < M; m++) {
        float acc = dot_canon_T(wT, xT + (size_t)m * K, K);
        h16 r = (h16)(acc + bf);
        if (relu && (float)r < 0.0f) r = (h16)0.0f;
        y[(size_t)m * N + n] = r;
      }
    }
    free(wT);
  }
  free(xT);
}

/* rows of width W: h = x (+ float(res16)); y = LN(h); outputs fp32 y and fp16 y */
void orc_layernorm(const float *x, const uint16_t *res16_, const float *gamma, const float *beta, float eps, int M,
                   int W, float *y, uint16_t *y16_) {
  const h16 *res16 = (const h16 *)res16_;
  h16 *y16 = (h16 *)y16_;
  for (int m = 0; m < M; m++) {
    float h[4096], o[4096];
    for (int i = 0; i < W; i++) h[i] = res16 ? x[(size_t)m * W + i] + (float)res16[(size_t)m * W + i] : x[(size_t)m * W + i];
    layernorm_canon(h, gamma, beta, eps, o, W);
    for (int i = 0; i < W; i++) {
      if (y) y[(size_t)m * W + i] = o[i];
      if (y16) y16[(size_t)m * W + i] = (h16)o[i];
    }
  }
}

/* q [M][H*64]; K,V [H][T][64] (row stride 64) ; nkeys[m]; out [M][H*64] */
void orc_attention(const uint16_t *q_, const uint16_t *K_, const uint16_t *V_, const int *nkeys, int M, int H, long T,
                   uint16_t *out_) {
  const h16 *q = (const h16 *)q_, *K = (const h16 *)K_, *V = (const h16 *)V_;
  h16 *out = (h16 *)out_;
#pragma omp parallel for collapse(2) schedule(dynamic)
  for (int m = 0; m < M; m++)
    for (int h = 0; h < H; h++)
      attention_head_canon(q + ((size_t)m * H + h) * HD, K + (size_t)h * T * HD, V + (size_t)h * T * HD, HD, nkeys[m],
                           out + ((size_t)m * H + h) * HD);
}

float orc_exp(float x) { return ma_exp(x); }

/* y[i] = ma_exp(x[i]): the sampler restatement (tests/sampler_oracle.py) calls this once per kept set */
void orc_exp_n(const float *x, int n, float *y) {
  for (int i = 0; i < n; i++) y[i] = ma_exp(x[i]);
}

/* ------------------------------------------------------------------ the decoder */

typedef struct {
  h16 *wq, *wk, *wv, *wo, *w1, *w2; /* lane-transposed rows */
  h16 *bq, *bk, *bv, *bo, *b1, *b2;
  float *ln1g, *ln1b, *ln2g, *ln2b;
} orc_layer;

typedef struct {
  int n_layers, vocab, tmax;
  orc_layer *L;
  h16 *lm_head;    /* [vocab][1024] lane-transposed */
  h16 *tok_table;  /* [codebook][1024] = fp16(input_layer(fp16(codebook)))  (shape_opt.py:243) */
  int codebook;
  float *extra;    /* [3][1024]   shape_opt.py:209 */
  float *tok_pos;  /* [12][1024]  shape_opt.py:213 */
  float *cond;     /* [2][1024]   shape_opt.py:216 */
  float *pos;      /* [npos][1024] OPTLearnedPositionalEmbedding incl. the 2 offset rows */
  int npos;
  h16 *kc, *vc;    /* [layer][head][tmax][64] */
  int t;           /* cached positions */
} orc_dec;

static h16 *dup_T(const uint16_t *src, int N, int K) {
  h16 *d = (h16 *)malloc(sizeof(h16) * (size_t)N * K);
#pragma omp parallel for schedule(static)
  for (int n = 0; n < N; n++) transpose_row_h16((const h16 *)src + (size_t)n * K, d + (size_t)n * K, K);
  return d;
}
static h16 *dup_h(const uint16_t *src, size_t n) {
  h16 *d = (h16 *)malloc(sizeof(h16) * n);
  memcpy(d, src, sizeof(h16) * n);
  return d;
}
static float *dup_f(const float *src, size_t n) {
  float *d = (float *)malloc(sizeof(float) * n);
  memcpy(d, src, sizeof(float) * n);
  return d;
}

/* OpenMP team size of every parallel loop below (bench.py picks the fastest for the host it runs on: on a box whose
 * container sees more logical CPUs than it may use, the default of one thread per CPU is several times slower). */
void orc_set_threads(int n) {
#ifdef _OPENMP
  omp_set_num_threads(n > 0 ? n : 1);
#else
  (void)n;
#endif
}
int orc_max_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

void *orc_dec_create(int n_layers, int vocab, int tmax) {
  orc_dec *o = (orc_dec *)calloc(1, sizeof(orc_dec));
  o->n_layers = n_layers;
  o->vocab = vocab;
  o->tmax = tmax;
  o->L = (orc_layer *)calloc(n_layers, sizeof(orc_layer));
  size_t kv = (size_t)n_layers * NHEAD * tmax * HD;
  o->kc = (h16 *)calloc(kv, sizeof(h16));
  o->vc = (h16 *)calloc(kv, sizeof(h16));
  return o;
}

void orc_dec_set_layer(void *h, int i, const uint16_t *wq, const uint16_t *bq, const uint16_t *wk, const uint16_t *bk,
                       const uint16_t *wv, const uint16_t *bv, const uint16_t *wo, const uint16_t *bo,
                       const uint16_t *w1, const uint16_t *b1, const uint16_t *w2, const uint16_t *b2,
                       const float *ln1g, const float *ln1b, const float *ln2g, const float *ln2b) {
  orc_layer *l = &((orc_dec *)h)->L[i];
  l->wq = dup_T(wq, HID, HID); l->wk = dup_T(wk, HID, HID); l->wv = dup_T(wv, HID, HID); l->wo = dup_T(wo, HID, HID);
  l->w1 = dup_T(w1, FFN, HID); l->w2 = dup_T(w2, HID, FFN);
  l->bq = dup_h(bq, HID); l->bk = dup_h(bk, HID); l->bv = dup_h(bv, HID); l->bo = dup_h(bo, HID);
  l->b1 = dup_h(b1, FFN); l->b2 = dup_h(b2, HID);
  l->ln1g = dup_f(ln1g, HID); l->ln1b = dup_f(ln1b, HID); l->ln2g = dup_f(ln2g, HID); l->ln2b = dup_f(ln2b, HID);
}

/* codebook16 [codebook][1024], input_layer W16 [1024][1024] b16 [1024]: builds tok_table with the canonical linear */
void orc_dec_set_globals(void *h, const uint16_t *lm_head, const uint16_t *codebook16, int codebook,
                         const uint16_t *in_w, const uint16_t *in_b, const float *extra, const float *tok_pos,
                         const float *cond, const float *pos, int npos) {
  orc_dec *o = (orc_dec *)h;
  o->lm_head = dup_T(lm_head, o->vocab, HID);
  o->codebook = codebook;
  o->tok_table = (h16 *)malloc(sizeof(h16) * (size_t)codebook * HID);
  orc_linear(in_w, in_b, codebook16, codebook, HID, HID, 0, (uint16_t *)o->tok_table);
  o->extra = dup_f(extra, 3 * HID);
  o->tok_pos = dup_f(tok_pos, 12 * HID);
  o->cond = dup_f(cond, 2 * HID);
  o->pos = dup_f(pos, (size_t)npos * HID);
  o->npos = npos;
}

const uint16_t *orc_dec_tok_table(void *h) { return (const uint16_t *)((orc_dec *)h)->tok_table; }
int orc_dec_len(void *h) { return ((orc_dec *)h)->t; }
void orc_dec_reset(void *h) { ((orc_dec *)h)->t = 0; }

void orc_dec_destroy(void *h) {
  orc_dec *o = (orc_dec *)h;
  for (int i = 0; i < o->n_layers; i++) {
    orc_layer *l = &o->L[i];
    free(l->wq); free(l->wk); free(l->wv); free(l->wo); free(l->w1); free(l->w2);
    free(l->bq); free(l->bk); free(l->bv); free(l->bo); free(l->b1); free(l->b2);
    free(l->ln1g); free(l->ln1b); free(l->ln2g); free(l->ln2b);
  }
  free(o->L); free(o->lm_head); free(o->tok_table); free(o->extra); free(o->tok_pos); free(o->cond); free(o->pos);
  free(o->kc); free(o->vc); free(o);
}

/* y16[m][n] = fp16(dot + b) for M rows with weight reuse; xT [M][K] lane-transposed fp32 */
static void linear_T(const h16 *wT, const h16 *b, const float *xT, int M, int N, int K, int relu, h16 *y) {
#pragma omp parallel for schedule(static)
  for (int n = 0; n < N; n++) {
    float bf = b ? (float)b[n] : 0.0f;
    for (int m = 0; m < M; m++) {
      float acc = dot_canon_T(wT + (size_t)n * K, xT + (size_t)m * K, K);
      h16 r = (h16)(acc + bf);
      if (relu && (float)r < 0.0f) r = (h16)0.0f;
      y[(size_t)m * N + n] = r;
    }
  }
}

static void to_xT(const float *hrow, float *xT, int M, int K) { /* fp32 rows -> fp16 round -> transposed fp32 */
#pragma omp parallel for schedule(static)
  for (int m = 0; m < M; m++) {
    h16 tmp[4096];
    for (int i = 0; i < K; i++) tmp[i] = (h16)hrow[(size_t)m * K + i];
    transpose_x_f32(tmp, xT + (size_t)m * K, K);
  }
}
static void h16_to_xT(const h16 *rows, float *xT, int M, int K) {
#pragma omp parallel for schedule(static)
  for (int m = 0; m < M; m++) transpose_x_f32(rows + (size_t)m * K, xT + (size_t)m * K, K);
}

/* Runs M new tokens whose fp32 input embeddings (already incl. positions) are hid[M][1024], occupying
 * absolute positions t..t+M-1 (causal among themselves).  Writes fp16 logits of every row if
 * logits_all, else of the last row, to `logits`. (OPTDecoderLayer post-LN; modeling_opt.py:202-254) */
static void run_tokens(orc_dec *o, float *hid, int M, uint16_t *logits_, int logits_all) {
  h16 *logits = (h16 *)logits_;
  int T = o->tmax, t0 = o->t;
  float *xT = (float *)malloc(sizeof(float) * (size_t)M * FFN);
  h16 *q = (h16 *)malloc(sizeof(h16) * (size_t)M * HID);
  h16 *k = (h16 *)malloc(sizeof(h16) * (size_t)M * HID);
  h16 *v = (h16 *)malloc(sizeof(h16) * (size_t)M * HID);
  h16 *a = (h16 *)malloc(sizeof(h16) * (size_t)M * HID);
  h16 *y = (h16 *)malloc(sizeof(h16) * (size_t)M * HID);
  h16 *f = (h16 *)malloc(sizeof(h16) * (size_t)M * FFN);
  for (int li = 0; li < o->n_layers; li++) {
    orc_layer *l = &o->L[li];
    h16 *kc = o->kc + (size_t)li * NHEAD * T * HD, *vc = o->vc + (size_t)li * NHEAD * T * HD;
    to_xT(hid, xT, M, HID);
    linear_T(l->wq, l->bq, xT, M, HID, HID, 0, q);
    linear_T(l->wk, l->bk, xT, M, HID, HID, 0, k);
    linear_T(l->wv, l->bv, xT, M, HID, HID, 0, v);
    for (int m = 0; m < M; m++)
      for (int hh = 0; hh < NHEAD; hh++) {
        memcpy(kc + ((size_t)hh * T + t0 + m) * HD, k + (size_t)m * HID + hh * HD, HD * sizeof(h16));
        memcpy(vc + ((size_t)hh * T + t0 + m) * HD, v + (size_t)m * HID + hh * HD, HD * sizeof(h16));
      }
#pragma omp parallel for collapse(2) schedule(dynamic)
    for (int m = 0; m < M; m++)
      for (int hh = 0; hh < NHEAD; hh++)
        attention_head_canon(q + (size_t)m * HID + hh * HD, kc + (size_t)hh * T * HD, vc + (size_t)hh * T * HD, HD,
                             t0 + m + 1, a + (size_t)m * HID + hh * HD);
    h16_to_xT(a, xT, M, HID);
    linear_T(l->wo, l->bo, xT, M, HID, HID, 0, y);
#pragma omp parallel for schedule(static)
    for (int m = 0; m < M; m++) {
      float h[HID];
      for (int i = 0; i < HID; i++) h[i] = hid[(size_t)m * HID + i] + (float)y[(size_t)m * HID + i];
      layernorm_canon(h, l->ln1g, l->ln1b, MA_LN_EPS, hid + (size_t)m * HID, HID);
    }
    to_xT(hid, xT, M, HID);
    linear_T(l->w1, l->b1, xT, M, FFN, HID, 1, f);
    h16_to_xT(f, xT, M, FFN);
    linear_T(l->w2, l->b2, xT, M, HID, FFN, 0, y);
#pragma omp parallel for schedule(static)
    for (int m = 0; m < M; m++) {
      float h[HID];
      for (int i = 0; i < HID; i++) h[i] = hid[(size_t)m * HID + i] + (float)y[(size_t)m * HID + i];
      layernorm_canon(h, l->ln2g, l->ln2b, MA_LN_EPS, hid + (size_t)m * HID, HID);
    }
  }
  /* no final_layer_norm / project_out for opt-350m (shape_opt.py:223-228,420-424); lm_head has no bias (:22) */
  if (logits) {
    if (logits_all) {
      to_xT(hid, xT, M, HID);
      linear_T(o->lm_head, NULL, xT, M, o->vocab, HID, 0, logits);
    } else {
      to_xT(hid + (size_t)(M - 1) * HID, xT, 1, HID);
      linear_T(o->lm_head, NULL, xT, 1, o->vocab, HID, 0, logits);
    }
  }
  o->t = t0 + M;
  free(xT); free(q); free(k); free(v); free(a); free(y); free(f);
}

/* step 0 of generate(): inputs_embeds = prefix + cond_embed(0) (shape_opt.py:331-337), + positions
 * rows 2..258 (modeling_opt.py:61-71), hidden = emb + pos (shape_opt.py:364). */
void orc_dec_prefill(void *h, const float *prefix, int n, uint16_t *logits, float *hidden_out) {
  orc_dec *o = (orc_dec *)h;
  float *hid = (float *)malloc(sizeof(float) * (size_t)n * HID);
  for (int s = 0; s < n; s++)
    for (int i = 0; i < HID; i++)
      hid[(size_t)s * HID + i] = (prefix[(size_t)s * HID + i] + o->cond[i]) + o->pos[(size_t)(o->t + s + 2) * HID + i];
  run_tokens(o, hid, n, logits, 0);
  if (hidden_out) memcpy(hidden_out, hid, sizeof(float) * (size_t)n * HID);
  free(hid);
}

/* one decode step: token `tok` is the gen_count-th generated token (gen_count >= 1), shape_opt.py:318-328 */
void orc_dec_step(void *h, int tok, int gen_count, uint16_t *logits, float *hidden_out) {
  orc_dec *o = (orc_dec *)h;
  float hid[HID];
  const float *F, *C = o->cond + HID, *P = o->pos + (size_t)(o->t + 2) * HID;
  if (tok < 3) {
    F = o->tok_pos + (size_t)tok * HID; /* specials use their own id (shape_opt.py:455-458) */
    for (int i = 0; i < HID; i++) hid[i] = ((o->extra[(size_t)tok * HID + i] + F[i]) + C[i]) + P[i];
  } else {
    int r = (gen_count - 2) % 9;
    if (r < 0) r += 9; /* torch remainder is floored */
    F = o->tok_pos + (size_t)(r + 3) * HID;
    const h16 *X = o->tok_table + (size_t)(tok - 3) * HID;
    for (int i = 0; i < HID; i++) hid[i] = (((float)X[i] + F[i]) + C[i]) + P[i];
  }
  run_tokens(o, hid, 1, logits, 0);
  if (hidden_out) memcpy(hidden_out, hid, sizeof(float) * HID);
}

/* read back a cache row for tests: kv 0 = K, 1 = V */
void orc_dec_get_kv(void *h, int layer, int kv, int pos, uint16_t *out) {
  orc_dec *o = (orc_dec *)h;
  const h16 *c = (kv ? o->vc : o->kc) + (size_t)layer * NHEAD * o->tmax * HD;
  for (int hh = 0; hh < NHEAD; hh++) memcpy(out + hh * HD, c + ((size_t)hh * o->tmax + pos) * HD, HD * sizeof(h16));
}
