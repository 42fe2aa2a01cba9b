// api_encoder.cu -- ma_encoder_forward (a1-a8) and ma_detokenize (a17-a18): host orchestration of the
// canonical Linear / LayerNorm / attention kernels plus the glue kernels of glue.cu.
//
// dtype flow mirrors the reference under fp16 autocast (SURVEY.md 8a): Linear in/out fp16 with fp32
// accumulation, LayerNorm and softmax statistics fp32, fp32 residual stream in the encoder's cross /
// self-attention stack and in BERT, fp16 residual stream in the 16 "transformer" blocks after post_kl.
#include <algorithm>

#include "canon.cuh"
#include "internal.h"
#include "internal_enc.h"

namespace ma {

constexpr int EW = 768, EH = 12, NPTS = 4096, NLAT = 257;
constexpr int ENC_CHUNK = 8;  // shapes per pass

static inline size_t al(size_t x) { return (x + 255) / 256 * 256; }

struct Carver {
  char* base;
  size_t off = 0;
  explicit Carver(void* b) : base((char*)b) {}
  template <typename T>
  T* take(size_t n) {
    T* p = base ? (T*)(base + off) : nullptr;
    off += al(n * sizeof(T));
    return p;
  }
};

struct EncWs {
  __half *data16, *dproj16, *lnd16, *kv16, *kh, *vh;  // 4096-row buffers
  float* x32;                                         // residual stream [rows][768]
  __half *x16r, *ln16, *q16, *qkv16, *qh, *attn16, *y16, *f16, *lat16, *cat16, *out16;
  int* nkeys;
  void* attn_scratch;
  size_t attn_scratch_bytes, total;
};

static EncWs carve_enc(void* base, int Bc) {
  Carver c(base);
  EncWs w;
  const size_t P = (size_t)Bc * NPTS, R = (size_t)Bc * NLAT;
  w.data16 = c.take<__half>(P * 256);
  w.dproj16 = c.take<__half>(P * EW);
  w.lnd16 = c.take<__half>(P * EW);
  w.kv16 = c.take<__half>(P * 2 * EW);
  w.kh = c.take<__half>(P * EW);
  w.vh = c.take<__half>(P * EW);
  w.x32 = c.take<float>(R * EW);
  w.x16r = c.take<__half>(R * EW);
  w.ln16 = c.take<__half>(R * EW);
  w.q16 = c.take<__half>(R * EW);
  w.qkv16 = c.take<__half>(R * 3 * EW);
  w.qh = c.take<__half>(R * EW);
  w.attn16 = c.take<__half>(R * EW);
  w.y16 = c.take<__half>(R * EW);
  w.f16 = c.take<__half>(R * 4 * EW);
  w.lat16 = c.take<__half>(R * 256);
  w.cat16 = c.take<__half>(R * 2 * EW);
  w.out16 = c.take<__half>(R * 1024);
  w.nkeys = c.take<int>(R);
  w.attn_scratch_bytes = attention_scratch_bytes((int)R, EH, NPTS);
  w.attn_scratch = c.take<char>(w.attn_scratch_bytes);
  w.total = c.off;
  return w;
}

#define TRY(x) do { if (x) return 1; } while (0)

static int g_use_tc = 2;  // 0: canonical CUDA-core kernels; 1: GEMMs of the encoder / detokenizer on the tensor cores;
                          // 2: their attention on the tensor cores too (ma_set_tensor_cores)

// nn.Linear of the tolerance-checked stages: tensor cores when the shape allows, canonical CUDA-core kernel otherwise
static unsigned long long g_tc_calls = 0, g_tc_fallbacks = 0;   // Linear calls of these stages: on the tensor cores / not tileable
static int enc_linear(const __half* W, const __half* bias, const __half* x, int ldx, __half* y, int ldy, int M, int N,
                      int K, int epi, cudaStream_t st) {
  if (g_use_tc && linear_tc_supported(M, N, K, ldx, ldy, x, W, y)) {
    g_tc_calls++;
    return launch_linear_tc(W, bias, x, ldx, y, ldy, M, N, K, epi, st);
  }
  if (g_use_tc) g_tc_fallbacks++;   // small-M / odd shapes (cond_head_proj on 1 row per shape, pre_kl N = 128 ...)
  return launch_linear(W, bias, x, ldx, y, ldy, M, N, K, epi, st);
}

// Dense attention of n_slots x rows_per_slot queries over the n keys of their slot.  q [rows][ldq] (head h at 64h), kh
// [slot][H][n][64] already scattered; V is still in its source matrix (vsrc, vld, vcol0, vstride as for
// scatter_heads) and is laid out here the way the chosen kernel wants it: transposed + zero-padded for the tensor-core attention, head-
// major for the canonical kernel.
static int enc_attention(const __half* q, int ldq, const __half* kh, const __half* vsrc, int vld, int vcol0,
                         int vstride, __half* vbuf, int n, int rows_per_slot, int n_slots, const int* nkeys,
                         __half* out, void* scratch, cudaStream_t st) {
  const long Tpad = ((long)n + 127) / 128 * 128;
  if (g_use_tc >= 2 && attention_tc_supported(ldq, EW, n, Tpad, n, q, kh, vbuf, out)) {
    TRY(launch_scatter_heads_t(vsrc, vld, vcol0, vstride, EH, n, Tpad, n_slots, vbuf, st));
    return launch_attention_tc(q, ldq, kh, vbuf, n, Tpad, EH, rows_per_slot, n_slots, n, 0.125f, out, EW, st);
  }
  const long rows = (long)n_slots * n;
  TRY(launch_scatter_heads(vsrc, vld, vcol0, vstride, EH, n, n, vbuf, rows, st));
  return launch_attention(q, ldq, kh, vbuf, n, EH, rows_per_slot, nullptr, nkeys, n, n_slots * rows_per_slot, 0.125f, out,
                          EW, scratch, st);
}

// x += c_proj(attn(c_qkv(ln_1 x))) ; x += c_proj(gelu(c_fc(ln_2 x)))   (transformer_blocks.py:109-112)
// n tokens per shape; residual stream fp32 (x32) or fp16 (x16r).
static int miche_block(const ma_miche_block& b, const EncWs& w, int Bc, int n, bool fp16_stream, cudaStream_t st) {
  const int M = Bc * n;
  if (fp16_stream) TRY(launch_layernorm(nullptr, w.x16r, b.ln1_g, b.ln1_b, MA_LN_EPS, M, EW, nullptr, w.ln16, st));
  else TRY(launch_layernorm(w.x32, nullptr, b.ln1_g, b.ln1_b, MA_LN_EPS, M, EW, nullptr, w.ln16, st));
  TRY(enc_linear((const __half*)b.c_qkv_w, nullptr, w.ln16, EW, w.qkv16, 3 * EW, M, 3 * EW, EW, MA_EPI_NONE, st));
  // qkv viewed [B,n,12,192]: head h = columns 192h .. 192h+191 = q | k | v  (transformer_blocks.py:60-62)
  TRY(launch_scatter_heads(w.qkv16, 3 * EW, 0, 192, EH, 1, 1, w.qh, M, st));
  TRY(launch_scatter_heads(w.qkv16, 3 * EW, 64, 192, EH, n, n, w.kh, M, st));
  TRY(launch_fill_i32(w.nkeys, n, M, st));
  TRY(enc_attention(w.qh, EW, w.kh, w.qkv16, 3 * EW, 128, 192, w.vh, n, n, Bc, w.nkeys, w.attn16, w.attn_scratch, st));
  TRY(enc_linear((const __half*)b.c_proj_w, (const __half*)b.c_proj_b, w.attn16, EW, w.y16, EW, M, EW, EW,
                    MA_EPI_NONE, st));
  TRY(launch_residual_add(fp16_stream ? nullptr : w.x32, w.x16r, w.y16, (long)M * EW, st));
  if (fp16_stream) TRY(launch_layernorm(nullptr, w.x16r, b.ln2_g, b.ln2_b, MA_LN_EPS, M, EW, nullptr, w.ln16, st));
  else TRY(launch_layernorm(w.x32, nullptr, b.ln2_g, b.ln2_b, MA_LN_EPS, M, EW, nullptr, w.ln16, st));
  TRY(enc_linear((const __half*)b.fc_w, (const __half*)b.fc_b, w.ln16, EW, w.f16, 4 * EW, M, 4 * EW, EW, MA_EPI_GELU,
                    st));
  TRY(enc_linear((const __half*)b.proj_w, (const __half*)b.proj_b, w.f16, 4 * EW, w.y16, EW, M, EW, 4 * EW,
                    MA_EPI_NONE, st));
  TRY(launch_residual_add(fp16_stream ? nullptr : w.x32, w.x16r, w.y16, (long)M * EW, st));
  return 0;
}

static int encoder_chunk(const ma_encoder_weights* e, const __half* pc, int Bc, float* point_feature, float* prefix,
                         const EncWs& w, cudaStream_t st) {
  const long P = (long)Bc * NPTS;
  const int R = Bc * NLAT;
  // a1/a2: Fourier features + normals -> input_proj (sal_perceiver.py:87-90)
  TRY(launch_fourier_embed(pc, P, w.data16, st));
  TRY(enc_linear((const __half*)e->input_proj_w, (const __half*)e->input_proj_b, w.data16, 256, w.dproj16, EW, (int)P,
                    EW, 256, MA_EPI_NONE, st));
  // a3: cross attention block (transformer_blocks.py:223-226): x = query
  TRY(launch_convert_rows(e->query, 0, EW, w.x32, 0, EW, R, EW, NLAT, st));
  TRY(launch_layernorm(w.x32, nullptr, e->ln1_g, e->ln1_b, MA_LN_EPS, R, EW, nullptr, w.ln16, st));
  TRY(enc_linear((const __half*)e->cq_w, nullptr, w.ln16, EW, w.q16, EW, R, EW, EW, MA_EPI_NONE, st));
  TRY(launch_layernorm(nullptr, w.dproj16, e->ln2_g, e->ln2_b, MA_LN_EPS, (int)P, EW, nullptr, w.lnd16, st));
  TRY(enc_linear((const __half*)e->ckv_w, nullptr, w.lnd16, EW, w.kv16, 2 * EW, (int)P, 2 * EW, EW, MA_EPI_NONE, st));
  // kv viewed [B,4096,12,128]: head h = columns 128h..: k | v  (transformer_blocks.py:171-173)
  TRY(launch_scatter_heads(w.kv16, 2 * EW, 0, 128, EH, NPTS, NPTS, w.kh, P, st));
  TRY(launch_fill_i32(w.nkeys, NPTS, R, st));
  TRY(enc_attention(w.q16, EW, w.kh, w.kv16, 2 * EW, 64, 128, w.vh, NPTS, NLAT, Bc, w.nkeys, w.attn16, w.attn_scratch,
                    st));
  TRY(enc_linear((const __half*)e->cproj_w, (const __half*)e->cproj_b, w.attn16, EW, w.y16, EW, R, EW, EW,
                    MA_EPI_NONE, st));
  TRY(launch_residual_add(w.x32, nullptr, w.y16, (long)R * EW, st));
  TRY(launch_layernorm(w.x32, nullptr, e->ln3_g, e->ln3_b, MA_LN_EPS, R, EW, nullptr, w.ln16, st));
  TRY(enc_linear((const __half*)e->fc_w, (const __half*)e->fc_b, w.ln16, EW, w.f16, 4 * EW, R, 4 * EW, EW, MA_EPI_GELU,
                    st));
  TRY(enc_linear((const __half*)e->proj_w, (const __half*)e->proj_b, w.f16, 4 * EW, w.y16, EW, R, EW, 4 * EW,
                    MA_EPI_NONE, st));
  TRY(launch_residual_add(w.x32, nullptr, w.y16, (long)R * EW, st));
  // a4: 8 self-attention blocks over the 257 latents, then ln_post -> point_feature (fp32)
  for (int i = 0; i < 8; i++) TRY(miche_block(e->enc[i], w, Bc, NLAT, false, st));
  TRY(launch_layernorm(w.x32, nullptr, e->lnpost_g, e->lnpost_b, MA_LN_EPS, R, EW, point_feature, w.ln16, st));
  // a8: prefix[:,0] = cond_head_proj(pf[:,0])   (row 0 of every shape: input rows are NLAT*EW apart)
  TRY(enc_linear((const __half*)e->cond_head_w, (const __half*)e->cond_head_b, w.ln16, NLAT * EW, w.out16, 1024, Bc,
                    1024, EW, MA_EPI_NONE, st));
  TRY(launch_convert_rows(w.out16, 1, 1024, prefix, 0, (long)NLAT * 1024, Bc, 1024, 0, st));
  // a7: to_shape_latents: pre_kl -> mean (first 64 channels) -> post_kl -> 16 blocks with an fp16 stream
  const int L = Bc * 256;
  for (int b = 0; b < Bc; b++)  // latent rows 1..256 of each shape, fp16, packed [256*Bc][768]
    TRY(launch_convert_rows(w.ln16 + ((size_t)b * NLAT + 1) * EW, 1, EW, w.cat16 + (size_t)b * 256 * 2 * EW, 1, 2 * EW,
                            256, EW, 0, st));
  TRY(enc_linear((const __half*)e->pre_kl_w, (const __half*)e->pre_kl_b, w.cat16, 2 * EW, w.y16, 128, L, 128, EW,
                    MA_EPI_NONE, st));
  cudaMemsetAsync(w.lat16, 0, (size_t)L * 256 * sizeof(__half), st);
  TRY(launch_convert_rows(w.y16, 1, 128, w.lat16, 1, 256, L, 64, 0, st));
  TRY(enc_linear((const __half*)e->post_kl_w, (const __half*)e->post_kl_b, w.lat16, 256, w.x16r, EW, L, EW, 256,
                    MA_EPI_NONE, st));
  for (int i = 0; i < 16; i++) TRY(miche_block(e->dec[i], w, Bc, 256, true, st));
  // prefix[:,1:] = cond_proj(cat[pf[:,1:], shape_latents])   (meshanything.py:130)
  TRY(launch_convert_rows(w.x16r, 1, EW, w.cat16 + EW, 1, 2 * EW, L, EW, 0, st));
  TRY(enc_linear((const __half*)e->cond_w, (const __half*)e->cond_b, w.cat16, 2 * EW, w.out16, 1024, L, 1024, 2 * EW,
                    MA_EPI_NONE, st));
  for (int b = 0; b < Bc; b++)
    TRY(launch_convert_rows(w.out16 + (size_t)b * 256 * 1024, 1, 1024, prefix + ((size_t)b * NLAT + 1) * 1024, 0, 1024,
                            256, 1024, 0, st));
  return 0;
}

// ---- detokenizer ---------------------------------------------------------------------------------
constexpr int DET_CHUNK = 8;

struct DetWs {
  __half *code16, *face16, *pf16, *pfin16, *x16, *qkv16, *qh, *kh, *vh, *attn16, *y16, *f16, *logits16;
  float *x32, *tmp32;
  int *mask, *nkeys;
  void* attn_scratch;
  size_t attn_scratch_bytes, total;
};

static DetWs carve_det(void* base, int Bc, int F) {
  Carver c(base);
  DetWs w;
  const size_t S = (size_t)(NLAT + F), R = (size_t)Bc * S, BF = (size_t)Bc * F, BP = (size_t)Bc * NLAT;
  w.code16 = c.take<__half>(BF * 3072);
  w.face16 = c.take<__half>(BF * EW);
  w.pfin16 = c.take<__half>(BP * EW);
  w.pf16 = c.take<__half>(BP * EW);
  w.x16 = c.take<__half>(R * EW);
  w.qkv16 = c.take<__half>(R * 3 * EW);
  w.qh = c.take<__half>(R * EW);
  w.kh = c.take<__half>(R * EW);
  w.vh = c.take<__half>((size_t)Bc * ((S + 127) / 128 * 128) * EW);  // room for V^T padded to 128 keys (tensor-core path)
  w.attn16 = c.take<__half>(R * EW);
  w.y16 = c.take<__half>(R * EW);
  w.f16 = c.take<__half>(R * 4 * EW);
  w.logits16 = c.take<__half>(BF * 1152);
  w.x32 = c.take<float>(R * EW);
  w.tmp32 = c.take<float>(R * EW);
  w.mask = c.take<int>(BF);
  w.nkeys = c.take<int>(R);
  w.attn_scratch_bytes = attention_scratch_bytes((int)R, EH, (int)S);
  w.attn_scratch = c.take<char>(w.attn_scratch_bytes);
  w.total = c.off;
  return w;
}

static int detok_chunk(const ma_tokenizer_weights* t, const int32_t* gen_ids, int max_new, int Bc, int F,
                       const float* point_feature, float* out_xyz, int32_t* ids_out, const DetWs& w, cudaStream_t st) {
  const int S = NLAT + F, R = Bc * S, BF = Bc * F, BP = Bc * NLAT;
  // process_point_feature (meshanything.py:42-48)
  TRY(launch_convert_rows(point_feature, 0, EW, w.pfin16, 1, EW, BP, EW, 0, st));
  TRY(enc_linear((const __half*)t->cond_w, (const __half*)t->cond_b, w.pfin16, EW, w.pf16, EW, BP, EW, EW, MA_EPI_NONE,
                    st));
  // row 0 of every shape uses cond_head_proj instead
  TRY(enc_linear((const __half*)t->cond_head_w, (const __half*)t->cond_head_b, w.pfin16, NLAT * EW, w.y16, EW, Bc, EW,
                    EW, MA_EPI_NONE, st));
  TRY(launch_convert_rows(w.y16, 1, EW, w.pf16, 1, (long)NLAT * EW, Bc, EW, 0, st));
  TRY(launch_add_table(w.pf16, nullptr, t->point_pe, NLAT, w.tmp32, BP, st));
  // faces (meshanything.py:54-60): codes -> project_down_codebook -> mask -> + pos_embedding -> LN
  TRY(launch_gather_codes(gen_ids, max_new, Bc, F, t->codebook, w.code16, w.mask, ids_out, st));
  TRY(enc_linear((const __half*)t->down_w, (const __half*)t->down_b, w.code16, 3072, w.face16, EW, BF, EW, 3072,
                    MA_EPI_NONE, st));
  TRY(launch_add_table(w.face16, w.mask, t->pos_embedding, F, w.tmp32 + (size_t)BP * EW, BF, st));
  // LayerNorms write straight into the concatenated [Bc][257+F][768] stream
  for (int b = 0; b < Bc; b++) {
    TRY(launch_layernorm(w.tmp32 + (size_t)b * NLAT * EW, nullptr, t->pln_g, t->pln_b, MA_LN_EPS, NLAT, EW,
                         w.x32 + (size_t)b * S * EW, w.x16 + (size_t)b * S * EW, st));
    TRY(launch_layernorm(w.tmp32 + ((size_t)BP + (size_t)b * F) * EW, nullptr, t->ln_g, t->ln_b, MA_LN_EPS, F, EW,
                         w.x32 + ((size_t)b * S + NLAT) * EW, w.x16 + ((size_t)b * S + NLAT) * EW, st));
  }
  TRY(launch_fill_i32(w.nkeys, S, R, st));
  for (int i = 0; i < t->n_layers; i++) {  // BERT post-LN layer, no attention mask (meshanything.py:62-64)
    const ma_bert_layer& l = t->layer[i];
    TRY(enc_linear((const __half*)l.in_w, (const __half*)l.in_b, w.x16, EW, w.qkv16, 3 * EW, R, 3 * EW, EW, MA_EPI_NONE,
                      st));
    TRY(launch_scatter_heads(w.qkv16, 3 * EW, 0, 64, EH, 1, 1, w.qh, R, st));
    TRY(launch_scatter_heads(w.qkv16, 3 * EW, EW, 64, EH, S, S, w.kh, R, st));
    TRY(enc_attention(w.qh, EW, w.kh, w.qkv16, 3 * EW, 2 * EW, 64, w.vh, S, S, Bc, w.nkeys, w.attn16, w.attn_scratch,
                      st));
    TRY(enc_linear((const __half*)l.out_w, (const __half*)l.out_b, w.attn16, EW, w.y16, EW, R, EW, EW, MA_EPI_NONE, st));
    TRY(launch_layernorm(w.x32, w.y16, l.n1_g, l.n1_b, 1e-12f, R, EW, w.x32, w.x16, st));
    TRY(enc_linear((const __half*)l.l1_w, (const __half*)l.l1_b, w.x16, EW, w.f16, 4 * EW, R, 4 * EW, EW, MA_EPI_GELU,
                      st));
    TRY(enc_linear((const __half*)l.l2_w, (const __half*)l.l2_b, w.f16, 4 * EW, w.y16, EW, R, EW, 4 * EW, MA_EPI_NONE,
                      st));
    TRY(launch_layernorm(w.x32, w.y16, l.n2_g, l.n2_b, 1e-12f, R, EW, w.x32, w.x16, st));
  }
  // decoded[:, 257:] -> to_coor_logits -> argmax -> undiscretize (masked faces -> NaN)
  for (int b = 0; b < Bc; b++)
    TRY(enc_linear((const __half*)t->coor_w, (const __half*)t->coor_b, w.x16 + ((size_t)b * S + NLAT) * EW, EW,
                      w.logits16 + (size_t)b * F * 1152, 1152, F, 1152, EW, MA_EPI_NONE, st));
  TRY(launch_coords(w.logits16, w.mask, out_xyz, BF, st));
  return 0;
}

}  // namespace ma

using namespace ma;

extern "C" {

void ma_tensor_core_linear_counts(unsigned long long* on_tensor_cores, unsigned long long* canonical_fallback) {
  if (on_tensor_cores) *on_tensor_cores = g_tc_calls;
  if (canonical_fallback) *canonical_fallback = g_tc_fallbacks;
}

int ma_set_tensor_cores(int enable) {
  const int old = g_use_tc;
  g_use_tc = enable < 0 ? 0 : (enable > 2 ? 2 : enable);
  return old;
}

int ma_attention_tc_f16(const void* q, int ldq, const void* K, const void* Vt, long T, long Tpad, int H,
                        int rows_per_slot, int n_slots, int nkeys, float scale, void* out, int ldo, void* stream) {
  return launch_attention_tc((const __half*)q, ldq, (const __half*)K, (const __half*)Vt, T, Tpad, H, rows_per_slot,
                             n_slots, nkeys, scale, (__half*)out, ldo, (cudaStream_t)stream);
}

int ma_transpose_heads_f16(const void* src, int ld, int col0, int head_stride, int H, int n, long Tpad, int n_slots,
                           void* dst, void* stream) {
  return launch_scatter_heads_t((const __half*)src, ld, col0, head_stride, H, n, Tpad, n_slots, (__half*)dst,
                                (cudaStream_t)stream);
}

int ma_linear_tc_f16(const void* W, const void* bias, const void* x, int ldx, void* y, int ldy, int M, int N, int K,
                     int epilogue, void* stream) {
  if (!linear_tc_supported(M, N, K, ldx, ldy, x, W, y)) {
    set_error("ma_linear_tc_f16: unsupported shape (M >= 64, N %% 128 == 0, K %% 64 == 0, 16-byte alignment)");
    return 1;
  }
  return launch_linear_tc((const __half*)W, (const __half*)bias, (const __half*)x, ldx, (__half*)y, ldy, M, N, K, epilogue,
                          (cudaStream_t)stream);
}

// ---- test hooks: the glue kernels of glue.cu, one entry point per launcher.  Each refuses what its kernel cannot take
// (null pointers, non-positive counts, a width or an alignment its vector accesses need) before anything is launched.
static bool aligned(const void* p, int bytes) { return ((uintptr_t)p & (uintptr_t)(bytes - 1)) == 0; }

int ma_fourier_embed_f16(const void* pc, long rows, void* out, void* stream) {
  if (!pc || !out || rows <= 0 || !aligned(out, 8)) {
    set_error("ma_fourier_embed_f16: bad arguments (non-null pointers, rows > 0, out 8-byte aligned)");
    return 1;
  }
  return launch_fourier_embed((const __half*)pc, rows, (__half*)out, (cudaStream_t)stream);
}

int ma_scatter_heads_f16(const void* src, int ld, int col0, int head_stride, int H, int rows_per_slot, long T, void* dst,
                         long rows, void* stream) {
  if (!src || !dst || ld <= 0 || col0 < 0 || head_stride < 0 || H <= 0 || rows_per_slot <= 0 || T <= 0 || rows <= 0 ||
      ld % 8 || col0 % 8 || head_stride % 8 || !aligned(src, 16) || !aligned(dst, 16)) {
    set_error("ma_scatter_heads_f16: bad arguments (non-null 16-byte aligned pointers, positive counts, ld, col0 and "
              "head_stride multiples of 8)");
    return 1;
  }
  return launch_scatter_heads((const __half*)src, ld, col0, head_stride, H, rows_per_slot, T, (__half*)dst, rows,
                              (cudaStream_t)stream);
}

int ma_residual_add(float* x32, void* x16, const void* y, long n, void* stream) {
  if (!y || !x32 == !x16 || n <= 0 || n % 4 || !aligned(y, 8) || !aligned(x32, 16) || !aligned(x16, 8)) {
    set_error("ma_residual_add: bad arguments (exactly one of x32 / x16, y non-null, n > 0 and n %% 4 == 0, aligned)");
    return 1;
  }
  return launch_residual_add(x32, (__half*)x16, (const __half*)y, n, (cudaStream_t)stream);
}

int ma_convert_rows(const void* src, int src_f16, long lds, void* dst, int dst_f16, long ldd, long rows, int cols,
                    long src_rows_mod, void* stream) {
  if (!src || !dst || lds <= 0 || ldd <= 0 || rows <= 0 || cols <= 0 || cols % 4 || src_rows_mod < 0) {
    set_error("ma_convert_rows: bad arguments (non-null pointers, positive strides and counts, cols %% 4 == 0, "
              "src_rows_mod >= 0)");
    return 1;
  }
  return launch_convert_rows(src, src_f16, lds, dst, dst_f16, ldd, rows, cols, src_rows_mod, (cudaStream_t)stream);
}

int ma_add_table(const void* y16, const int* mask, const float* table, int table_rows, float* out, long rows,
                 void* stream) {
  if (!y16 || !table || !out || table_rows <= 0 || rows <= 0 || !aligned(y16, 8) || !aligned(table, 16) ||
      !aligned(out, 16)) {
    set_error("ma_add_table: bad arguments (non-null aligned y16 / table / out, positive counts)");
    return 1;
  }
  return launch_add_table((const __half*)y16, mask, table, table_rows, out, rows, (cudaStream_t)stream);
}

int ma_gather_codes(const int32_t* gen_ids, int max_new, int B, int F, const float* codebook, void* code16, int* mask,
                    int32_t* ids_out, void* stream) {
  if (!gen_ids || !codebook || !code16 || !mask || max_new <= 0 || B <= 0 || F <= 0) {
    set_error("ma_gather_codes: bad arguments (non-null pointers, positive counts)");
    return 1;
  }
  return launch_gather_codes(gen_ids, max_new, B, F, codebook, (__half*)code16, mask, ids_out, (cudaStream_t)stream);
}

int ma_coords(const void* logits, const int* mask, float* xyz, long faces, void* stream) {
  if (!logits || !mask || !xyz || faces <= 0) {
    set_error("ma_coords: bad arguments (non-null pointers, faces > 0)");
    return 1;
  }
  return launch_coords((const __half*)logits, mask, xyz, faces, (cudaStream_t)stream);
}

size_t ma_encoder_workspace_bytes(int B) { return carve_enc(nullptr, std::min(B, ENC_CHUNK)).total; }

int ma_encoder_forward(const ma_encoder_weights* e, const void* pc_normal, int B, float* point_feature, float* prefix,
                       void* ws, void* stream) {
  if (!e || !pc_normal || !point_feature || !prefix || !ws || B <= 0) {
    set_error("ma_encoder_forward: bad arguments");
    return 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  for (int b0 = 0; b0 < B; b0 += ENC_CHUNK) {
    const int Bc = std::min(ENC_CHUNK, B - b0);
    EncWs w = carve_enc(ws, Bc);
    cudaMemsetAsync(w.attn_scratch, 0, w.attn_scratch_bytes, st);
    if (encoder_chunk(e, (const __half*)pc_normal + (size_t)b0 * NPTS * 6, Bc, point_feature + (size_t)b0 * NLAT * EW,
                      prefix + (size_t)b0 * NLAT * 1024, w, st))
      return 1;
  }
  return 0;
}

size_t ma_detokenize_workspace_bytes(int B, int F) { return carve_det(nullptr, std::min(B, DET_CHUNK), F).total; }

int ma_detokenize(const ma_tokenizer_weights* t, const int32_t* gen_ids, int max_new, int B, int F,
                  const float* point_feature, float* out_xyz, int32_t* ids_out, void* ws, void* stream) {
  if (!t || !gen_ids || !point_feature || !out_xyz || !ws || B <= 0 || F <= 0 || max_new != 9 * F + 2) {
    set_error("ma_detokenize: bad arguments (max_new must be 9F+2)");
    return 1;
  }
  if (F > 18000 || (long)(NLAT + F) * std::min(B, DET_CHUNK) > 65535) {
    set_error("ma_detokenize: F=%d too large", F);
    return 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  for (int b0 = 0; b0 < B; b0 += DET_CHUNK) {
    const int Bc = std::min(DET_CHUNK, B - b0);
    DetWs w = carve_det(ws, Bc, F);
    cudaMemsetAsync(w.attn_scratch, 0, w.attn_scratch_bytes, st);
    if (detok_chunk(t, gen_ids + (size_t)b0 * max_new, max_new, Bc, F, point_feature + (size_t)b0 * NLAT * EW,
                    out_xyz + (size_t)b0 * F * 9, ids_out ? ids_out + (size_t)b0 * F * 9 : nullptr, w, st))
      return 1;
  }
  return 0;
}

}  // extern "C"
