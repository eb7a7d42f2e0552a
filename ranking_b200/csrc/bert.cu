// K15 TFR-BERT (extension/premade/tfrbert_task.py): a post-LN BERT encoder over every
// (query, document) token sequence of a list, the tanh pooler on its [CLS] row, Dropout and
// Dense(1).  The math is written out in include/tfr_b200.h; this file is the glue around the
// DIN's pieces (din.cuh):
//
//   x0   = LN_e(Word[w] + Pos[t] + Type[k]), dropped    emb_ln_fwd_kernel (gather + LN + dropout)
//   per layer:
//     qkv = x [Wq | Wk | Wv] + b                       one GEMM, packed kernel [E, 3E]
//     o    = softmax(q k / sqrt(dh) - 1e9 [token masked]) (dropped) v
//                                                      din_attn_* (SIMT) / din_tc_attn_* (wgmma)
//     x'   = LN_1(drop(o Wo + bo) + x)                 GEMM + ln_fwd_kernel
//     a    = gelu(x' W1 + b1)                          GEMM (bias epilogue) + gelu_fwd_kernel
//     x''  = LN_2(drop(a W2 + b2) + x')                GEMM + ln_fwd_kernel
//   score = drop(tanh(x_L[CLS] Wp + bp)) . w_s + b_s    GEMM on the strided CLS rows + head kernel
//
// The backward walks the same steps in reverse.  LayerNorm dgamma / dbeta and every dW are
// per-CTA (per-split) partials reduced in fixed order, the attention core has no atomics and
// the embedding tables' gradients are tfr_embedding_bwd's radix-sorted segment sums, so two
// identical calls give identical bits.
#include <cstring>
#include <type_traits>

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "din.cuh"
#include "mlp.h"
#include "tc_gemm_bf16.cuh"

namespace tfr {
namespace {

constexpr float kLnEps = 1e-12f;
constexpr int kLnWarps = 8;   // rows per CTA of the LayerNorm kernels (one warp each)

struct BertPlan {
  int V, E, H, dh, I, NL, P, Tv;
  int S, L, M;
  float hdrop, adrop, sdrop;
  int passes;
  bool tc;
  bool h16;     // TFR_PREC_BF16 / TFR_PREC_FP16: 16-bit activations and GEMM operands (see the
                // 16-bit path below)
  bool f16;     // TFR_PREC_FP16: the 16-bit type is fp16, else bf16
  int sms;
  unsigned long long seed;
  // parameters (floats)
  size_t word, pos, type, emb_g;
  size_t layer0, layer_size, pool, n_params;
  // workspace (floats)
  size_t xs_off[TFR_BERT_MAX_LAYERS + 1];
  size_t xhe_off, rse_off, pos_ids_off;
  size_t qkv_off[TFR_BERT_MAX_LAYERS], o_off[TFR_BERT_MAX_LAYERS], lse_off[TFR_BERT_MAX_LAYERS];
  size_t xh1_off[TFR_BERT_MAX_LAYERS], rs1_off[TFR_BERT_MAX_LAYERS], x1_off[TFR_BERT_MAX_LAYERS];
  size_t u_off[TFR_BERT_MAX_LAYERS], a_off[TFR_BERT_MAX_LAYERS];
  size_t xh2_off[TFR_BERT_MAX_LAYERS], rs2_off[TFR_BERT_MAX_LAYERS];
  size_t pre_off, pooled_off;
  size_t g_off, dres_off, dy_off, tmp_off, do_off, dqkv_off, da_off, dsum_off, dpre_off;
  size_t part_off, part_stride, cs_off, cs_stride;
  size_t emb_ws_off, emb_ws_floats;
  int rows_per_split, splits, s_rows_per_split, s_splits;
  // 16-bit modes: the GEMM outputs y / y2 (consumed by the next LayerNorm), the [CLS] rows'
  // gradient, and the weight shadows W [in, out] (wb) and W^T [out, in] (wbt) of Wqkv, Wo, W1,
  // W2 per layer, then Wp, at the same 16-bit offsets in both
  size_t ytmp_off, dcls_off, wb_off, wbt_off, sh_layer, sh_total;
  size_t ws_floats;

  // per-layer parameter offsets: Wqkv [E, 3E], bqkv [3E], Wo [E, E], bo, gamma_1, beta_1,
  // W1 [E, I], b1 [I], W2 [I, E], b2, gamma_2, beta_2
  __host__ __device__ size_t wqkv(int l) const { return layer0 + (size_t)l * layer_size; }
  __host__ __device__ size_t bqkv(int l) const { return wqkv(l) + (size_t)E * 3 * E; }
  __host__ __device__ size_t wo(int l) const { return bqkv(l) + 3 * (size_t)E; }
  __host__ __device__ size_t bo(int l) const { return wo(l) + (size_t)E * E; }
  __host__ __device__ size_t g1(int l) const { return bo(l) + E; }
  __host__ __device__ size_t w1(int l) const { return g1(l) + 2 * (size_t)E; }
  __host__ __device__ size_t b1(int l) const { return w1(l) + (size_t)E * I; }
  __host__ __device__ size_t w2(int l) const { return b1(l) + I; }
  __host__ __device__ size_t b2(int l) const { return w2(l) + (size_t)I * E; }
  __host__ __device__ size_t g2(int l) const { return b2(l) + E; }
  __host__ __device__ size_t wp() const { return pool; }
  __host__ __device__ size_t bp() const { return pool + (size_t)E * E; }
  __host__ __device__ size_t ws_() const { return bp() + E; }
  __host__ __device__ size_t bs() const { return ws_() + E; }
  __host__ __device__ size_t sh_wqkv(int l) const { return (size_t)l * sh_layer; }
  __host__ __device__ size_t sh_wo(int l) const { return sh_wqkv(l) + (size_t)E * 3 * E; }
  __host__ __device__ size_t sh_w1(int l) const { return sh_wo(l) + (size_t)E * E; }
  __host__ __device__ size_t sh_w2(int l) const { return sh_w1(l) + (size_t)E * I; }
  __host__ __device__ size_t sh_wp() const { return (size_t)NL * sh_layer; }
  // dropout sites (site seeds as the DIN's: seed * 0x100000001B3 + site)
  int site_emb() const { return 1; }
  int site_attn(int l) const { return 2 + 3 * l; }
  int site_h1(int l) const { return 3 + 3 * l; }
  int site_h2(int l) const { return 4 + 3 * l; }
  int site_score() const { return 2 + 3 * NL; }
};

size_t al64(size_t x) { return (x + 63) / 64 * 64; }

__host__ __device__ inline unsigned long long site_seed(unsigned long long seed, int site) {
  return seed * 0x100000001B3ull + (unsigned long long)site;
}

// Every limit, with no CUDA call (num_sms() comes after, in make_bert_plan).
int check_bert_cfg(const tfr_bert_cfg* c) {
  TFR_REQUIRE(c != nullptr, "cfg must not be NULL");
  TFR_REQUIRE(c->vocab_size >= 1 && c->vocab_size < (1 << 30),
              "vocab_size %d must be in [1, 2^30)", c->vocab_size);
  TFR_REQUIRE(c->hidden_size >= 4 && c->hidden_size <= TFR_BERT_MAX_HIDDEN,
              "hidden_size %d must be in [4, %d]", c->hidden_size, TFR_BERT_MAX_HIDDEN);
  TFR_REQUIRE(c->num_heads >= 1 && c->hidden_size % c->num_heads == 0,
              "num_heads %d must divide hidden_size %d", c->num_heads, c->hidden_size);
  const int dh = c->hidden_size / c->num_heads;
  TFR_REQUIRE(dh % 4 == 0 && dh >= 4 && dh <= 128,
              "head size hidden_size / num_heads = %d must be a multiple of 4 in [4, 128]", dh);
  TFR_REQUIRE(c->intermediate_size >= 4 && c->intermediate_size % 4 == 0 &&
                  c->intermediate_size <= TFR_BERT_MAX_INTERMEDIATE,
              "intermediate_size %d must be a multiple of 4 in [4, %d]", c->intermediate_size,
              TFR_BERT_MAX_INTERMEDIATE);
  TFR_REQUIRE(c->num_layers >= 1 && c->num_layers <= TFR_BERT_MAX_LAYERS,
              "num_layers %d must be in [1, %d]", c->num_layers, TFR_BERT_MAX_LAYERS);
  TFR_REQUIRE(c->max_position >= 1 && c->max_position <= TFR_BERT_MAX_POSITION,
              "max_position %d must be in [1, %d]", c->max_position, TFR_BERT_MAX_POSITION);
  TFR_REQUIRE(c->type_vocab_size >= 1 && c->type_vocab_size <= TFR_BERT_MAX_TYPES,
              "type_vocab_size %d must be in [1, %d]", c->type_vocab_size, TFR_BERT_MAX_TYPES);
  TFR_REQUIRE(c->hidden_dropout >= 0.f && c->hidden_dropout < 1.f &&
                  c->attention_dropout >= 0.f && c->attention_dropout < 1.f &&
                  c->output_dropout >= 0.f && c->output_dropout < 1.f,
              "dropout rates must be in [0, 1)");
  TFR_REQUIRE(c->precision == TFR_PREC_FP32 || c->precision == TFR_PREC_TF32 ||
                  c->precision == TFR_PREC_BF16 || c->precision == TFR_PREC_FP16,
              "precision %d must be TFR_PREC_FP32 (%d), TFR_PREC_TF32 (%d), TFR_PREC_BF16 (%d) "
              "or TFR_PREC_FP16 (%d)",
              c->precision, TFR_PREC_FP32, TFR_PREC_TF32, TFR_PREC_BF16, TFR_PREC_FP16);
  // the 16-bit GEMM engine reads 16-byte rows: hidden, intermediate and head sizes in whole
  // 8-element chunks
  const bool h16 = c->precision == TFR_PREC_BF16 || c->precision == TFR_PREC_FP16;
  TFR_REQUIRE(!h16 || (c->hidden_size % 8 == 0 && c->intermediate_size % 8 == 0 && dh % 8 == 0),
              "%s needs hidden_size %d, intermediate_size %d and head size %d to be "
              "multiples of 8", c->precision == TFR_PREC_FP16 ? "TFR_PREC_FP16" : "TFR_PREC_BF16",
              c->hidden_size, c->intermediate_size, dh);
  return TFR_OK;
}

int check_bert_shape(const tfr_bert_cfg* c, int S, int L) {
  TFR_REQUIRE(S >= 0, "number of sequences %d must be >= 0", S);
  TFR_REQUIRE(L >= 1 && L <= c->max_position, "seq_length %d must be in [1, max_position %d]",
              L, c->max_position);
  const long long wide = c->intermediate_size > 3 * c->hidden_size ? c->intermediate_size
                                                                    : 3 * c->hidden_size;
  TFR_REQUIRE((long long)S * L * wide < (1ll << 31),
              "S * L * max(I, 3E) = %lld must be < 2^31", (long long)S * L * wide);
  return TFR_OK;
}

void param_layout(const tfr_bert_cfg* c, BertPlan* p) {
  p->V = c->vocab_size; p->E = c->hidden_size; p->H = c->num_heads; p->dh = p->E / p->H;
  p->I = c->intermediate_size; p->NL = c->num_layers; p->P = c->max_position;
  p->Tv = c->type_vocab_size;
  const size_t E = p->E, I = p->I;
  p->word = 0;
  p->pos = p->word + (size_t)p->V * E;
  p->type = p->pos + (size_t)p->P * E;
  p->emb_g = p->type + (size_t)p->Tv * E;
  p->layer0 = p->emb_g + 2 * E;
  p->layer_size = E * 3 * E + 3 * E + E * E + E + 2 * E + E * I + I + I * E + E + 2 * E;
  p->pool = p->layer0 + p->NL * p->layer_size;
  p->n_params = p->pool + E * E + E + E + 1;
}

// Row splits of M rows into about one range of whole 32-row blocks per SM.
void row_splits(size_t M, int target, int* rows_per, int* splits) {
  const int kb = (int)((M + 31) / 32);
  const int kb_per = kb > 0 ? (kb + target - 1) / target : 1;
  *rows_per = kb_per * 32;
  *splits = kb > 0 ? (kb + kb_per - 1) / kb_per : 1;
}

size_t h16_floats(size_t n) { return al64((n + 1) / 2); }   // floats that hold n 16-bit values

// Split count of a 16-bit dW GEMM (mn = 1: Kin x Nout output tiles of 128 x 128, `rows` of k in
// blocks of 64), from a cost model of the persistent grid: whole waves of tiles x splits work
// items over the SMs, each split's k blocks at about 0.5 us (a 128 x 128 x 64 bf16 block on
// one SM), plus writing and reading back one fp32 partial per split at about 3 TB/s.  Every
// split holds at least one k block.
int dw_splits(int sms, size_t Kin, size_t Nout, size_t rows) {
  const size_t tiles = ((Kin + 127) / 128) * ((Nout + 127) / 128);
  const int nkb = (int)((rows + 63) / 64);
  int best = 1;
  double best_t = 0.0;
  for (int s = 1; s <= 16 && s <= nkb; ++s) {
    const int per = (nkb + s - 1) / s;
    if ((nkb + per - 1) / per != s) continue;   // an empty split: the same as a smaller s
    const double waves = (double)((tiles * s + sms - 1) / sms);
    const double t = waves * per * 0.46e-6 + (double)s * Kin * Nout * 8.0 / 3e12;
    if (s == 1 || t < best_t) { best = s; best_t = t; }
  }
  return best;
}

size_t dw_stride(size_t Kin, size_t Nout) { return (Kin + 127) / 128 * 128 * Nout; }

// The 16-bit modes' workspace (the same for bf16 and fp16): 16-bit activations and backward
// signals, fp32 LayerNorm state, residual gradient and partials; offsets in floats.
void layout16(BertPlan* p) {
  const size_t M = (size_t)p->M, E = p->E, I = p->I, H = p->H, Sz = (size_t)p->S;
  size_t w = 0;
  for (int l = 0; l <= p->NL; ++l) { p->xs_off[l] = w; w += h16_floats(M * E); }
  p->xhe_off = w; w += al64(M * E);
  p->rse_off = w; w += al64(M);
  p->pos_ids_off = w; w += al64(M);
  for (int l = 0; l < p->NL; ++l) {
    p->qkv_off[l] = w; w += h16_floats(M * 3 * E);
    p->o_off[l] = w; w += h16_floats(M * E);
    p->lse_off[l] = w; w += al64(2 * M * H);
    p->xh1_off[l] = w; w += al64(M * E);
    p->rs1_off[l] = w; w += al64(M);
    p->x1_off[l] = w; w += h16_floats(M * E);
    p->u_off[l] = w; w += h16_floats(M * I);
    p->a_off[l] = w; w += h16_floats(M * I);
    p->xh2_off[l] = w; w += al64(M * E);
    p->rs2_off[l] = w; w += al64(M);
  }
  p->ytmp_off = w; w += h16_floats(M * E);
  p->pre_off = w; w += h16_floats(Sz * E);
  p->pooled_off = w; w += al64(Sz * E);
  p->g_off = w; w += al64(M * E);
  p->dres_off = w; w += al64(M * E);
  p->dy_off = w; w += al64(M * E);   // 16-bit in the layers, fp32 for the embedding tables
  p->tmp_off = w; w += h16_floats(M * E);
  p->do_off = w; w += h16_floats(M * E);
  p->dqkv_off = w; w += h16_floats(M * 3 * E);
  p->da_off = w; w += h16_floats(M * I);
  p->dsum_off = w; w += al64(M * H);
  p->dpre_off = w; w += h16_floats(Sz * E);
  p->dcls_off = w; w += h16_floats(Sz * E);
  const int nsplit = p->splits > p->s_splits ? p->splits : p->s_splits;
  // LayerNorm partials (2E per split) and the dW GEMMs' split partials share one region
  p->part_stride = al64(2 * E);
  size_t part = (size_t)nsplit * p->part_stride;
  const size_t shapes[5][3] = {{E, 3 * E, M}, {E, E, M}, {E, I, M}, {I, E, M}, {E, E, Sz}};
  for (auto& s : shapes) {
    const size_t v = (size_t)dw_splits(p->sms, s[0], s[1], s[2]) * dw_stride(s[0], s[1]);
    if (v > part) part = v;
  }
  p->part_off = w; w += al64(part);
  p->cs_stride = al64(I > 3 * E ? I : 3 * E);
  p->cs_off = w; w += (size_t)nsplit * p->cs_stride;
  p->emb_ws_off = w; w += p->emb_ws_floats;
  p->sh_layer = 4 * E * E + 2 * E * I;
  p->sh_total = (size_t)p->NL * p->sh_layer + E * E;
  p->wb_off = w; w += h16_floats(p->sh_total);
  p->wbt_off = w; w += h16_floats(p->sh_total);
  p->ws_floats = w;
}

int make_bert_plan(const tfr_bert_cfg* c, int S, int L, BertPlan* p) {
  int rc = check_bert_cfg(c);
  if (rc) return rc;
  rc = check_bert_shape(c, S, L);
  if (rc) return rc;
  std::memset(p, 0, sizeof(*p));
  param_layout(c, p);
  p->S = S; p->L = L; p->M = S * L;
  p->hdrop = c->training ? c->hidden_dropout : 0.f;
  p->adrop = c->training ? c->attention_dropout : 0.f;
  p->sdrop = c->training ? c->output_dropout : 0.f;
  p->seed = c->seed;
  p->tc = c->precision == TFR_PREC_TF32;
  p->h16 = c->precision == TFR_PREC_BF16 || c->precision == TFR_PREC_FP16;
  p->f16 = c->precision == TFR_PREC_FP16;
  p->passes = p->tc ? 1 : 3;
  if (p->h16) {
    p->sms = num_sms();
    row_splits((size_t)p->M, p->sms, &p->rows_per_split, &p->splits);
    row_splits((size_t)S, p->sms, &p->s_rows_per_split, &p->s_splits);
    size_t eb = 0;
    const int tables[3] = {p->V, p->P, p->Tv};
    for (int t : tables) {
      const size_t b = tfr_embedding_workspace_bytes(p->M > 0 ? p->M : 1, 1, t, p->E);
      if (b > eb) eb = b;
    }
    p->emb_ws_floats = al64((eb + 3) / 4 + 64);
    layout16(p);
    return TFR_OK;
  }
  const size_t M = (size_t)p->M, E = p->E, I = p->I, H = p->H, Sz = (size_t)S;
  size_t w = 0;
  for (int l = 0; l <= p->NL; ++l) { p->xs_off[l] = w; w += al64(M * E); }
  p->xhe_off = w; w += al64(M * E);
  p->rse_off = w; w += al64(M);
  p->pos_ids_off = w; w += al64(M);   // int32 position index of every token
  for (int l = 0; l < p->NL; ++l) {
    p->qkv_off[l] = w; w += al64(M * 3 * E);
    p->o_off[l] = w; w += al64(M * E);
    p->lse_off[l] = w; w += al64(2 * M * H);
    p->xh1_off[l] = w; w += al64(M * E);
    p->rs1_off[l] = w; w += al64(M);
    p->x1_off[l] = w; w += al64(M * E);
    p->u_off[l] = w; w += al64(M * I);
    p->a_off[l] = w; w += al64(M * I);
    p->xh2_off[l] = w; w += al64(M * E);
    p->rs2_off[l] = w; w += al64(M);
  }
  p->pre_off = w; w += al64(Sz * E);
  p->pooled_off = w; w += al64(Sz * E);
  p->g_off = w; w += al64(M * E);
  p->dres_off = w; w += al64(M * E);
  p->dy_off = w; w += al64(M * E);
  p->tmp_off = w; w += al64(M * E);
  p->do_off = w; w += al64(M * E);
  p->dqkv_off = w; w += al64(M * 3 * E);
  p->da_off = w; w += al64(M * I);
  p->dsum_off = w; w += al64(M * H);
  p->dpre_off = w; w += al64(Sz * E);
  const int target = num_sms();
  row_splits(M, target, &p->rows_per_split, &p->splits);
  row_splits(Sz, target, &p->s_rows_per_split, &p->s_splits);
  const int nsplit = p->splits > p->s_splits ? p->splits : p->s_splits;
  // dW partials: {Kin, Nout} of dWqkv, dWo / dWp, dW1, dW2; and the LayerNorm 2E partials
  size_t wmax = 2 * E;
  const size_t shapes[3][2] = {{E, 3 * E}, {E, I}, {I, E}};
  for (auto& s : shapes) {
    const size_t v = (s[0] + 127) / 128 * 128 * s[1];
    if (v > wmax) wmax = v;
  }
  p->part_stride = al64(wmax);
  p->part_off = w; w += (size_t)nsplit * p->part_stride;
  p->cs_stride = al64(I > 3 * E ? I : 3 * E);
  p->cs_off = w; w += (size_t)nsplit * p->cs_stride;
  size_t eb = 0;
  const int tables[3] = {p->V, p->P, p->Tv};
  for (int t : tables) {
    const size_t b = tfr_embedding_workspace_bytes(p->M > 0 ? p->M : 1, 1, t, p->E);
    if (b > eb) eb = b;
  }
  p->emb_ws_floats = al64((eb + 3) / 4 + 64);
  p->emb_ws_off = w; w += p->emb_ws_floats;
  p->ws_floats = w;
  return TFR_OK;
}

using bf16 = __nv_bfloat16;

// Element access of the kernels that run on fp32 or (16-bit modes) bf16 / fp16 rows: fp32 in
// registers, 16-bit stores rounded to nearest even (fp16: subnormals kept, magnitudes past
// 65504 stored as inf).
__device__ __forceinline__ float ldf(const float* p) { return *p; }
__device__ __forceinline__ float ldf(const bf16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ float ldf(const __half* p) { return __half2float(*p); }
__device__ __forceinline__ void stf(float* p, float v) { *p = v; }
__device__ __forceinline__ void stf(bf16* p, float v) { *p = __float2bfloat16_rn(v); }
__device__ __forceinline__ void stf(__half* p, float v) { *p = __float2half_rn(v); }
template <typename T>
__device__ __forceinline__ T rn16(float v) {
  if constexpr (std::is_same_v<T, __half>) return __float2half_rn(v);
  else return __float2bfloat16_rn(v);
}

// ---------------------------------------------------------------------------------------------
// LayerNorm over rows of width E <= 32 * NPL, one warp per row; column c = lane + 32 k.
// ---------------------------------------------------------------------------------------------
template <int NPL, typename T>
__device__ __forceinline__ void ln_row(float (&z)[NPL], int lane, int E, float* rs_out,
                                       float* xhat_row, T* out_row, const float* gamma,
                                       const float* beta, float odrop,
                                       unsigned long long oseed, size_t ebase) {
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < NPL; ++k)
    if (lane + 32 * k < E) sum += z[k];
  const float mean = warp_sum(sum) / E;
  float sq = 0.f;
#pragma unroll
  for (int k = 0; k < NPL; ++k)
    if (lane + 32 * k < E) sq += (z[k] - mean) * (z[k] - mean);
  const float rs = rsqrtf(warp_sum(sq) / E + kLnEps);
  const float kscale = odrop > 0.f ? 1.f / (1.f - odrop) : 1.f;
#pragma unroll
  for (int k = 0; k < NPL; ++k) {
    const int c = lane + 32 * k;
    if (c < E) {
      const float xh = (z[k] - mean) * rs;
      xhat_row[c] = xh;
      float v = xh * gamma[c] + beta[c];
      if (odrop > 0.f) v = din_uniform(oseed, ebase + c) >= odrop ? v * kscale : 0.f;
      stf(out_row + c, v);
    }
  }
  if (lane == 0) *rs_out = rs;
}

// x0[m] = dropout(LN_e(Word[w] + Pos[t] + Type[k])); ids outside [0, V) / [0, T_v) add no row
// and are counted into *bad_ids.  Also writes the position index t of every token.
template <int NPL, typename T = float>
__global__ void __launch_bounds__(kLnWarps * 32)
emb_ln_fwd_kernel(const int32_t* __restrict__ wid, const int32_t* __restrict__ tid, int M, int L,
                  const float* __restrict__ params, BertPlan p, float drop,
                  unsigned long long dseed, float* __restrict__ xhat, float* __restrict__ rstd,
                  T* __restrict__ out, int32_t* __restrict__ pos_ids, int* bad_ids) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kLnWarps + (threadIdx.x >> 5);
  if (row >= M) return;
  const int E = p.E;
  const int t = row % L;
  const int w = wid[row], k = tid[row];
  const bool wok = w >= 0 && w < p.V, kok = k >= 0 && k < p.Tv;
  if (lane == 0) {
    pos_ids[row] = t;
    if (bad_ids && (!wok || !kok)) atomicAdd(bad_ids, (int)!wok + (int)!kok);
  }
  const float* wr = params + p.word + (size_t)(wok ? w : 0) * E;
  const float* pr = params + p.pos + (size_t)t * E;
  const float* kr = params + p.type + (size_t)(kok ? k : 0) * E;
  float z[NPL];
#pragma unroll
  for (int j = 0; j < NPL; ++j) {
    const int c = lane + 32 * j;
    z[j] = 0.f;
    if (c < E) z[j] = (wok ? wr[c] : 0.f) + pr[c] + (kok ? kr[c] : 0.f);
  }
  const size_t e0 = (size_t)row * E;
  ln_row<NPL>(z, lane, E, rstd + row, xhat + e0, out + e0, params + p.emb_g,
              params + p.emb_g + E, drop, dseed, e0);
}

// out = LN(dropout(y) + xres) * gamma + beta; `y` may alias `xhat` (a row is read completely
// before it is written).  T: the element type of y, xres and out (xhat stays fp32).
template <int NPL, typename T = float>
__global__ void __launch_bounds__(kLnWarps * 32)
ln_fwd_kernel(const T* y, const T* __restrict__ xres, int M, int E,
              const float* __restrict__ gamma, const float* __restrict__ beta, float drop,
              unsigned long long dseed, float* xhat, float* __restrict__ rstd,
              T* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kLnWarps + (threadIdx.x >> 5);
  if (row >= M) return;
  const float kscale = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  const size_t e0 = (size_t)row * E;
  float z[NPL];
#pragma unroll
  for (int k = 0; k < NPL; ++k) {
    const int c = lane + 32 * k;
    z[k] = 0.f;
    if (c < E) {
      float v = ldf(y + e0 + c);
      if (drop > 0.f) v = din_uniform(dseed, e0 + c) >= drop ? v * kscale : 0.f;
      z[k] = v + ldf(xres + e0 + c);
    }
  }
  ln_row<NPL>(z, lane, E, rstd + row, xhat + e0, out + e0, gamma, beta, 0.f, 0, 0);
}

// LayerNorm backward over rows [blockIdx.x * rows_per, ...), one warp per row:
//   g'   = gdrop'(g)   (the dropout that followed the LayerNorm: the embedding's)
//   dz   = rstd (g' gamma - mean(g' gamma) - xhat mean(g' gamma xhat))   -> dres (may be NULL)
//   dy   = ydrop'(dz)  (the dropout on the branch that was added before it)
// and this CTA's partial sums dgamma = sum g' xhat, dbeta = sum g' into partial[blockIdx.x],
// in fixed order: warps own rows round-robin, then the warps' sums are added in warp order.
// T: the element type of dy (dres stays fp32).
template <int NPL, typename T = float>
__global__ void __launch_bounds__(kLnWarps * 32)
ln_bwd_kernel(const float* __restrict__ g, const float* __restrict__ xhat,
              const float* __restrict__ rstd, const float* __restrict__ gamma, int M, int E,
              int rows_per, float gdrop, unsigned long long gseed, float ydrop,
              unsigned long long yseed, float* __restrict__ dres, T* __restrict__ dy,
              float* __restrict__ partial, size_t pstride) {
  __shared__ float red[kLnWarps][TFR_BERT_MAX_HIDDEN];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int beg = blockIdx.x * rows_per, end = min(M, beg + rows_per);
  const float gscale = gdrop > 0.f ? 1.f / (1.f - gdrop) : 1.f;
  const float yscale = ydrop > 0.f ? 1.f / (1.f - ydrop) : 1.f;
  float ag[NPL], ab[NPL];
#pragma unroll
  for (int k = 0; k < NPL; ++k) ag[k] = ab[k] = 0.f;
  for (int row = beg + warp; row < end; row += kLnWarps) {
    const size_t e0 = (size_t)row * E;
    float gv[NPL], xv[NPL];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < NPL; ++k) {
      const int c = lane + 32 * k;
      gv[k] = xv[k] = 0.f;
      if (c < E) {
        float v = g[e0 + c];
        if (gdrop > 0.f) v = din_uniform(gseed, e0 + c) >= gdrop ? v * gscale : 0.f;
        gv[k] = v;
        xv[k] = xhat[e0 + c];
        const float dx = v * gamma[c];
        s1 += dx;
        s2 += dx * xv[k];
      }
    }
    s1 = warp_sum(s1) / E;
    s2 = warp_sum(s2) / E;
    const float rs = rstd[row];
#pragma unroll
    for (int k = 0; k < NPL; ++k) {
      const int c = lane + 32 * k;
      if (c < E) {
        const float dz = rs * (gv[k] * gamma[c] - s1 - xv[k] * s2);
        if (dres) dres[e0 + c] = dz;
        stf(dy + e0 + c,
            ydrop > 0.f ? (din_uniform(yseed, e0 + c) >= ydrop ? dz * yscale : 0.f) : dz);
        ag[k] += gv[k] * xv[k];
        ab[k] += gv[k];
      }
    }
  }
  // two rounds through shared memory (dgamma, then dbeta): 8 x 1024 floats each
  for (int round = 0; round < 2; ++round) {
#pragma unroll
    for (int k = 0; k < NPL; ++k) {
      const int c = lane + 32 * k;
      if (c < E) red[warp][c] = round == 0 ? ag[k] : ab[k];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < E; c += blockDim.x) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < kLnWarps; ++w) s += red[w][c];
      partial[(size_t)blockIdx.x * pstride + round * E + c] = s;
    }
    __syncthreads();
  }
}

__device__ __forceinline__ float gelu_tanh(float u) {
  const float k0 = 0.7978845608028654f;   // sqrt(2 / pi)
  return 0.5f * u * (1.f + tanhf(k0 * (u + 0.044715f * u * u * u)));
}

template <typename T>
__global__ void __launch_bounds__(256)
gelu_fwd_kernel(const T* __restrict__ u, size_t n, T* __restrict__ a) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) stf(a + i, gelu_tanh(ldf(u + i)));
}

// da *= gelu'(u), in place.
template <typename T>
__global__ void __launch_bounds__(256)
gelu_bwd_kernel(const T* __restrict__ u, size_t n, T* __restrict__ da) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float k0 = 0.7978845608028654f, x = ldf(u + i);
  const float t = tanhf(k0 * (x + 0.044715f * x * x * x));
  stf(da + i, ldf(da + i) * (0.5f * (1.f + t) + 0.5f * x * (1.f - t * t) * k0 *
                                                    (1.f + 3.f * 0.044715f * x * x)));
}

// dst = a + b, elementwise
template <typename T>
__global__ void __launch_bounds__(256)
add_kernel(const T* __restrict__ a, const float* __restrict__ b, size_t n,
           float* __restrict__ dst) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = ldf(a + i) + b[i];
}

// Score head, one warp per sequence: pooled = tanh(pre), score = dropout(pooled) . w_s + b_s.
template <typename T>
__global__ void __launch_bounds__(256)
head_fwd_kernel(const T* __restrict__ pre, int S, int E, const float* __restrict__ w,
                const float* __restrict__ b, float drop, unsigned long long dseed,
                float* __restrict__ pooled, float* __restrict__ scores) {
  const int lane = threadIdx.x & 31;
  const int s = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (s >= S) return;
  const float kscale = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  float acc = 0.f;
  for (int c = lane; c < E; c += 32) {
    const size_t e = (size_t)s * E + c;
    const float t = tanhf(ldf(pre + e));
    pooled[e] = t;
    float v = t;
    if (drop > 0.f) v = din_uniform(dseed, e) >= drop ? t * kscale : 0.f;
    acc += v * w[c];
  }
  acc = warp_sum(acc);
  if (lane == 0) scores[s] = acc + b[0];
}

// dpre[s, c] = ds_s w_s[c] keep (1 - pooled^2);  dw_s[c] = sum_s ds_s dropout(pooled)[s, c],
// db_s = sum_s ds_s, both summed over s in order (one thread per column; thread E: db_s).
template <typename T>
__global__ void __launch_bounds__(256)
head_bwd_kernel(const float* __restrict__ pooled, const float* __restrict__ dscores, int S, int E,
                const float* __restrict__ w, float drop, unsigned long long dseed,
                T* __restrict__ dpre, float* __restrict__ dw, float* __restrict__ db) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c > E) return;
  const float kscale = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  float acc = 0.f;
  if (c == E) {
    for (int s = 0; s < S; ++s) acc += dscores[s];
    db[0] = acc;
    return;
  }
  const float wc = w[c];
  for (int s = 0; s < S; ++s) {
    const size_t e = (size_t)s * E + c;
    const float t = pooled[e];
    const float keep = drop > 0.f ? (din_uniform(dseed, e) >= drop ? kscale : 0.f) : 1.f;
    const float ds = dscores[s];
    acc += ds * t * keep;
    stf(dpre + e, ds * wc * keep * (1.f - t * t));
  }
  dw[c] = acc;
}

unsigned blocks_for(size_t n, int per) { return (unsigned)((n + per - 1) / per); }

#define TFR_BERT_LN_DISPATCH(E, kernel, grid, ...)                                     \
  ((E) <= 128   ? (kernel<4><<<grid, kLnWarps * 32, 0, st>>>(__VA_ARGS__), 0)          \
   : (E) <= 256 ? (kernel<8><<<grid, kLnWarps * 32, 0, st>>>(__VA_ARGS__), 0)          \
   : (E) <= 512 ? (kernel<16><<<grid, kLnWarps * 32, 0, st>>>(__VA_ARGS__), 0)         \
                : (kernel<32><<<grid, kLnWarps * 32, 0, st>>>(__VA_ARGS__), 0))

int attn_fwd(const BertPlan& p, const float* qkv, const uint8_t* mask, unsigned long long s,
             float* O, float* lse, cudaStream_t st) {
  return p.tc ? din_tc_attn_fwd(qkv, mask, p.S, p.L, p.H, p.dh, p.adrop, s, O, lse, st)
              : din_attn_fwd(qkv, mask, p.S, p.L, p.H, p.dh, p.adrop, s, O, lse, st);
}

int attn_bwd(const BertPlan& p, const float* qkv, const uint8_t* mask, unsigned long long s,
             const float* O, const float* lse, const float* dO, float* dsum, float* dqkv,
             cudaStream_t st) {
  return p.tc ? din_tc_attn_bwd(qkv, mask, p.S, p.L, p.H, p.dh, p.adrop, s, O, lse, dO, dsum,
                                dqkv, st)
              : din_attn_bwd(qkv, mask, p.S, p.L, p.H, p.dh, p.adrop, s, O, lse, dO, dsum, dqkv,
                             st);
}

// dW of a [Kin, Nout] kernel + its bias over M rows of A (lda) and dZ (pitch Nout).
int dense_grad(const BertPlan& p, float* ws, const float* A, int lda, int Kin, const float* dZ,
               int Nout, int M, bool seq_rows, float* grads_w, cudaStream_t st) {
  const int rows_per = seq_rows ? p.s_rows_per_split : p.rows_per_split;
  const int splits = seq_rows ? p.s_splits : p.splits;
  float* cs = ws + p.cs_off;
  int rc = mlp_colsum(dZ, M, Nout, rows_per, splits, cs, p.cs_stride, 0, st);
  if (rc) return rc;
  return din_weight_grad(A, lda, Kin, dZ, Nout, Nout, M, splits, ws + p.part_off, p.part_stride,
                         cs, p.cs_stride, grads_w, p.passes, st);
}

int ln_bwd(const BertPlan& p, float* ws, const float* g, size_t xh_off, size_t rs_off,
           const float* gamma, float gdrop, unsigned long long gseed, float ydrop,
           unsigned long long yseed, float* dres, float* dy, float* dgamma, cudaStream_t st) {
  TFR_BERT_LN_DISPATCH(p.E, ln_bwd_kernel, p.splits, g, ws + xh_off, ws + rs_off, gamma, p.M, p.E,
                       p.rows_per_split, gdrop, gseed, ydrop, yseed, dres, dy, ws + p.part_off,
                       p.part_stride);
  TFR_LAUNCH_OK();
  return mlp_reduce_partials(ws + p.part_off, p.splits, p.part_stride, 2 * (size_t)p.E, dgamma,
                             st);
}

int bert_fwd(const int32_t* wid, const uint8_t* mask, const int32_t* tid, const BertPlan& p,
             const float* params, float* ws, float* scores, int* bad_ids, cudaStream_t st) {
  const int E = p.E, I = p.I, M = p.M;
  const size_t MI = (size_t)M * I;
  const unsigned ln_grid = blocks_for(M, kLnWarps);
  TFR_BERT_LN_DISPATCH(E, emb_ln_fwd_kernel, ln_grid, wid, tid, M, p.L, params, p,
                       p.hdrop, site_seed(p.seed, p.site_emb()), ws + p.xhe_off, ws + p.rse_off,
                       ws + p.xs_off[0], reinterpret_cast<int32_t*>(ws + p.pos_ids_off), bad_ids);
  TFR_LAUNCH_OK();
  int rc;
  for (int l = 0; l < p.NL; ++l) {
    const float* x = ws + p.xs_off[l];
    float* qkv = ws + p.qkv_off[l];
    rc = din_gemm(x, E, 0, params + p.wqkv(l), 3 * E, 1, qkv, 3 * E, M, 3 * E, E,
                  params + p.bqkv(l), TFR_ACT_NONE, p.passes, st);
    if (rc) return rc;
    rc = attn_fwd(p, qkv, mask, site_seed(p.seed, p.site_attn(l)), ws + p.o_off[l],
                  ws + p.lse_off[l], st);
    if (rc) return rc;
    float* y1 = ws + p.xh1_off[l];
    rc = din_gemm(ws + p.o_off[l], E, 0, params + p.wo(l), E, 1, y1, E, M, E, E,
                  params + p.bo(l), TFR_ACT_NONE, p.passes, st);
    if (rc) return rc;
    TFR_BERT_LN_DISPATCH(E, ln_fwd_kernel, ln_grid, y1, x, M, E, params + p.g1(l),
                         params + p.g1(l) + E, p.hdrop, site_seed(p.seed, p.site_h1(l)), y1,
                         ws + p.rs1_off[l], ws + p.x1_off[l]);
    TFR_LAUNCH_OK();
    rc = din_gemm(ws + p.x1_off[l], E, 0, params + p.w1(l), I, 1, ws + p.u_off[l], I, M, I, E,
                  params + p.b1(l), TFR_ACT_NONE, p.passes, st);
    if (rc) return rc;
    gelu_fwd_kernel<<<blocks_for(MI, 256), 256, 0, st>>>(ws + p.u_off[l], MI, ws + p.a_off[l]);
    TFR_LAUNCH_OK();
    float* y2 = ws + p.xh2_off[l];
    rc = din_gemm(ws + p.a_off[l], I, 0, params + p.w2(l), E, 1, y2, E, M, E, I,
                  params + p.b2(l), TFR_ACT_NONE, p.passes, st);
    if (rc) return rc;
    TFR_BERT_LN_DISPATCH(E, ln_fwd_kernel, ln_grid, y2, ws + p.x1_off[l], M, E, params + p.g2(l),
                         params + p.g2(l) + E, p.hdrop, site_seed(p.seed, p.site_h2(l)), y2,
                         ws + p.rs2_off[l], ws + p.xs_off[l + 1]);
    TFR_LAUNCH_OK();
  }
  // pooler on the [CLS] rows (row 0 of every sequence: lda = L E), then the score head
  rc = din_gemm(ws + p.xs_off[p.NL], p.L * E, 0, params + p.wp(), E, 1, ws + p.pre_off, E, p.S,
                E, E, params + p.bp(), TFR_ACT_NONE, p.passes, st);
  if (rc) return rc;
  head_fwd_kernel<<<blocks_for(p.S, 8), 256, 0, st>>>(
      ws + p.pre_off, p.S, E, params + p.ws_(), params + p.bs(), p.sdrop,
      site_seed(p.seed, p.site_score()), ws + p.pooled_off, scores);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

int bert_bwd(const int32_t* wid, const uint8_t* mask, const int32_t* tid, const BertPlan& p,
             const float* params, const float* dscores, float* ws, float* grads,
             cudaStream_t st) {
  const int E = p.E, I = p.I, M = p.M, S = p.S;
  const size_t ME = (size_t)M * E, MI = (size_t)M * I;
  float* g = ws + p.g_off;       // d loss / d (current layer's output)
  float* dres = ws + p.dres_off;
  float* dy = ws + p.dy_off;
  float* tmp = ws + p.tmp_off;
  float* dO = ws + p.do_off;
  float* dqkv = ws + p.dqkv_off;
  float* da = ws + p.da_off;
  float* dpre = ws + p.dpre_off;
  // score head and pooler
  head_bwd_kernel<<<blocks_for(E + 1, 256), 256, 0, st>>>(
      ws + p.pooled_off, dscores, S, E, params + p.ws_(), p.sdrop,
      site_seed(p.seed, p.site_score()), dpre, grads + p.ws_(), grads + p.bs());
  TFR_LAUNCH_OK();
  const float* xl = ws + p.xs_off[p.NL];
  int rc = dense_grad(p, ws, xl, p.L * E, E, dpre, E, S, true, grads + p.wp(), st);
  if (rc) return rc;
  TFR_CUDA_OK(cudaMemsetAsync(g, 0, ME * sizeof(float), st));
  rc = din_gemm(dpre, E, 0, params + p.wp(), E, 0, g, p.L * E, S, E, E, nullptr, TFR_ACT_NONE,
                p.passes, st);
  if (rc) return rc;
  for (int l = p.NL - 1; l >= 0; --l) {
    // x'' = LN_2(drop(a W2 + b2) + x'):  dres = d x' (residual), dy = d(a W2 + b2)
    rc = ln_bwd(p, ws, g, p.xh2_off[l], p.rs2_off[l], params + p.g2(l), 0.f, 0, p.hdrop,
                site_seed(p.seed, p.site_h2(l)), dres, dy, grads + p.g2(l), st);
    if (rc) return rc;
    rc = dense_grad(p, ws, ws + p.a_off[l], I, I, dy, E, M, false, grads + p.w2(l), st);
    if (rc) return rc;
    rc = din_gemm(dy, E, 0, params + p.w2(l), E, 0, da, I, M, I, E, nullptr, TFR_ACT_NONE,
                  p.passes, st);
    if (rc) return rc;
    gelu_bwd_kernel<<<blocks_for(MI, 256), 256, 0, st>>>(ws + p.u_off[l], MI, da);
    TFR_LAUNCH_OK();
    rc = dense_grad(p, ws, ws + p.x1_off[l], E, E, da, I, M, false, grads + p.w1(l), st);
    if (rc) return rc;
    rc = din_gemm(da, I, 0, params + p.w1(l), I, 0, tmp, E, M, E, I, nullptr, TFR_ACT_NONE,
                  p.passes, st);
    if (rc) return rc;
    add_kernel<<<blocks_for(ME, 256), 256, 0, st>>>(tmp, dres, ME, g);   // d x'
    TFR_LAUNCH_OK();
    // x' = LN_1(drop(o Wo + bo) + x)
    rc = ln_bwd(p, ws, g, p.xh1_off[l], p.rs1_off[l], params + p.g1(l), 0.f, 0, p.hdrop,
                site_seed(p.seed, p.site_h1(l)), dres, dy, grads + p.g1(l), st);
    if (rc) return rc;
    rc = dense_grad(p, ws, ws + p.o_off[l], E, E, dy, E, M, false, grads + p.wo(l), st);
    if (rc) return rc;
    rc = din_gemm(dy, E, 0, params + p.wo(l), E, 0, dO, E, M, E, E, nullptr, TFR_ACT_NONE,
                  p.passes, st);
    if (rc) return rc;
    rc = attn_bwd(p, ws + p.qkv_off[l], mask, site_seed(p.seed, p.site_attn(l)), ws + p.o_off[l],
                  ws + p.lse_off[l], dO, ws + p.dsum_off, dqkv, st);
    if (rc) return rc;
    const float* x = ws + p.xs_off[l];
    rc = dense_grad(p, ws, x, E, E, dqkv, 3 * E, M, false, grads + p.wqkv(l), st);
    if (rc) return rc;
    rc = din_gemm(dqkv, 3 * E, 0, params + p.wqkv(l), 3 * E, 0, tmp, E, M, E, 3 * E, nullptr,
                  TFR_ACT_NONE, p.passes, st);
    if (rc) return rc;
    add_kernel<<<blocks_for(ME, 256), 256, 0, st>>>(tmp, dres, ME, g);   // d x
    TFR_LAUNCH_OK();
  }
  // embeddings: x0 = dropout(LN_e(sum)) -> d sum, then one segment sum per table
  rc = ln_bwd(p, ws, g, p.xhe_off, p.rse_off, params + p.emb_g, p.hdrop,
              site_seed(p.seed, p.site_emb()), 0.f, 0, nullptr, dy, grads + p.emb_g, st);
  if (rc) return rc;
  void* ews = ws + p.emb_ws_off;
  rc = tfr_embedding_bwd(wid, M, 1, dy, E, 1, p.V, E, TFR_COMBINER_SUM, 0, ews,
                         grads + p.word, nullptr, st);
  if (rc) return rc;
  rc = tfr_embedding_bwd(reinterpret_cast<const int32_t*>(ws + p.pos_ids_off), M, 1, dy, E, 1,
                         p.P, E, TFR_COMBINER_SUM, 0, ews, grads + p.pos, nullptr, st);
  if (rc) return rc;
  return tfr_embedding_bwd(tid, M, 1, dy, E, 1, p.Tv, E, TFR_COMBINER_SUM, 0, ews,
                           grads + p.type, nullptr, st);
}

// ---------------------------------------------------------------------------------------------
// 16-bit modes (TFR_PREC_BF16, TFR_PREC_FP16), one code path templated on the element type T
// (bf16 or fp16).  Activations, GEMM operands and backward signals are T in the workspace; every
// projection runs on the 16-bit wgmma engine (tc_gemm_bf16.cu), the attention core on
// din_bf16.cu.  Parameters, gradients, LayerNorm state, the residual gradient g / dres
// and every partial sum stay fp32:
//   forward   out = T(A W + b)       A K-major, W^T [out, in] shadow K-major (mn = 0)
//   backward  dW  = A^T dZ           both as stored, MN-major (mn = 1), fp32 split partials
//                                    reduced in fixed order
//             db  = colsum(dZ)       fp32 column sums of the 16-bit dZ, per row range
//             dA  = T(dZ W^T)        dZ K-major, W [in, out] shadow K-major (mn = 0)
// ---------------------------------------------------------------------------------------------

// wb = T(W) [in, out] and wbt = T(W)^T [out, in] of every projection kernel: blockIdx.y
// picks the matrix (Wqkv, Wo, W1, W2 of each layer, then Wp), 32 x 32 tiles through shared
// memory so both stores are coalesced.
template <typename T>
__global__ void __launch_bounds__(256)
shadow_kernel(const float* __restrict__ params, BertPlan p, T* __restrict__ wb,
              T* __restrict__ wbt) {
  __shared__ float tile[32][33];
  const int e = blockIdx.y, l = e / 4;
  size_t src, dst;
  int kin = p.E, nout = p.E;
  if (e == 4 * p.NL) {
    src = p.wp(); dst = p.sh_wp();
  } else if (e % 4 == 0) {
    src = p.wqkv(l); dst = p.sh_wqkv(l); nout = 3 * p.E;
  } else if (e % 4 == 1) {
    src = p.wo(l); dst = p.sh_wo(l);
  } else if (e % 4 == 2) {
    src = p.w1(l); dst = p.sh_w1(l); nout = p.I;
  } else {
    src = p.w2(l); dst = p.sh_w2(l); kin = p.I;
  }
  const int tn = (nout + 31) / 32, ntiles = ((kin + 31) / 32) * tn;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int ti = blockIdx.x; ti < ntiles; ti += gridDim.x) {
    const int k0 = (ti / tn) * 32, n0 = (ti % tn) * 32;
    for (int r = ty; r < 32; r += 8) {
      const int k = k0 + r, n = n0 + tx;
      if (k < kin && n < nout) {
        const float v = params[src + (size_t)k * nout + n];
        wb[dst + (size_t)k * nout + n] = rn16<T>(v);
        tile[r][tx] = v;
      }
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
      const int n = n0 + r, k = k0 + tx;
      if (n < nout && k < kin) wbt[dst + (size_t)n * kin + k] = rn16<T>(tile[tx][r]);
    }
    __syncthreads();
  }
}

// mlp_colsum over 16-bit dZ: partial[z][n] = sum of rows [z rows_per, ...) of column n, in row
// order.
template <typename T>
__global__ void __launch_bounds__(256)
colsum16_kernel(const T* __restrict__ dZ, int M, int N, int rows_per,
                   float* __restrict__ partial, size_t pstride) {
  const int z = blockIdx.x;
  const int mbeg = z * rows_per, mend = min(M, mbeg + rows_per);
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    float acc = 0.f;
    for (int m = mbeg; m < mend; ++m) acc += ldf(dZ + (size_t)m * N + n);
    partial[(size_t)z * pstride + n] = acc;
  }
}

// g[s L E + c] = dcls[s E + c]: the [CLS] rows' gradient into the (zeroed) residual gradient.
template <typename T>
__global__ void __launch_bounds__(256)
cls_scatter_kernel(const T* __restrict__ dcls, int S, int E, int L, float* __restrict__ g) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)S * E) return;
  const size_t s = i / E, c = i % E;
  g[s * L * E + c] = ldf(dcls + i);
}

#define TFR_BERT_LN_DISPATCH16(E, kernel, grid, ...)                                      \
  ((E) <= 128   ? (kernel<4, T><<<grid, kLnWarps * 32, 0, st>>>(__VA_ARGS__), 0)         \
   : (E) <= 256 ? (kernel<8, T><<<grid, kLnWarps * 32, 0, st>>>(__VA_ARGS__), 0)         \
   : (E) <= 512 ? (kernel<16, T><<<grid, kLnWarps * 32, 0, st>>>(__VA_ARGS__), 0)        \
                : (kernel<32, T><<<grid, kLnWarps * 32, 0, st>>>(__VA_ARGS__), 0))

template <typename T>
T* h16(float* ws, size_t off) { return reinterpret_cast<T*>(ws + off); }

// C [GM, GN] (ldc) = T(A B^T (+ bias)): A [GM, GK] (lda), B [GN, GK] (ldb), both K-major.
template <typename T>
int bgemm(const T* A, int lda, const T* B, int ldb, T* C, int ldc, int GM, int GN,
          int GK, const float* bias, cudaStream_t st) {
  tcb::GemmDesc g{};
  g.f16 = std::is_same_v<T, __half>;
  g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.C = C; g.ldc = ldc;
  g.GM = GM; g.GN = GN; g.GK = GK;
  g.mn = 0;
  g.epi = bias ? tcb::EPI_BIAS_ACT : tcb::EPI_STORE;
  g.bias = bias; g.act = TFR_ACT_NONE;
  g.splits = 1;
  return tcb::gemm(g, st);
}

// grads_w[0 .. Kin Nout + Nout) = {A^T dZ, column sums of dZ} over M rows of A [M, Kin] (lda)
// and dZ [M, Nout].
template <typename T>
int dense_grad16(const BertPlan& p, float* ws, const T* A, int lda, int Kin,
                    const T* dZ, int Nout, int M, bool seq_rows, float* grads_w,
                    cudaStream_t st) {
  const int rows_per = seq_rows ? p.s_rows_per_split : p.rows_per_split;
  const int splits = seq_rows ? p.s_splits : p.splits;
  float* cs = ws + p.cs_off;
  colsum16_kernel<<<splits, 256, 0, st>>>(dZ, M, Nout, rows_per, cs, p.cs_stride);
  TFR_LAUNCH_OK();
  int rc = mlp_reduce_partials(cs, splits, p.cs_stride, (size_t)Nout,
                               grads_w + (size_t)Kin * Nout, st);
  if (rc) return rc;
  const int ksplits = dw_splits(p.sms, Kin, Nout, M);
  const size_t stride = dw_stride(Kin, Nout);
  tcb::GemmDesc g{};
  g.A = A; g.lda = lda; g.B = dZ; g.ldb = Nout;
  g.C = ws + p.part_off; g.ldc = Nout;
  g.GM = Kin; g.GN = Nout; g.GK = M;
  g.mn = 1; g.epi = tcb::EPI_STORE;
  g.splits = ksplits; g.split_stride = stride;
  g.f16 = std::is_same_v<T, __half>;
  rc = tcb::gemm(g, st);
  if (rc) return rc;
  return mlp_reduce_partials(ws + p.part_off, ksplits, stride, (size_t)Kin * Nout, grads_w, st);
}

template <typename T>
int ln_bwd16(const BertPlan& p, float* ws, const float* g, size_t xh_off, size_t rs_off,
                const float* gamma, float ydrop, unsigned long long yseed, float* dres, T* dy,
                float* dgamma, cudaStream_t st) {
  TFR_BERT_LN_DISPATCH16(p.E, ln_bwd_kernel, p.splits, g, ws + xh_off, ws + rs_off, gamma,
                            p.M, p.E, p.rows_per_split, 0.f, 0ull, ydrop, yseed, dres, dy,
                            ws + p.part_off, p.part_stride);
  TFR_LAUNCH_OK();
  return mlp_reduce_partials(ws + p.part_off, p.splits, p.part_stride, 2 * (size_t)p.E, dgamma,
                             st);
}

template <typename T>
int bert_fwd16(const int32_t* wid, const uint8_t* mask, const int32_t* tid, const BertPlan& p,
                  const float* params, float* ws, float* scores, int* bad_ids, cudaStream_t st) {
  const int E = p.E, I = p.I, M = p.M;
  const size_t MI = (size_t)M * I;
  T* wbt = h16<T>(ws, p.wbt_off);
  shadow_kernel<T><<<dim3(64, 4 * p.NL + 1), 256, 0, st>>>(params, p, h16<T>(ws, p.wb_off), wbt);
  TFR_LAUNCH_OK();
  const unsigned ln_grid = blocks_for(M, kLnWarps);
  TFR_BERT_LN_DISPATCH16(E, emb_ln_fwd_kernel, ln_grid, wid, tid, M, p.L, params, p, p.hdrop,
                            site_seed(p.seed, p.site_emb()), ws + p.xhe_off, ws + p.rse_off,
                            h16<T>(ws, p.xs_off[0]), reinterpret_cast<int32_t*>(ws + p.pos_ids_off),
                            bad_ids);
  TFR_LAUNCH_OK();
  T* y = h16<T>(ws, p.ytmp_off);
  int rc;
  for (int l = 0; l < p.NL; ++l) {
    const T* x = h16<T>(ws, p.xs_off[l]);
    T* qkv = h16<T>(ws, p.qkv_off[l]);
    T* o = h16<T>(ws, p.o_off[l]);
    T* x1 = h16<T>(ws, p.x1_off[l]);
    T* u = h16<T>(ws, p.u_off[l]);
    T* a = h16<T>(ws, p.a_off[l]);
    rc = bgemm(x, E, wbt + p.sh_wqkv(l), E, qkv, 3 * E, M, 3 * E, E, params + p.bqkv(l), st);
    if (rc) return rc;
    rc = din16_attn_fwd(qkv, mask, p.S, p.L, p.H, p.dh, p.adrop,
                           site_seed(p.seed, p.site_attn(l)), o, ws + p.lse_off[l], st);
    if (rc) return rc;
    rc = bgemm(o, E, wbt + p.sh_wo(l), E, y, E, M, E, E, params + p.bo(l), st);
    if (rc) return rc;
    TFR_BERT_LN_DISPATCH16(E, ln_fwd_kernel, ln_grid, y, x, M, E, params + p.g1(l),
                              params + p.g1(l) + E, p.hdrop, site_seed(p.seed, p.site_h1(l)),
                              ws + p.xh1_off[l], ws + p.rs1_off[l], x1);
    TFR_LAUNCH_OK();
    rc = bgemm(x1, E, wbt + p.sh_w1(l), E, u, I, M, I, E, params + p.b1(l), st);
    if (rc) return rc;
    gelu_fwd_kernel<<<blocks_for(MI, 256), 256, 0, st>>>(u, MI, a);
    TFR_LAUNCH_OK();
    rc = bgemm(a, I, wbt + p.sh_w2(l), I, y, E, M, E, I, params + p.b2(l), st);
    if (rc) return rc;
    TFR_BERT_LN_DISPATCH16(E, ln_fwd_kernel, ln_grid, y, x1, M, E, params + p.g2(l),
                              params + p.g2(l) + E, p.hdrop, site_seed(p.seed, p.site_h2(l)),
                              ws + p.xh2_off[l], ws + p.rs2_off[l], h16<T>(ws, p.xs_off[l + 1]));
    TFR_LAUNCH_OK();
  }
  T* pre = h16<T>(ws, p.pre_off);
  rc = bgemm(h16<T>(ws, p.xs_off[p.NL]), p.L * E, wbt + p.sh_wp(), E, pre, E, p.S, E, E,
             params + p.bp(), st);
  if (rc) return rc;
  head_fwd_kernel<<<blocks_for(p.S, 8), 256, 0, st>>>(
      pre, p.S, E, params + p.ws_(), params + p.bs(), p.sdrop, site_seed(p.seed, p.site_score()),
      ws + p.pooled_off, scores);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

template <typename T>
int bert_bwd16(const int32_t* wid, const uint8_t* mask, const int32_t* tid, const BertPlan& p,
                  const float* params, const float* dscores, float* ws, float* grads,
                  cudaStream_t st) {
  const int E = p.E, I = p.I, M = p.M, S = p.S;
  const size_t ME = (size_t)M * E, MI = (size_t)M * I;
  float* g = ws + p.g_off;       // d loss / d (current layer's output), fp32
  float* dres = ws + p.dres_off;
  T* dy = h16<T>(ws, p.dy_off);
  T* tmp = h16<T>(ws, p.tmp_off);
  T* dO = h16<T>(ws, p.do_off);
  T* dqkv = h16<T>(ws, p.dqkv_off);
  T* da = h16<T>(ws, p.da_off);
  T* dpre = h16<T>(ws, p.dpre_off);
  const T* wb = h16<T>(ws, p.wb_off);
  head_bwd_kernel<<<blocks_for(E + 1, 256), 256, 0, st>>>(
      ws + p.pooled_off, dscores, S, E, params + p.ws_(), p.sdrop,
      site_seed(p.seed, p.site_score()), dpre, grads + p.ws_(), grads + p.bs());
  TFR_LAUNCH_OK();
  const T* xl = h16<T>(ws, p.xs_off[p.NL]);
  int rc = dense_grad16(p, ws, xl, p.L * E, E, dpre, E, S, true, grads + p.wp(), st);
  if (rc) return rc;
  T* dcls = h16<T>(ws, p.dcls_off);
  rc = bgemm(dpre, E, wb + p.sh_wp(), E, dcls, E, S, E, E, nullptr, st);
  if (rc) return rc;
  TFR_CUDA_OK(cudaMemsetAsync(g, 0, ME * sizeof(float), st));
  cls_scatter_kernel<<<blocks_for((size_t)S * E, 256), 256, 0, st>>>(dcls, S, E, p.L, g);
  TFR_LAUNCH_OK();
  for (int l = p.NL - 1; l >= 0; --l) {
    // x'' = LN_2(drop(a W2 + b2) + x'):  dres = d x' (residual), dy = d(a W2 + b2)
    rc = ln_bwd16(p, ws, g, p.xh2_off[l], p.rs2_off[l], params + p.g2(l), p.hdrop,
                     site_seed(p.seed, p.site_h2(l)), dres, dy, grads + p.g2(l), st);
    if (rc) return rc;
    rc = dense_grad16(p, ws, h16<T>(ws, p.a_off[l]), I, I, dy, E, M, false, grads + p.w2(l), st);
    if (rc) return rc;
    rc = bgemm(dy, E, wb + p.sh_w2(l), E, da, I, M, I, E, nullptr, st);
    if (rc) return rc;
    gelu_bwd_kernel<<<blocks_for(MI, 256), 256, 0, st>>>(h16<T>(ws, p.u_off[l]), MI, da);   // du
    TFR_LAUNCH_OK();
    rc = dense_grad16(p, ws, h16<T>(ws, p.x1_off[l]), E, E, da, I, M, false, grads + p.w1(l), st);
    if (rc) return rc;
    rc = bgemm(da, I, wb + p.sh_w1(l), I, tmp, E, M, E, I, nullptr, st);
    if (rc) return rc;
    add_kernel<<<blocks_for(ME, 256), 256, 0, st>>>(tmp, dres, ME, g);   // d x'
    TFR_LAUNCH_OK();
    // x' = LN_1(drop(o Wo + bo) + x)
    rc = ln_bwd16(p, ws, g, p.xh1_off[l], p.rs1_off[l], params + p.g1(l), p.hdrop,
                     site_seed(p.seed, p.site_h1(l)), dres, dy, grads + p.g1(l), st);
    if (rc) return rc;
    rc = dense_grad16(p, ws, h16<T>(ws, p.o_off[l]), E, E, dy, E, M, false, grads + p.wo(l), st);
    if (rc) return rc;
    rc = bgemm(dy, E, wb + p.sh_wo(l), E, dO, E, M, E, E, nullptr, st);
    if (rc) return rc;
    rc = din16_attn_bwd(h16<T>(ws, p.qkv_off[l]), mask, p.S, p.L, p.H, p.dh, p.adrop,
                           site_seed(p.seed, p.site_attn(l)), h16<T>(ws, p.o_off[l]),
                           ws + p.lse_off[l], dO, ws + p.dsum_off, dqkv, st);
    if (rc) return rc;
    const T* x = h16<T>(ws, p.xs_off[l]);
    rc = dense_grad16(p, ws, x, E, E, dqkv, 3 * E, M, false, grads + p.wqkv(l), st);
    if (rc) return rc;
    rc = bgemm(dqkv, 3 * E, wb + p.sh_wqkv(l), 3 * E, tmp, E, M, E, 3 * E, nullptr, st);
    if (rc) return rc;
    add_kernel<<<blocks_for(ME, 256), 256, 0, st>>>(tmp, dres, ME, g);   // d x
    TFR_LAUNCH_OK();
  }
  // embeddings: fp32 d sum for the tables' segment sums
  float* dsum_e = ws + p.dy_off;
  rc = ln_bwd(p, ws, g, p.xhe_off, p.rse_off, params + p.emb_g, p.hdrop,
              site_seed(p.seed, p.site_emb()), 0.f, 0, nullptr, dsum_e, grads + p.emb_g, st);
  if (rc) return rc;
  void* ews = ws + p.emb_ws_off;
  rc = tfr_embedding_bwd(wid, M, 1, dsum_e, E, 1, p.V, E, TFR_COMBINER_SUM, 0, ews,
                         grads + p.word, nullptr, st);
  if (rc) return rc;
  rc = tfr_embedding_bwd(reinterpret_cast<const int32_t*>(ws + p.pos_ids_off), M, 1, dsum_e, E, 1,
                         p.P, E, TFR_COMBINER_SUM, 0, ews, grads + p.pos, nullptr, st);
  if (rc) return rc;
  return tfr_embedding_bwd(tid, M, 1, dsum_e, E, 1, p.Tv, E, TFR_COMBINER_SUM, 0, ews,
                           grads + p.type, nullptr, st);
}

float* ws_align(void* w) {
  uintptr_t a = reinterpret_cast<uintptr_t>(w);
  return reinterpret_cast<float*>((a + 255) & ~(uintptr_t)255);
}

}  // namespace
}  // namespace tfr

using namespace tfr;

extern "C" size_t tfr_bert_param_count(const tfr_bert_cfg* cfg) {
  if (check_bert_cfg(cfg)) return 0;
  BertPlan p;
  std::memset(&p, 0, sizeof(p));
  param_layout(cfg, &p);
  return p.n_params;
}

extern "C" size_t tfr_bert_workspace_bytes(const tfr_bert_cfg* cfg, int S, int L) {
  BertPlan p;
  if (make_bert_plan(cfg, S, L, &p)) return 0;
  return p.ws_floats * sizeof(float) + 256;
}

extern "C" int tfr_bert_fwd(const int32_t* word_ids, const uint8_t* input_mask,
                            const int32_t* type_ids, int S, int L, const tfr_bert_cfg* cfg,
                            const float* params, void* workspace, float* scores, int* bad_ids,
                            void* stream) {
  int rc = check_bert_cfg(cfg);
  if (rc) return rc;
  rc = check_bert_shape(cfg, S, L);
  if (rc) return rc;
  TFR_REQUIRE(word_ids && input_mask && type_ids && params && workspace && scores,
              "NULL argument");
  if (S == 0) return TFR_OK;
  BertPlan p;
  rc = make_bert_plan(cfg, S, L, &p);
  if (rc) return rc;
  if (p.f16)
    return bert_fwd16<__half>(word_ids, input_mask, type_ids, p, params, ws_align(workspace),
                              scores, bad_ids, (cudaStream_t)stream);
  if (p.h16)
    return bert_fwd16<bf16>(word_ids, input_mask, type_ids, p, params, ws_align(workspace), scores,
                            bad_ids, (cudaStream_t)stream);
  return bert_fwd(word_ids, input_mask, type_ids, p, params, ws_align(workspace), scores, bad_ids,
                  (cudaStream_t)stream);
}

extern "C" int tfr_bert_bwd(const int32_t* word_ids, const uint8_t* input_mask,
                            const int32_t* type_ids, int S, int L, const tfr_bert_cfg* cfg,
                            const float* params, const float* dscores, void* workspace,
                            float* grads, void* stream) {
  int rc = check_bert_cfg(cfg);
  if (rc) return rc;
  rc = check_bert_shape(cfg, S, L);
  if (rc) return rc;
  TFR_REQUIRE(word_ids && input_mask && type_ids && params && dscores && workspace && grads,
              "NULL argument");
  BertPlan p;
  rc = make_bert_plan(cfg, S, L, &p);
  if (rc) return rc;
  if (S == 0) {
    TFR_CUDA_OK(cudaMemsetAsync(grads, 0, p.n_params * sizeof(float), (cudaStream_t)stream));
    return TFR_OK;
  }
  if (p.f16)
    return bert_bwd16<__half>(word_ids, input_mask, type_ids, p, params, dscores,
                              ws_align(workspace), grads, (cudaStream_t)stream);
  if (p.h16)
    return bert_bwd16<bf16>(word_ids, input_mask, type_ids, p, params, dscores,
                            ws_align(workspace), grads, (cudaStream_t)stream);
  return bert_bwd(word_ids, input_mask, type_ids, p, params, dscores, ws_align(workspace), grads,
                  (cudaStream_t)stream);
}
