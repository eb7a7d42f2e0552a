/*
 * tfr_b200.h — C ABI of the H100-native learning-to-rank hot path.
 *
 * The reference (tensorflow/ranking) has no FFI: its seam is the Python class
 * surface `tfr.keras.losses / tfr.keras.metrics / tfr.keras.model`
 * (SURVEY.md §8b).  This header is the C boundary a replacement for that path
 * binds to; `ranking_b200/_C.py` is the ctypes binding, and INTEGRATION.md shows
 * the stub a tensorflow_ranking maintainer would add.  Each entry point cites
 * the reference code it replaces (paths relative to tensorflow_ranking/python/).
 *
 * Conventions
 *   - every data pointer is a DEVICE pointer owned by the caller unless the
 *     name ends in `_host` or the entry point says otherwise (tfr_elwc_parse works on
 *     host buffers); the library never allocates or frees caller memory
 *   - config structs are HOST pointers, read during the call
 *   - `stream` is a cudaStream_t passed as void*; calls are stream-ordered,
 *     re-entrant and keep no global state besides the last-error string
 *   - return value: 0 on success, a tfr_status otherwise; tfr_last_error() gives
 *     the message (argument errors map to Python ValueError, as the reference
 *     raises for bad keys / shapes: keras/losses.py:108-109, losses_impl.py:52-58)
 *   - scores/labels/weights are row-major fp32 [B, N]; a label < 0 marks padding
 *     (utils.py:78-81) unless an explicit `mask` (uint8, 1 = valid) is given
 */
#ifndef TFR_B200_H_
#define TFR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  TFR_OK = 0,
  TFR_INVALID_ARGUMENT = 1,
  TFR_UNSUPPORTED = 2,
  TFR_CUDA_ERROR = 3
} tfr_status;

/* phi of the pairwise family: losses_impl.py:933-998 */
typedef enum {
  TFR_PHI_LOGISTIC = 0,      /* PairwiseLogisticLoss  :933-940 */
  TFR_PHI_HINGE = 1,         /* PairwiseHingeLoss     :943-948 */
  TFR_PHI_SOFT_ZERO_ONE = 2, /* PairwiseSoftZeroOneLoss :951-958 */
  TFR_PHI_MSE = 3            /* PairwiseMSELoss       :961-998 */
} tfr_phi;

/* LambdaWeight family: losses_impl.py:170-454 */
typedef enum {
  TFR_LAMBDA_NONE = 0,
  TFR_LAMBDA_LABEL_DIFF = 1, /* :210-216 */
  TFR_LAMBDA_DCG = 2,        /* :299-369 (NDCG = normalized) */
  TFR_LAMBDA_DCG_V2 = 3,     /* :372-394 */
  TFR_LAMBDA_YETI = 4,       /* :397-407 */
  TFR_LAMBDA_PRECISION = 5   /* :410-454 */
} tfr_lambda_kind;

/* gain functions: keras/utils.py:50-91 */
typedef enum {
  TFR_GAIN_IDENTITY = 0,
  TFR_GAIN_POW2_MINUS_1 = 1,
  TFR_GAIN_TABLE = 2         /* caller supplies gain_fn(cleaned labels) [B, N] */
} tfr_gain_fn;

/* rank discount functions: keras/utils.py:65-107, losses_impl.py:111 */
typedef enum {
  TFR_DISC_INVERSE = 0,       /* divide_no_nan(1, r) */
  TFR_DISC_LOG2_INVERSE = 1,  /* ln2 / ln(1 + r) */
  TFR_DISC_LOG1P_INVERSE = 2, /* 1 / ln(1 + r) */
  TFR_DISC_TABLE = 3          /* caller supplies disc[r], r = 0 .. N+1 */
} tfr_disc_fn;

typedef struct {
  int32_t kind;            /* tfr_lambda_kind */
  int32_t topn;            /* <= 0 means list_size */
  int32_t gain_fn;         /* tfr_gain_fn; for PRECISION: table = positive_fn(labels) or
                              IDENTITY meaning labels >= 1 */
  int32_t disc_fn;         /* tfr_disc_fn */
  int32_t normalized;      /* multiply gains by inverse_max_dcg (:261-266) */
  float smooth_fraction;   /* alpha of :365-367 */
  const float* gain_table; /* device [B, N] or NULL */
  const float* disc_table; /* device [N + 2] or NULL */
} tfr_lambda_cfg;

const char* tfr_last_error(void);
int tfr_version(void);
/* number of CUDA kernels this library has launched so far in this process */
unsigned long long tfr_launch_count(void);

/* ---------------------------------------------------------------------------
 * K1  pairwise loss family, fused forward + backward, one CTA per list.
 * Replaces _PairwiseLoss._compute_unreduced_loss_impl and everything under it
 * (losses_impl.py:61-74, 483-537, 863-998) plus the LambdaWeight pair weights
 * (:170-454) without materialising any [B, N, N] tensor.
 *   W_ij = [l_i > l_j] valid_i valid_j lambda_ij w_i           (constant)
 *   loss_sum[b] = sum_ij W_ij phi((s_i - s_j)/T),  w_sum[b] = sum_ij W_ij,
 *   nnz[b] = #{W_ij != 0},  row_loss[b,i] = sum_j W_ij phi(.),
 *   grad[b,k] = grad_scale * d loss_sum[b] / d s_k
 * item_w: NULL, or [B, N] (w_per_item = 1), or [B] per-list (w_per_item = 0).
 * Any output pointer except loss_sum may be NULL.
 * ------------------------------------------------------------------------- */
int tfr_pairwise_loss_fwd_bwd(const float* scores, const float* labels,
                              const float* item_w, int w_per_item,
                              const uint8_t* mask, int B, int N,
                              float temperature, int phi,
                              const tfr_lambda_cfg* lam_host, float grad_scale,
                              float* grad, float* row_loss, float* loss_sum,
                              float* w_sum, float* nnz, int32_t* ranks_out,
                              void* stream);

/* Parity helper: materialise lambda pair weights [B, N, N] for given ranks
 * (_LambdaWeight.pair_weights, losses_impl.py:181-193).  Small N only. */
int tfr_lambda_pair_weights(const float* labels, const int32_t* ranks, int B,
                            int N, const tfr_lambda_cfg* lam_host, float* out,
                            void* stream);

/* 1-based ranks of scores, descending, ties by index, invalid entries last
 * (losses_impl.py:483-500 + utils.py:167-195 with shuffle_ties=False). */
int tfr_sorted_ranks(const float* scores, const float* labels,
                     const uint8_t* mask, int B, int N, int32_t* ranks,
                     void* stream);

/* ---------------------------------------------------------------------------
 * K2  ApproxNDCG (mode 0) / ApproxMRR (mode 1), fused forward + backward.
 * Replaces approx_ranks, ndcg, inverse_max_dcg, _safe_default_gain_fn and the
 * two loss classes (losses_impl.py:33-49, 77-167, 1579-1632).
 *   loss[b]   = -ndcg_b (or -mrr_b)                       (unweighted)
 *   weight[b] = [sum l > 0] * (item_w ? sum(w l)/sum(l) : 1)   (:1004-1015,1602)
 *   grad[b,k] = grad_scale * (scale_by_weight ? weight[b] : 1) * d loss[b]/d s_k
 * ------------------------------------------------------------------------- */
int tfr_approx_loss_fwd_bwd(const float* scores, const float* labels,
                            const float* item_w, int w_per_item,
                            const uint8_t* mask, int B, int N,
                            float temperature, int mode, float grad_scale,
                            int scale_by_weight, float* grad, float* loss,
                            float* weight, void* stream);

/* ---------------------------------------------------------------------------
 * K3  Softmax loss, fused forward + backward (losses_impl.py:1119-1197, with
 * DCGLambdaWeight.individual_weights :281-296 when lam_host->kind == DCG).
 *   loss[b] = xent(l'/sum l', s/T masked to ln 1e-10), weight[b] = sum l'
 *   where l' = (lambda individual weight or label) * item weight
 * ------------------------------------------------------------------------- */
int tfr_softmax_loss_fwd_bwd(const float* scores, const float* labels,
                             const float* item_w, int w_per_item,
                             const uint8_t* mask, int B, int N,
                             float temperature, const tfr_lambda_cfg* lam_host,
                             float grad_scale, int scale_by_weight, float* grad,
                             float* loss, float* weight, void* stream);

/* ---------------------------------------------------------------------------
 * K3b  Pointwise and remaining listwise losses, fused forward + backward.
 *   SIGMOID_CE     SigmoidCrossEntropyLoss  losses_impl.py:1425-1446
 *   MEAN_SQUARED   MeanSquaredLoss          :1449-1469   (pass temperature = 1)
 *     item weight w_i = (label_i >= 0 ? w : 0) * mask_i  (:1287-1293);
 *     row[b,i] = loss_i * w_i (optional), loss[b] = sum_i row, weight[b] = sum_i w_i,
 *     nonzero[b] = #{w_i != 0}; grad = grad_scale * d loss[b] / d scores.
 *   UNIQUE_SOFTMAX UniqueSoftmaxLoss        :1250-1281
 *   LIST_MLE       ListMLELoss              :1541-1576; rank_weight (optional, [N]) is
 *     ListMLELambdaWeight's discount of ranks 1..N (:457-480).  Label ties are ordered
 *     by index (the reference shuffles them randomly); invalid items are last.
 *     loss[b] = list loss, weight[b] = label-weighted mean of the item weights
 *     (:1004-1015, 1 without weights); grad = grad_scale * d loss[b] / d scores.
 *     With order_scores [B, N] the order is a plain descending sort of those scores and
 *     only the first topk (> 0) positions contribute: the Plackett-Luce term of
 *     CoupledRankDistilLoss (:1984-2116) for one sampled teacher permutation; weight[b]
 *     is then additionally zero for lists whose cleaned labels sum to 0.
 * ------------------------------------------------------------------------- */
typedef enum {
  TFR_MISC_SIGMOID_CE = 0,
  TFR_MISC_MEAN_SQUARED = 1,
  TFR_MISC_UNIQUE_SOFTMAX = 2,
  TFR_MISC_LIST_MLE = 3
} tfr_misc_loss;

int tfr_misc_loss_fwd_bwd(const float* scores, const float* labels,
                          const float* item_w, int w_per_item,
                          const uint8_t* mask, int B, int N, float temperature,
                          int kind, const float* rank_weight,
                          const float* order_scores, int topk, float grad_scale,
                          float* grad, float* row, float* loss, float* weight,
                          float* nonzero, void* stream);

/* ---------------------------------------------------------------------------
 * K3c  Listwise losses of losses_impl.py outside the Keras RankingLossKey subset
 * (SURVEY.md §8 f1), one CTA per list, nothing of size N x N in memory:
 *   CIRCLE            CircleLoss                  losses_impl.py:1036-1116
 *     scores are clipped to [0, 1] (no temperature); p0 = gamma, p1 = margin;
 *     loss[b] = log1p(sum over pairs l_i > l_j of exp(gamma (a_i + c_j)));
 *     weight[b] = list weight * (#pairs / #pairs): NaN for a list without a valid pair,
 *     as the reference's sum(w) / count(w > 0) (:1108-1110).
 *   NEURAL_SORT_CE    NeuralSortCrossEntropyLoss  losses_impl.py:1635-1675
 *   NEURAL_SORT_NDCG  NeuralSortNDCGLoss          losses_impl.py:1678-1708
 *     deterministic NeuralSort rows (losses_impl.py:1711-1801) of scores / temperature;
 *     weight[b] = list weight * [sum of the cleaned labels > 0].
 * loss[b] = list loss, grad = grad_scale * d loss[b] / d scores (raw scores).
 * ------------------------------------------------------------------------- */
typedef enum {
  TFR_EXTRA_CIRCLE = 0,
  TFR_EXTRA_NEURAL_SORT_CE = 1,
  TFR_EXTRA_NEURAL_SORT_NDCG = 2
} tfr_extra_loss;

int tfr_extra_loss_fwd_bwd(const float* scores, const float* labels,
                           const float* item_w, int w_per_item,
                           const uint8_t* mask, int B, int N, float temperature,
                           int kind, float p0, float p1, float grad_scale,
                           float* grad, float* loss, float* weight, void* stream);

/* OrdinalLoss (losses_impl.py:1850-1918): scores [B, N, K] (K = ordinal_size heads per
 * item), head k against [label >= k + 1] (+ the fractional part with
 * use_fraction_label); grad [B, N, K]; row / loss / weight / nonzero as for the
 * pointwise kinds of tfr_misc_loss_fwd_bwd. */
int tfr_ordinal_loss_fwd_bwd(const float* scores, const float* labels,
                             const float* item_w, int w_per_item,
                             const uint8_t* mask, int B, int N, int K,
                             float temperature, int use_fraction_label,
                             float grad_scale, float* grad, float* row,
                             float* loss, float* weight, float* nonzero,
                             void* stream);

/* ---------------------------------------------------------------------------
 * GumbelSampler.sample (losses_impl.py:540-649): `sample_size` perturbed copies of
 * every list; row b * sample_size + s of out_logits [B * sample_size, N] is
 *   log(softmax((scores[b] + G) / temperature) + 1e-20),
 *   G = -log(-log(u + 1e-20) + 1e-20),  items with label < 0 at log(1e-20).
 * u in [0, 1) is a counter hash: top 24 bits of splitmix64_mix(seed +
 * 0x9E3779B97F4A7C15 * (e + 1)) * 2^-24 for element e = (b * sample_size + s) * N + i
 * (the reference draws tf.random.uniform).  Labels / weights are tiled by the caller.
 * Forward: pass out_logits.  Backward: pass grad_out [B * sample_size, N] and
 * grad_scores [B, N] with the same seed (the noise is regenerated, not stored).
 * mode 1 samples the TEACHER of CoupledRankDistilLoss (losses_impl.py:2031-2046):
 * out = log(softmax((label valid ? label : log 1e-10) + G) + 1e-10); scores may be NULL,
 * forward only.
 * ------------------------------------------------------------------------- */
int tfr_gumbel_sample(const float* scores, const float* labels, int B, int N,
                      int sample_size, float temperature, uint64_t seed, int mode,
                      float* out_logits, const float* grad_out,
                      float* grad_scores, void* stream);

/* ---------------------------------------------------------------------------
 * K4  NDCG@k and MRR@k for several cut-offs in one launch; per-list shared-memory
 * bitonic sort, ties by index, invalid entries last.  Replaces
 * metrics_impl.py:63-151, 228-266, 429-459, 631-670 and utils.py:115-164.
 *   topns_host[n_topn]: cut-offs (<= 0 means list_size)
 *   ndcg/mrr: [B, n_topn];  ndcg_w / mrr_w: [B] per-list weights after the
 *   batch-average rule of metrics_impl.py:63-119 (single-process batch);
 *   raw: [B, 5] = {sum w, sum w*gain, sum gain, sum w*rel, sum rel} per list,
 *   rel = [label >= 1] — required scratch; data-parallel callers all-reduce the
 *   batch statistics derived from it (the rule couples lists across ranks)
 * gain_fn / disc_fn as above (tables: gain_table [B,N] of cleaned labels,
 * disc_table [N+2]).  Any of ndcg/mrr may be NULL.
 * ------------------------------------------------------------------------- */
int tfr_rank_metrics(const float* scores, const float* labels,
                     const float* item_w, int w_per_item, const uint8_t* mask,
                     int B, int N, const int32_t* topns_host, int n_topn,
                     int gain_fn, int disc_fn, const float* gain_table,
                     const float* disc_table, float* ndcg, float* ndcg_w,
                     float* mrr, float* mrr_w, float* raw, void* stream);

/* The same launch can also emit the other metrics of `default_keras_metrics()`
 * (keras/metrics.py:131-153) from the one score sort; every pointer is optional.
 *   dcg        [B, T]  sum_{k < cut} w gain(l) disc(k)       DCGMetric  :673-705
 *                      (divide by ndcg_w for the reference's per-list value)
 *   precision  [B, T]  #rel in top cut / min(cut, #valid)    PrecisionMetric :180-207, 564
 *   recall     [B, T]  #rel in top cut / #rel                RecallMetric :154-177, 539
 *   map        [B, T]  MeanAveragePrecisionMetric :589-628
 *   hits       [B, T]  HitsMetric :462-506
 *   arp        [B, 2]  {value, per-list weight = sum w l}    ARPMetric :509-536
 *   opa        [B, 2]  {value, per-list weight}              OPAMetric :708-743
 *   bpref      [B, T]  BPrefMetric :825-898, TREC form (use_trec_version=True)
 *   bpref_alt  [B, T]  the same with R as the denominator (use_trec_version=False)
 * precision / recall / map / hits / bpref use mrr_w as their per-list weight (relevance =
 * [label >= 1]); dcg uses ndcg_w. */
typedef struct {
  float* dcg;
  float* precision;
  float* recall;
  float* map;
  float* hits;
  float* arp;
  float* opa;
  float* bpref;
  float* bpref_alt;
} tfr_metric_ext;

/* Shared memory per list: 8 P + 17 N + 144 bytes (P = next power of two >= N), plus 1 KB
 * when any extended output is requested: 205,968 bytes at N = 8192, so every output works up
 * to the 8192-item maximum on an H100 (232,448-byte opt-in limit).  The size is checked
 * against the device's opt-in limit before any CUDA call; a list that does not fit returns
 * TFR_INVALID_ARGUMENT with a message naming the largest list_size accepted for the call. */
int tfr_rank_metrics_ext(const float* scores, const float* labels,
                         const float* item_w, int w_per_item,
                         const uint8_t* mask, int B, int N,
                         const int32_t* topns_host, int n_topn, int gain_fn,
                         int disc_fn, const float* gain_table,
                         const float* disc_table, float* ndcg, float* ndcg_w,
                         float* mrr, float* mrr_w, float* raw,
                         const tfr_metric_ext* ext, void* stream);

/* Diversity metrics (metrics_impl.py:313-427, 746-823): labels [B, N, S] hold per-subtopic
 * relevance (-1 pads).  precision_ia / alpha_dcg: [B, n_topn] (alpha_dcg unnormalised:
 * divide by list_w for the reference's per-list value); list_w [B]: per-list weights
 * with relevance = [any subtopic >= 1]; raw [B, 5] scratch as in tfr_rank_metrics.
 * Shared memory per list: 8 P + 17 N + 4 S + 1,168 bytes: at most 222,352 bytes at N = 8192,
 * S = 4096, so every N <= 8192 and S <= 4096 fits an H100; checked and rejected like
 * tfr_rank_metrics_ext on devices with less. */
int tfr_div_metrics(const float* scores, const float* labels, const float* item_w,
                    int w_per_item, const uint8_t* mask, int B, int N, int S,
                    const int32_t* topns_host, int n_topn, float alpha,
                    int disc_fn, const float* disc_table, float* precision_ia,
                    float* alpha_dcg, float* list_w, float* raw, void* stream);


/* out2[0] = scale * sum_i v[i] * (w ? w[i] : 1); out2[1] = sum_i (w ? w[i] : 1).
 * Deterministic single-CTA reduction (Keras Mean state / loss reduction). */
int tfr_weighted_sum(const float* v, const float* w, int n, float scale,
                     float* out2, void* stream);

/* ---------------------------------------------------------------------------
 * K5/K6  scorer tower: create_tower (keras/layers.py:26-77) over the flattened
 * [M = B*N, D] matrix + RestoreList fill (keras/layers.py:231-265).
 * Parameters live in ONE flat fp32 buffer (so data-parallel training needs a
 * single all-reduce): for each Dense i: W_i [in, out] row-major (Keras kernel
 * layout) then b_i [out].  Gradients use the same layout.
 * precision: how the GEMMs are evaluated
 *   TFR_PREC_FP32   fp32 CUDA-core FFMA
 *   TFR_PREC_TF32X3 wgmma tf32, 3-pass error-compensated split (~fp32)
 *   TFR_PREC_TF32   wgmma tf32, 1 pass
 *   TFR_PREC_BF16   wgmma bf16 (bf16 operands, fp32 accumulate)
 * ------------------------------------------------------------------------- */
typedef enum {
  TFR_PREC_FP32 = 0,
  TFR_PREC_TF32X3 = 1,
  TFR_PREC_TF32 = 2,
  TFR_PREC_BF16 = 3
} tfr_precision;

typedef enum { TFR_ACT_NONE = 0, TFR_ACT_RELU = 1 } tfr_activation;

#define TFR_MLP_MAX_LAYERS 8

typedef struct {
  int32_t n_dense;                        /* Dense layers incl. the output one */
  int32_t dims[TFR_MLP_MAX_LAYERS + 1];   /* dims[0] = D, dims[i] = units of Dense i */
  int32_t activation;                     /* tfr_activation, hidden layers */
  /* create_tower options (keras/layers.py:65-76).  Layer order per hidden layer:
   * Dense -> [BatchNormalization] -> activation -> [Dropout]. */
  int32_t use_batch_norm;                 /* BN after every hidden Dense (:71-72) */
  int32_t input_batch_norm;               /* BN on the inputs (:67-68) */
  float bn_epsilon;                       /* Keras default 1e-3 */
  float bn_momentum;                      /* `batch_norm_moment`, default 0.999 */
  float dropout;                          /* rate in [0, 1) (:74-75) */
  int32_t training;                       /* 1: batch statistics, moving-average update,
                                             dropout active; 0: inference */
  uint64_t dropout_seed;                  /* vary per step; same value -> same mask.
                                             Dropout mask: element i (row-major) of hidden
                                             layer d is dropped iff u < dropout, with
                                             u = (splitmix64_mix(s + 0x9E3779B97F4A7C15 *
                                             (i + 1)) >> 40) * 2^-24 and
                                             s = seed * 0x100000001B3 + d + 1; kept
                                             values are scaled by 1 / (1 - dropout). */
  float* bn_state;                        /* device, tfr_mlp_bn_state_count floats: per BN
                                             layer (input BN first) moving_mean[w] then
                                             moving_variance[w]; required with any BN */
} tfr_mlp_cfg;

/* Flat parameter layout: W_0 [dims0, dims1] (Keras kernel layout), b_0, W_1, b_1, ...
 * then, if input_batch_norm, gamma[D], beta[D]; then for every hidden layer with BN
 * gamma[h], beta[h].  Gradients use the same layout. */
size_t tfr_mlp_param_count(const tfr_mlp_cfg* cfg);
size_t tfr_mlp_bn_state_count(const tfr_mlp_cfg* cfg);
/* bytes of caller-provided workspace that carries activations from fwd to bwd */
size_t tfr_mlp_workspace_bytes(const tfr_mlp_cfg* cfg, int M);

/* X [M, dims[0]] row-major: fp32 for TFR_PREC_FP32 / TF32X3 / TF32, bf16 (2-byte) for
 * TFR_PREC_BF16 — in that mode hidden activations and backward signals are also bf16 in
 * the workspace, parameters / gradients / scores stay fp32, layer widths must be
 * multiples of 8 and BatchNormalization / Dropout are not offered.
 * scores_out [M, dims[n_dense]]; if mask (uint8 [M]) is given and the output
 * width is 1, masked-out rows are set to ln(1e-10) (RestoreList). */
int tfr_mlp_fwd(const void* X, int M, const tfr_mlp_cfg* cfg,
                const float* params, const uint8_t* mask, void* workspace,
                float* scores_out, int precision, void* stream);

/* dscores [M, dims[n_dense]] -> grads (flat, same layout as params).
 * Must follow a tfr_mlp_fwd on the same X / workspace. */
int tfr_mlp_bwd(const void* X, int M, const tfr_mlp_cfg* cfg,
                const float* params, const float* dscores, const uint8_t* mask,
                void* workspace, float* grads, int precision, void* stream);

/* ---------------------------------------------------------------------------
 * K10  neural additive ranking model: GAMLayer (keras/layers.py:591-803) over the
 * flattened [M = B*N] rows.  Example feature f owns columns [feature_offsets[f],
 * feature_offsets[f + 1]) of X [M, D] (D = feature_offsets[F], feature_offsets[0] = 0,
 * width d_f in [1, 32]) and has its own tower create_tower(hidden, 1): Dense -> [BN] ->
 * activation -> [Dropout] per hidden layer, then Dense(1); s_f = tower_f(x_f).
 * Context feature j (input [M, context_dims[j]]) has a tower create_tower(context_hidden,
 * F) followed by a softmax over its F outputs; w = sum_j softmax_j and
 *   logits = sum_f s_f w_f      (with context inputs)
 *   logits = sum_f s_f          (without; also when n_context > 0 and none are passed)
 * Limits: F <= TFR_GAM_MAX_FEATURES, 0..4 example hidden layers of width 1..64, d_f <= 32;
 * context towers need F <= 8 (the tower kernels' output_units limit).
 *
 * Flat parameter layout: example towers 0..F-1, then context towers 0..C-1; every tower's
 * slice is exactly the tfr_mlp layout of its dims (W_0, b_0, ..., W_L, b_L, then BN
 * gamma / beta per hidden layer).  bn_state is concatenated in the same tower order, each
 * slice the tfr_mlp bn_state layout.  Gradients use the parameter layout.
 * Dropout: example tower f, hidden layer d (width h) drops (row m, unit u) iff the
 * tfr_mlp mask of the block-diagonal layer of width F*h drops element m*(F*h) + f*h + u
 * (same seed s = dropout_seed * 0x100000001B3 + d + 1); a one-feature GAM without context
 * therefore draws exactly the mask of the equivalent tower.  Context tower j draws the
 * tfr_mlp mask of its own dims with dropout_seed + (j + 1) * 0xD1B54A32D192ED03.
 * Example towers are evaluated on chip, one (row, feature) tower per thread, recomputed
 * from X in every sweep: no per-feature hidden activation is ever written to memory.
 * ------------------------------------------------------------------------- */
#define TFR_GAM_MAX_FEATURES 512
#define TFR_GAM_MAX_HIDDEN 4
#define TFR_GAM_MAX_CONTEXT 16

typedef struct {
  int32_t n_features;                                  /* F >= 1 */
  int32_t feature_offsets[TFR_GAM_MAX_FEATURES + 1];   /* column offsets into X, F + 1 */
  int32_t n_hidden;                                    /* example hidden layers, 0..4 */
  int32_t hidden[TFR_GAM_MAX_HIDDEN];                  /* shared example hidden widths */
  int32_t n_context;                                   /* C, 0..TFR_GAM_MAX_CONTEXT */
  int32_t context_dims[TFR_GAM_MAX_CONTEXT];           /* input width of context tower j */
  int32_t n_context_hidden;                            /* >= 0 */
  int32_t context_hidden[TFR_MLP_MAX_LAYERS - 1];
  /* create_tower options, as in tfr_mlp_cfg (no input BN) */
  int32_t activation;
  int32_t use_batch_norm;
  float bn_epsilon;
  float bn_momentum;
  float dropout;
  int32_t training;
  uint64_t dropout_seed;
  float* bn_state;                                     /* device, tfr_gam_bn_state_count */
} tfr_gam_cfg;

/* 0 when the configuration is out of range (tfr_last_error says why) */
size_t tfr_gam_param_count(const tfr_gam_cfg* cfg);
size_t tfr_gam_bn_state_count(const tfr_gam_cfg* cfg);
size_t tfr_gam_workspace_bytes(const tfr_gam_cfg* cfg, int M);

/* X [M, D] fp32; context_host: NULL (no context) or a HOST array of n_context device
 * pointers, context j fp32 [M, context_dims[j]].  logits [M] with the RestoreList
 * ln(1e-10) fill where mask (uint8 [M], optional) is 0; sublogits [M, F] and subweights
 * [C, M, F] (the per-context-tower softmax outputs) are optional. */
int tfr_gam_fwd(const float* X, const float* const* context_host, int M,
                const tfr_gam_cfg* cfg, const float* params, const uint8_t* mask,
                void* workspace, float* logits, float* sublogits, float* subweights,
                void* stream);
/* dlogits [M] -> grads (flat, parameter layout; context towers get 0 when no context is
 * passed).  Must follow a tfr_gam_fwd with the same inputs, cfg and workspace. */
int tfr_gam_bwd(const float* X, const float* const* context_host, int M,
                const tfr_gam_cfg* cfg, const float* params, const float* dlogits,
                const uint8_t* mask, void* workspace, float* grads, void* stream);

/* ---------------------------------------------------------------------------
 * K8  groupwise scoring folded into the tower (tfr.model._GroupwiseRankingModel,
 * model.py:273-421; group formation model.py:164-244 stays with the caller).
 *   X      [B * N, D] fp32 item features (NOT gathered)
 *   idx    [B, G, gs] int32: list positions of the members of every group; G = S * N
 *          (S = num_shuffles blocks of N rolling-window groups)
 *   gmask  [B, G] uint8: group validity (`indices_mask`)
 *   cfg    the group score function as a tower over the concatenated member features:
 *          dims[0] = gs * D, >= 1 hidden layer, output_units = gs
 *          (examples/tf_ranking_libsvm.py:313-349); no BN / Dropout on this path
 *   logits [B, N]: mean of the member scores every item received, 0 for items in no
 *          valid group (scatter_nd + div_no_nan, model.py:388-412)
 * The first Dense layer runs on the ungathered matrix (one GEMM per member slot) and the
 * gather happens on its [B * N, h1] outputs, so the [B, G, gs, D] tensor of the reference
 * is never formed.  precision: TFR_PREC_TF32X3 or TFR_PREC_TF32.
 * Within one shuffle block an item may occupy a given slot in at most one valid group
 * (true for rolling windows); tfr_group_mlp_check (host-synchronising) reports a
 * violation seen by the last forward.
 * ------------------------------------------------------------------------- */
/* K9  FlattenList's circular padding (keras/layers.py:163-173, utils.py:272-356): out[b, p]
 * = x[b, organized[p mod nv]] where organized lists the valid positions of list b in order
 * (then the invalid ones) and nv is their count — every slot of the flattened batch holds a
 * copy of a VALID row, which is what BatchNormalization statistics see in the reference.
 * x / out [B, N, row_bytes] (row_bytes % 16 == 0), is_valid [B, N] uint8, idx_out [B, N]
 * int32 (the gather indices, = utils.padded_nd_indices). */
int tfr_circular_pad_gather(const void* x, const uint8_t* is_valid, int B, int N,
                            int row_bytes, int32_t* idx_out, void* out, void* stream);

/* Group formation on the device (model.py:164-244): is_valid [B, N] uint8; perm NULL
 * (no shuffle: the reference's PREDICT mode) or [num_shuffles, B, N] int32 permutations
 * of the valid-first order (TF's shuffle stream is not reproducible, so the shuffle is an
 * input); idx [B, num_shuffles * N, gs] int32, gmask [B, num_shuffles * N] uint8. */
int tfr_group_indices(const uint8_t* is_valid, const int32_t* perm, int B, int N,
                      int num_shuffles, int gs, int32_t* idx, uint8_t* gmask, void* stream);
size_t tfr_group_mlp_workspace_bytes(const tfr_mlp_cfg* cfg, int B, int N, int G, int gs);
int tfr_group_mlp_fwd(const float* X, int B, int N, int G, int gs, const int32_t* idx,
                      const uint8_t* gmask, const tfr_mlp_cfg* cfg, const float* params,
                      void* workspace, float* logits_out, int precision, void* stream);
int tfr_group_mlp_bwd(const float* X, int B, int N, int G, int gs, const int32_t* idx,
                      const uint8_t* gmask, const tfr_mlp_cfg* cfg, const float* params,
                      const float* dlogits, void* workspace, float* grads, int precision,
                      void* stream);
int tfr_group_mlp_check(const tfr_mlp_cfg* cfg, int B, int N, int G, int gs,
                        void* workspace, void* stream);

/* Parity helper: one GEMM through the wgmma TF32 engine that the scorer tower
 * uses (D[GM,GN] = A[GM,GK] * B[GK,GN]).  a_mn/b_mn select the operand storage
 * (0: K contiguous, i.e. A stored [GM,GK], B stored [GN,GK]; 1: M/N contiguous,
 * i.e. A stored [GK,GM], B stored [GK,GN]); passes 1 = TF32, 3 = 3xTF32 (fp32-
 * faithful); epi 0 store, 1 bias+act (optionally writing ReLU sign bits to
 * mask_bits_out, word [(col / 32) * GM + row]), 2 relu-mask by aux, 3 relu-mask by
 * mask_bits_in.  See csrc/tc_gemm.cuh. */
int tfr_tc_gemm(const float* A, int lda, const float* B, int ldb, const float* B_lo,
                float* C, int ldc, int GM, int GN, int GK, int a_mn, int b_mn,
                int passes, int split_b, int epi, const float* bias,
                const float* aux, int act, int store_transposed, int splits,
                size_t split_stride, uint32_t* mask_bits_out,
                const uint32_t* mask_bits_in, void* stream);

/* Parity helper for the bf16 engine (Hopper wgmma, csrc/tc_gemm_bf16.cuh):
 * D[GM,GN] = A[GM,GK] * B[GK,GN] with bf16 operands and fp32 accumulation.
 *   mn = 0: A stored [GM,GK], B stored [GN,GK]; C bf16 [GM,GN]; epi 0 store, 1 bias+act
 *           (+ ReLU sign bits to mask_bits_out), 3 mask by mask_bits_in (+ fp32 column sums
 *           of C per CTA and epilogue warp into colsum[slot * colsum_stride + col],
 *           *colsum_slots_out slots);
 *   mn = 1: A stored [GK,GM], B stored [GK,GN]; the GK range is cut into `splits` pieces,
 *           piece z writes its fp32 partial to C + z * split_stride floats, with
 *           split_stride = roundup(GM, 128) * ldc. */
int tfr_tc_gemm_bf16(const void* A, int lda, const void* B, int ldb, void* C, int ldc,
                     int GM, int GN, int GK, int mn, int epi, const float* bias, int act,
                     uint32_t* mask_bits_out, const uint32_t* mask_bits_in,
                     float* colsum, int colsum_stride, int* colsum_slots_out,
                     int splits, size_t split_stride, void* stream);

/* ---------------------------------------------------------------------------
 * Input side (host code, no device work): a batch of serialized
 * `ExampleListWithContext` protos -> dense float buffers, with the padding /
 * truncation rules of data.py:133-208, 391-540 for FixedLen float / int64 features:
 *   context_out [B, sum context dims], example_out [B, list_size, sum example dims]
 *   (features in spec order; a missing feature or a padded slot takes its default; a
 *   present feature must have exactly `dim` values; int64 values are cast to float;
 *   examples past list_size are dropped), sizes_out [B] = untruncated list lengths,
 *   mask_out [B, list_size] = sequence_mask(sizes, list_size).  All pointers are HOST
 *   pointers (pinned memory recommended: the result feeds one H2D copy).  Lists are
 *   decoded in parallel by n_threads host threads (<= 0: all hardware threads).
 * tfr_masked_crc32c: the checksum of the TFRecord framing.
 * ------------------------------------------------------------------------- */
typedef struct {
  const char* name;
  int32_t dim;
  float default_value;
} tfr_feature_spec;

int tfr_elwc_parse(const uint8_t* const* records, const int64_t* record_sizes,
                   int B, int list_size, const tfr_feature_spec* context_spec,
                   int n_context, const tfr_feature_spec* example_spec,
                   int n_example, float* context_out, float* example_out,
                   int32_t* sizes_out, uint8_t* mask_out, int n_threads);
/* The other two record formats of data.py (`make_parsing_fn`, :857-911), same outputs:
 *   EXAMPLE_IN_EXAMPLE  an outer tf.Example with bytes features `serialized_context` and
 *                       `serialized_examples` (:133-208)
 *   SEQUENCE_EXAMPLE    context features in `context`, item i of every example feature in
 *                       frame i of its feature list (:572-711); the list length is the
 *                       longest requested feature list */
typedef enum {
  TFR_FORMAT_ELWC = 0,
  TFR_FORMAT_EXAMPLE_IN_EXAMPLE = 1,
  TFR_FORMAT_SEQUENCE_EXAMPLE = 2
} tfr_data_format;

int tfr_ranking_parse(int format, const uint8_t* const* records,
                      const int64_t* record_sizes, int B, int list_size,
                      const tfr_feature_spec* context_spec, int n_context,
                      const tfr_feature_spec* example_spec, int n_example,
                      float* context_out, float* example_out, int32_t* sizes_out,
                      uint8_t* mask_out, int n_threads);
uint32_t tfr_masked_crc32c(const uint8_t* data, size_t n);

/* ---------------------------------------------------------------------------
 * Fused optimizer over the flat parameter buffer (the reference delegates to
 * tf.keras.optimizers; Adagrad is what its examples use:
 * examples/tf_ranking_libsvm.py:386-387).  grad_scale multiplies the gradient
 * first (1/world_size for data parallel, extension/task.py:259).
 *   kind 0: SGD          p -= lr * g
 *   kind 1: Adagrad      a += g^2; p -= lr * g / (sqrt(a) + eps)   (Keras form)
 * ------------------------------------------------------------------------- */
int tfr_optimizer_step(float* params, const float* grads, float* accum, size_t n,
                       int kind, float lr, float eps, float grad_scale,
                       void* stream);

/* ---------------------------------------------------------------------------
 * K7  data-parallel step: all-reduce(SUM) of the flat gradient fused with the optimizer,
 * over NVLink peer memory (one process per GPU on one node).  Replaces the reference's
 * tf.distribute all-reduce + optimizer (keras/strategy_utils.py:45-116,
 * extension/task.py:256-262).
 *   tfr_dp_alloc   zero-filled device memory that peers may map + its 64-byte IPC handle
 *   tfr_dp_open    map a peer's allocation from its handle (exchange the handles with any
 *                  host-side channel, e.g. the process group)
 *   tfr_allreduce_optimizer_step
 *                  grad_ptrs / flag_ptrs: HOST arrays of `world` device pointers (own +
 *                  peer mappings): this step's gradient slot and the flag pad (>= 16
 *                  uint32, zero before the first step) of every rank.  `epoch` must grow by
 *                  one per step on every rank; alternate between TWO gradient slots from
 *                  step to step (the flag round of step e + 1 is what proves every peer
 *                  finished reading slot e % 2).  Sums in rank order (bit-identical
 *                  replicas), scales by grad_scale, applies kind 0 SGD / 1 Adagrad.
 *                  summed_out (optional): the unscaled sum.
 * ------------------------------------------------------------------------- */
int tfr_dp_alloc(size_t bytes, void** ptr_out, unsigned char* handle_out);
int tfr_dp_open(const unsigned char* handle, void** ptr_out);
int tfr_dp_close(void* peer_ptr);
int tfr_dp_free(void* ptr);
int tfr_allreduce_optimizer_step(const void* const* grad_ptrs, void* const* flag_ptrs,
                                 int rank, int world, uint32_t epoch, float* params,
                                 float* accum, float* summed_out, size_t n, int kind,
                                 float lr, float eps, float grad_scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif  /* TFR_B200_H_ */
