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
 * K3d  Click-model losses, fused forward + backward, one CTA per list, no float atomics
 * (two identical calls give identical bits).  Limits: 1 <= N <= 8192, temperature > 0.
 *
 * ClickEMLoss (losses_impl.py:1324-1422): examination logits e and relevance logits r,
 * element (b, i) at exam[(b N + i) stride] and rel[(b N + i) stride], stride 1 (two [B, N]
 * planes) or 2 (the Keras [B, N, 2] tensor in place: exam = base, rel = base + 1).
 *   valid_i = mask_i (if given) and label_i >= 0;  c_i = label_i >= 1 (clicked)
 *   e, r = e_i / T, r_i / T, both 0 on invalid items
 *   pe_i = c_i ? 1 : sigmoid(e - softplus(r)),  pr_i = c_i ? 1 : sigmoid(r - softplus(e))
 *          (posteriors; no gradient flows through them)
 *   loss_i = exam_weight * sce(pe_i, e) + rel_weight * sce(pr_i, r),
 *          sce(z, x) = max(x, 0) - x z + log1p(exp(-|x|))
 *   w_i = valid_i ? item weight : 0;  row[b, i] = loss_i w_i (optional),
 *   loss[b] = sum_i row, weight[b] = sum_i w_i, nonzero[b] = #{w_i != 0} (optional);
 *   d_exam = grad_scale exam_weight (sigmoid(e) - pe_i) w_i / T,
 *   d_rel  = grad_scale rel_weight (sigmoid(r) - pr_i) w_i / T, written with the input
 *   stride (both optional, both or neither); exactly 0 on invalid items.
 *
 * MixtureEMLoss (losses_impl.py:1472-1538): scores [B, N, M], 1 <= M <= 32 mixed models.
 *   valid_i = mask_i (if given) else label_i >= 0;  l_im = valid_i ? sce(label_i, s_im / T) : 0
 *   L_m = sum_i l_im (fp64),  q_m = exp(-alpha (L_m - min_k L_k)) (no gradient)
 *   loss[b] = sum_m q_m L_m / sum_m q_m
 *   weight[b] = list weight (sum_i w_i l_i / sum_i l_i over label_i >= 0, 1 without item_w;
 *               :1004-1015) x [sum of the valid labels > 0]
 *   grad[b, i, m] = grad_scale valid_i q_m / sum q (sigmoid(s_im / T) - label_i) / T
 *
 * Both return TFR_INVALID_ARGUMENT before any CUDA call for NULL inputs, N outside 1..8192,
 * M outside 1..32 or a stride other than 1 or 2.
 * ------------------------------------------------------------------------- */
int tfr_click_em_loss_fwd_bwd(const float* exam, const float* rel, int stride,
                              const float* labels, const float* item_w, int w_per_item,
                              const uint8_t* mask, int B, int N, float temperature,
                              float exam_weight, float rel_weight, float grad_scale,
                              float* d_exam, float* d_rel, float* row, float* loss,
                              float* weight, float* nonzero, void* stream);
int tfr_mixture_em_loss_fwd_bwd(const float* scores, const float* labels,
                                const float* item_w, int w_per_item, const uint8_t* mask,
                                int B, int N, int M, float temperature, float alpha,
                                float grad_scale, float* grad, float* loss, float* weight,
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
 *   TFR_PREC_FP16   wgmma fp16 (fp16 operands, fp32 accumulate): TFR-BERT only (K15); every
 *                   other entry point refuses it as it refuses an unknown value
 * ------------------------------------------------------------------------- */
typedef enum {
  TFR_PREC_FP32 = 0,
  TFR_PREC_TF32X3 = 1,
  TFR_PREC_TF32 = 2,
  TFR_PREC_BF16 = 3,
  TFR_PREC_FP16 = 4
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

/* Gradient of the tower's loss with respect to its input columns [col0, col0 + ncols):
 *   dX[m, c] (row pitch ldx) = sum_o dZ_0[m, o] W_0[col0 + c, o]
 * where dZ_0 is the gradient at the first Dense layer's pre-activation that the preceding
 * tfr_mlp_bwd or tfr_mlp_bwd_tasks (same cfg, M, params, workspace) left in the workspace.
 * Needs at least one hidden layer, precision TFR_PREC_TF32X3 or TFR_PREC_TF32 and no input BatchNormalization
 * (TFR_INVALID_ARGUMENT otherwise, before any CUDA call).  Does not change the workspace, so
 * tfr_mlp_bwd's results are the same with or without this call. */
int tfr_mlp_input_grad(const tfr_mlp_cfg* cfg, int M, const float* params, void* workspace,
                       int col0, int ncols, float* dX, int ldx, int precision, void* stream);

/* Multi-task scoring: one tower whose O = dims[n_dense] output units are O ranking tasks, in
 * a task-major ("planar") score layout that the per-list loss kernels read directly.
 *   score_planes [O, M]: score_planes[o * M + m] is row m's score for task o, so plane o is
 *   task o's [B, N] score matrix.  Unmasked values are bit-identical to tfr_mlp_fwd's
 *   scores_out[m * O + o]; if mask (uint8 [M]) is given, masked rows of EVERY plane are set to
 *   ln(1e-10) (RestoreList per task).
 * precision: TFR_PREC_FP32, TFR_PREC_TF32X3 or TFR_PREC_TF32.  1 <= O <= 8.  Anything else, and
 * NULL X / params / workspace / score_planes, is TFR_INVALID_ARGUMENT before any CUDA call.
 * The workspace is tfr_mlp_workspace_bytes(cfg, M), as for tfr_mlp_fwd. */
int tfr_mlp_fwd_tasks(const void* X, int M, const tfr_mlp_cfg* cfg, const float* params,
                      const uint8_t* mask, void* workspace, float* score_planes,
                      int precision, void* stream);

/* Backward of tfr_mlp_fwd_tasks (same X / workspace): the gradients tfr_mlp_bwd produces from
 * the interleaved signal dS[m, o] = w_o * dscore_planes[o * M + m], with rows the mask clears
 * set to 0 for every task.  task_weights_host: O host floats (the per-task loss weights), NULL
 * for all 1.  Same limits as tfr_mlp_fwd_tasks, plus dscore_planes / grads not NULL and every
 * weight finite (TFR_INVALID_ARGUMENT before any CUDA call).  tfr_mlp_input_grad may follow.
 * With O = 1, weight 1, the results are tfr_mlp_bwd's bits. */
int tfr_mlp_bwd_tasks(const void* X, int M, const tfr_mlp_cfg* cfg, const float* params,
                      const float* dscore_planes, const float* task_weights_host,
                      const uint8_t* mask, void* workspace, float* grads,
                      int precision, void* stream);

/* ---------------------------------------------------------------------------
 * K11  DocumentInteractionAttention (keras/layers.py:420-588): listwise self-attention over
 * the items of every list.  X [B, N, D] fp32 row-major, list_mask [B, N] uint8 (1 = valid;
 * NULL = all valid), h = head_size, H = num_heads, HH = H * h, L = num_layers.
 *   x_0 = relu(X W_in + b_in)                        (+ sigma g in training, GaussianNoise)
 *   per layer (Keras MultiHeadAttention, key_dim = output_shape = h):
 *     q = x Wq + bq, k = x Wk + bk, v = x Wv + bv    (kernels [h, H, h], biases [H, h])
 *     logit[b, head, i, j] = (q_i / sqrt(h)) . k_j, plus -1e9 (as an fp32 sum) when item j is
 *       padded (SelfAttentionMask: mask[b, i, j] = list_mask[b, j]); softmax over j.  Padded
 *       query rows attend to the valid items.  A list with no valid item attends uniformly
 *       while every |q_i . k_j / sqrt(h)| < 32: the fp32 spacing at 1e9 is 64, so larger
 *       logits round to -1e9 +- 64 (as in Keras) and the weights are no longer uniform.
 *     P~ = dropout(P) (training), o_i = sum_j P~_ij v_j, y = o Wo + bo  (Wo [H, h, h], bo [h])
 *     x_next = LayerNorm(dropout(y) + x), epsilon 1e-12, gamma / beta [h]
 *   out [B * N, h] with row pitch ldo: the last layer's LayerNorm output (ldo > h lets it land
 *   in a column block of a wider buffer, e.g. the scorer tower's input [X | out]).
 * Flat parameter layout (Keras get_weights() order): W_in [D, h], b_in [h], then per layer
 *   Wq [h, HH], bq [HH], Wk, bk, Wv, bv (same shapes), Wo [HH, h], bo [h], gamma [h], beta [h].
 *   Gradients use the same layout.
 * Random draws (training only), with u(s, e) the tower's counter hash (tfr_mlp_cfg dropout
 * mask: top 24 bits of splitmix64_mix(s + 0x9E3779B97F4A7C15 * (e + 1)) * 2^-24) and site
 * seeds s = seed * 0x100000001B3 + site:
 *   site 1          input noise, element e = m * h + c: g = sqrt(-2 ln(1 - u(s, 2e)))
 *                   * cos(2 pi u(s, 2e + 1))
 *   site 2 + 2 l    attention-probability dropout of layer l, element
 *                   e = ((b * H + head) * N + i) * N + j
 *   site 3 + 2 l    output dropout of layer l, element e = m * h + c
 *   an element is dropped iff u < dropout; kept values are scaled by 1 / (1 - dropout).
 * Precision (tfr_din_cfg.precision):
 *   TFR_PREC_FP32   (0, a zeroed struct)  projection GEMMs and input gradient in 3xTF32,
 *                   attention core (q.k, P~ v and their backward) in FP32 CUDA-core FMA
 *   TFR_PREC_TF32                         projection GEMMs and input gradient in one TF32
 *                   pass, attention core on wgmma TF32 (operands truncated to TF32, fp32
 *                   accumulate); softmax, masking and dropout in fp32 with the same draws
 *   any other value: TFR_INVALID_ARGUMENT.  The workspace is the same in both.
 * Limits (TFR_INVALID_ARGUMENT before any CUDA call): D % 4 == 0, h % 4 == 0, h <= 128,
 * 1 <= H * h <= 512, 1 <= L <= 8, N <= 1024.  Two identical calls give identical bits.
 * ------------------------------------------------------------------------- */
#define TFR_DIN_MAX_LAYERS 8
#define TFR_DIN_MAX_HH 512
#define TFR_DIN_MAX_LIST 1024

typedef struct {
  int32_t input_dim;            /* D */
  int32_t head_size;            /* h */
  int32_t num_heads;            /* H */
  int32_t num_layers;           /* L */
  float dropout;                /* rate in [0, 1) of both Dropout sites */
  float input_noise_stddev;     /* sigma; 0 = no GaussianNoise */
  int32_t training;             /* 1: dropout and noise active; 0: inference */
  uint64_t seed;                /* vary per step; same value -> same draws */
  int32_t precision;            /* TFR_PREC_FP32 (default) or TFR_PREC_TF32 */
} tfr_din_cfg;

/* 0 when the configuration is out of range (tfr_last_error says why) */
size_t tfr_din_param_count(const tfr_din_cfg* cfg);
size_t tfr_din_workspace_bytes(const tfr_din_cfg* cfg, int B, int N);
int tfr_din_fwd(const float* X, const uint8_t* list_mask, int B, int N, const tfr_din_cfg* cfg,
                const float* params, void* workspace, float* out, int ldo, void* stream);
/* dout [B * N, h] (row pitch lddo) -> grads (flat, parameter layout).  Must follow a
 * tfr_din_fwd with the same inputs, cfg and workspace.  The gradient with respect to X is
 * tfr_din_input_grad's, from what this call leaves in the workspace. */
int tfr_din_bwd(const float* X, const uint8_t* list_mask, int B, int N, const tfr_din_cfg* cfg,
                const float* params, const float* dout, int lddo, void* workspace,
                float* grads, void* stream);
/* Gradient of the DIN's loss with respect to its input columns [col0, col0 + ncols):
 *   dX[m, c] (row pitch ldx) (=, or += when accumulate) sum_o dZ_in[m, o] W_in[col0 + c, o]
 * dZ_in is the gradient at the input projection's pre-activation, i.e. the ReLU gate of
 * relu(X W_in + b_in) taken before the GaussianNoise.  It is what the preceding tfr_din_bwd
 * (same X, list_mask, B, N, cfg, params, workspace) left in the workspace.  One GEMM (K = h;
 * 3xTF32, or TF32 under TFR_PREC_TF32) in column chunks of at most 3 H h; with accumulate = 1 each chunk goes through the
 * workspace's scratch and is then added, so the result is exactly fp32(dX + G) with G the
 * accumulate = 0 result.  Never writes dZ_in: several windows can be taken, in any order, and
 * tfr_din_bwd's gradients are the same with or without this call.  Two identical calls give
 * identical bits.  TFR_INVALID_ARGUMENT before any CUDA call for the limits above, NULL
 * params / workspace / dX, a window outside [0, D), ldx < ncols or accumulate not 0 / 1;
 * B * N == 0 is a no-op. */
int tfr_din_input_grad(const tfr_din_cfg* cfg, int B, int N, const float* params,
                       void* workspace, int col0, int ncols, float* dX, int ldx,
                       int accumulate, void* stream);

/* ---------------------------------------------------------------------------
 * K13  DASALC scorer (research/dasalc.py:116-201): a latent-cross tower over the transformed
 * features X [M, D] and the DocumentInteractionAttention embedding E [M, h] (row pitch lde),
 * M = B * N flattened items, W = hidden_dim.  All BN layers are the non-fused tf.keras
 * BatchNormalization: population variance, moving = moving * momentum + batch * (1 - momentum)
 * in training, the moving statistics in inference.
 *   a0  = BN_in(X) + sigma g                       (GaussianNoise, training only)
 *   a_l = Dropout(BN_l(relu(a_{l-1} W_l + b_l)))   l = 1, 2 (exactly two hidden layers)
 *   t   = a_2 W_t + b_t,   c = BN_c(E) W_c + b_c
 *   s   = Dropout(relu(t * c + t)) w_o + b_o,      ln(1e-10) where mask (uint8 [M]) is 0
 * Flat parameter layout: W_1 [D, W] (Keras kernel layout), b_1 [W], W_2 [W, W], b_2, W_t [W, W],
 *   b_t, W_c [h, W], b_c, w_o [W], b_o [1], then gamma, beta of BN_in [D], BN_1 [W], BN_2 [W],
 *   BN_c [h].  Gradients use the same layout.
 * bn_state (device, tfr_dasalc_bn_state_count floats): moving mean then moving variance of
 *   BN_in, BN_1, BN_2, BN_c in that order.
 * Random draws (training only), with u(s, e) the tower's counter hash (tfr_mlp_cfg dropout
 * mask) and site seeds s = seed * 0x100000001B3 + site:
 *   site 1, 2   dropout after BN_1, BN_2, element e = m * W + j
 *   site 3      input noise, element e = m * D + j: g = sqrt(-2 ln(1 - u(s, 2e)))
 *               * cos(2 pi u(s, 2e + 1))  (the DIN's formula)
 *   site 4      cross dropout, element e = m * W + j
 *   an element is dropped iff u < dropout; kept values are scaled by 1 / (1 - dropout).
 * precision: TFR_PREC_TF32X3 (fp32-faithful) or TFR_PREC_TF32 (TFR_UNSUPPORTED otherwise).
 * Limits (TFR_INVALID_ARGUMENT before any CUDA call): D, W, h positive multiples of 4,
 * W <= 4096, h <= 128, 0 <= dropout < 1, input_noise_stddev >= 0, bn_epsilon > 0,
 * 0 <= bn_momentum <= 1, bn_state not NULL, M * max(D, W) < 2^31.  Two identical calls give
 * identical bits (no float atomics; fixed-order partial sums).
 * ------------------------------------------------------------------------- */
typedef struct {
  int32_t input_dim;            /* D */
  int32_t hidden_dim;           /* W */
  int32_t context_dim;          /* h, the DIN's head_size */
  float dropout;                /* rate of the three Dropout sites */
  float input_noise_stddev;     /* sigma; 0 = no GaussianNoise */
  float bn_epsilon;             /* tf.compat.v1 default 1e-3 */
  float bn_momentum;            /* `batch_norm_moment`, 0.9 in the reference recipe */
  int32_t training;             /* 1: batch statistics + moving update, noise and dropout */
  uint64_t seed;                /* vary per step; same value -> same draws */
  float* bn_state;              /* device, moving statistics (see above) */
} tfr_dasalc_cfg;

/* 0 when the configuration is out of range (tfr_last_error says why) */
size_t tfr_dasalc_param_count(const tfr_dasalc_cfg* cfg);
size_t tfr_dasalc_bn_state_count(const tfr_dasalc_cfg* cfg);
size_t tfr_dasalc_workspace_bytes(const tfr_dasalc_cfg* cfg, int M);
/* scores [M]; updates bn_state in training.  The workspace carries what tfr_dasalc_bwd needs. */
int tfr_dasalc_fwd(const float* X, const float* E, int lde, int M, const tfr_dasalc_cfg* cfg,
                   const float* params, const uint8_t* mask, void* workspace, float* scores,
                   int precision, void* stream);
/* dscores [M] -> grads (flat, parameter layout) and dE [M, h] (row pitch ldde) = dL/dE, the
 * input of tfr_din_bwd.  No gradient is formed for X.  Must follow a tfr_dasalc_fwd with the
 * same X, M, cfg, params, mask and workspace. */
int tfr_dasalc_bwd(const float* X, int M, const tfr_dasalc_cfg* cfg, const float* params,
                   const float* dscores, const uint8_t* mask, void* workspace, float* grads,
                   float* dE, int ldde, int precision, void* stream);
/* Multi-task DASALC: the same scorer with T = num_tasks output units, one per ranking task.
 * The parameter layout is tfr_dasalc_param_count's up to b_c, then w_o [W, T] (Keras kernel
 * layout) and b_o [T], then the BN gamma / beta as above; with T = 1 it is exactly that layout.
 *   score_planes [T, M]: score_planes[o * M + m] = Dropout(relu(t * c + t))[m] w_o[:, o] + b_o[o],
 *   so plane o is task o's [B, N] score matrix; masked rows are ln(1e-10) on every plane.
 * The random draws and the moving-statistics update are tfr_dasalc_fwd's (they do not depend
 * on T).  The backward takes dscore_planes [T, M] and task_weights_host (T host floats, NULL =
 * all 1) and forms the gradients of sum_o w_o L_o: the cross backward consumes the combined
 * signal sum_o w_o ds_o[m] w_o[:, o], rows the mask clears contribute 0 for every task, and
 * dw_o / db_o are reduced in a fixed order (two identical calls give identical bits).
 * Limits: tfr_dasalc_fwd's, plus 1 <= num_tasks <= 8, precision TFR_PREC_TF32X3 or
 * TFR_PREC_TF32, every weight finite and score_planes / dscore_planes / grads not NULL
 * (TFR_INVALID_ARGUMENT before any CUDA call; the size queries return 0).
 * With T = 1 and weight 1 the scores, grads, dE and bn_state are tfr_dasalc_fwd / _bwd's bits.
 * The workspace is tfr_dasalc_workspace_bytes_tasks(cfg, M, T). */
size_t tfr_dasalc_param_count_tasks(const tfr_dasalc_cfg* cfg, int num_tasks);
size_t tfr_dasalc_workspace_bytes_tasks(const tfr_dasalc_cfg* cfg, int M, int num_tasks);
int tfr_dasalc_fwd_tasks(const float* X, const float* E, int lde, int M,
                         const tfr_dasalc_cfg* cfg, const float* params, const uint8_t* mask,
                         void* workspace, float* score_planes, int num_tasks, int precision,
                         void* stream);
int tfr_dasalc_bwd_tasks(const float* X, int M, const tfr_dasalc_cfg* cfg, const float* params,
                         const float* dscore_planes, const float* task_weights_host,
                         const uint8_t* mask, void* workspace, float* grads, float* dE, int ldde,
                         int num_tasks, int precision, void* stream);
/* DASALC's feature transform (research/dasalc.py:127-129), elementwise over n floats:
 *   out = clip(sign(x) log1p(|x|), -cutoff, cutoff),  cutoff > 0; out may alias X. */
int tfr_symmetric_log1p_clip(const float* X, size_t n, float cutoff, float* out, void* stream);

/* ---------------------------------------------------------------------------
 * K15  TFR-BERT (extension/premade/tfrbert_task.py TFRBertScorer over tf-models-official's
 * BertEncoder).  tf-models is not part of the reference, so the formulas below are the
 * contract.  S sequences (the items of the lists, flattened) of L tokens each: ids
 * w[s, t] in [0, V), token mask tau[s, t] in {0, 1} (uint8) and type ids k[s, t] in [0, T_v),
 * int32 / uint8 [S, L] row-major.  E = hidden_size, H heads of dh = E / H, I = intermediate.
 *   x0[s, t] = dropout_h(LN_e(Word[w] + Pos[t] + Type[k]))
 *   per layer (post-LN):
 *     [q | k | v] = x Wqkv + bqkv                        heads contiguous in each block, as the
 *                                                        DIN's
 *     P   = softmax_j(q_i . k_j / sqrt(dh) - 1e9 (1 - tau_j))   (the DIN's rule: a sequence with
 *           no valid token attends 1/L to every token)
 *     o   = dropout_a(P) v,  y = o Wo + bo,  x' = LN_1(dropout_h(y) + x)
 *     u   = x' W1 + b1,  a = gelu(u) = 0.5 u (1 + tanh(sqrt(2/pi) (u + 0.044715 u^3)))
 *     x'' = LN_2(dropout_h(a W2 + b2) + x')
 *   pooled[s] = tanh(x_L[s, 0] Wp + bp)                  ([CLS] row)
 *   score[s]  = dropout_s(pooled[s]) . w_s + b_s          (TFRBertScorer: Dropout + Dense(1))
 * Every LayerNorm: (z - mean) / sqrt(var + 1e-12) * gamma + beta, population variance.
 * Flat parameter layout (floats, in this order; gradients use the same):
 *   word [V, E], position [max_position, E], type [T_v, E], gamma_e [E], beta_e [E],
 *   per layer: Wqkv [E, 3E] (columns: q, then k, then v), bqkv [3E], Wo [E, E], bo [E],
 *              gamma_1 [E], beta_1 [E], W1 [E, I], b1 [I], W2 [I, E], b2 [E], gamma_2 [E],
 *              beta_2 [E],
 *   Wp [E, E], bp [E], w_s [E], b_s [1].
 *   Kernels are [in, out] row-major (Keras Dense kernels).
 * Random draws (training only), with u(s, e) the tower's counter hash (see K11) and site seeds
 * s = seed * 0x100000001B3 + site; an element is dropped iff u < rate, kept values are scaled
 * by 1 / (1 - rate):
 *   site 1           dropout_h of the embedding output, element e = m * E + c (m = s L + t)
 *   site 2 + 3 l     dropout_a of layer l, e = ((s H + head) L + i) L + j
 *   site 3 + 3 l     dropout_h of layer l's attention output y, e = m * E + c
 *   site 4 + 3 l     dropout_h of layer l's FFN output, e = m * E + c
 *   site 2 + 3 NL    dropout_s of the pooled vector, e = s * E + c
 * Out-of-range ids (w outside [0, V), k outside [0, T_v)) add no row in the forward, get no
 * gradient, and are counted into *bad_ids (an int device counter, optional) by the forward.
 * Precision (tfr_bert_cfg.precision): TFR_PREC_FP32 (0, a zeroed struct) runs every GEMM in
 * 3xTF32 and the attention core in FP32 CUDA-core FMA; TFR_PREC_TF32 runs the GEMMs in one
 * TF32 pass and the attention core on wgmma TF32 (as tfr_din_cfg).  LayerNorm, GELU, softmax,
 * masking, dropout and the head are fp32 in both.
 * TFR_PREC_BF16 (mixed precision, Keras' 'mixed_bfloat16' policy): parameters, optimizer state
 * and gradients stay fp32 in the same flat layout (a checkpoint does not depend on precision);
 * the layers compute on bf16 values, rounded to nearest even at these points only:
 *   GEMM operands     bf16 shadows of Wqkv, Wo, W1, W2, Wp, refreshed from params by every
 *                     forward (the backward reuses them); the activations x_l, o, x', a and
 *                     the [CLS] rows; the backward signals dy, du, dqkv, dpre
 *   GEMM outputs      fp32 accumulation plus the fp32 bias, then rounded: qkv, y = o Wo + bo,
 *                     u, y2 = a W2 + b2, pre = x_L[CLS] Wp + bp, and every input-side
 *                     gradient (dO = dy Wo^T, da = dy W2^T, d x' = du W1^T, dx = dqkv Wqkv^T,
 *                     dCLS = dpre Wp^T)
 *   elementwise       computed in fp32, stored rounded: the LayerNorm outputs x_0, x', x''
 *                     and a = gelu(u); du = bf16(da gelu'(u)); dy = bf16(LN backward's dz,
 *                     dropout applied); dpre = bf16(head backward)
 *   attention         S = q k^T (fp32 accumulation) times 1 / sqrt(dh), masking, softmax
 *                     and dropout in fp32; P~ = bf16(dropout(P)) with P normalised;
 *                     o = bf16(P~ v).  Backward: dP = dO v^T in fp32, D_i = dO_i . o_i over
 *                     the stored bf16 values, dS = bf16(P (dP keep - D_i)) (the gradient of
 *                     the scaled logits), dq = bf16((dS k) / sqrt(dh)),
 *                     dk = bf16((dS^T q) / sqrt(dh)), dv = bf16(P~^T dO)
 * and stay fp32: the embedding tables and their gather, LayerNorm statistics and arithmetic
 * (xhat, rstd), the residual gradient, dgamma / dbeta, the dW partials and their fixed-order
 * reduction, the bias gradients (fp32 column sums of the bf16 dy / du / dqkv / dpre), the
 * embedding LayerNorm's gradient, the pooler tanh, the score head and the scores.  Dropout
 * draws are those of the other modes.  Extra limits: E, I and dh multiples of 8.
 * TFR_PREC_FP16 (mixed precision, Keras' 'mixed_float16' policy, the one the reference's recipe
 * names for GPUs): TFR_PREC_BF16's contract word for word with IEEE binary16 (fp16: 11
 * significant bits, round to nearest even, subnormals kept) in place of bf16 at every rounding
 * point above; the same fp32 values, dropout draws and extra limits.  Out of range: a value
 * whose magnitude rounds past 65504 is stored as +-inf, and every kernel passes inf and NaN on
 * as IEEE arithmetic gives them (nothing is clamped), so an overflow anywhere in the backward
 * reaches the gradient as inf or NaN.  Dynamic loss scaling (below, after AdamW) relies on
 * that.
 * Loss scaling: tfr_bert_bwd is linear in dscores in every mode.  A caller that passes
 * S * dscores (tfr_loss_scale_mul) gets every backward signal, and the fp32 gradient, scaled
 * by S: that is the whole interface between the encoder and the loss scale.  In fp16 it lifts
 * small backward signals out of fp16's subnormal range (below 2^-14, and 0 below 2^-25).
 * Limits (TFR_INVALID_ARGUMENT before any CUDA call, and 0 from the size queries): dh = E / H
 * a multiple of 4 in [4, 128], E <= 1024, I a multiple of 4 in [4, 4096], 1 <= layers <= 24,
 * 1 <= L <= max_position <= 512, 1 <= T_v <= 16, 1 <= V < 2^30, dropout rates in [0, 1),
 * S >= 0, S * L * max(I, 3E) < 2^31; NULL ids / mask / type ids / params / workspace / scores
 * (and dscores / grads in the backward).  Deterministic: no float atomics, so two identical
 * calls give identical bits.
 * ------------------------------------------------------------------------- */
#define TFR_BERT_MAX_LAYERS 24
#define TFR_BERT_MAX_HIDDEN 1024
#define TFR_BERT_MAX_INTERMEDIATE 4096
#define TFR_BERT_MAX_POSITION 512
#define TFR_BERT_MAX_TYPES 16

typedef struct {
  int32_t vocab_size;           /* V */
  int32_t hidden_size;          /* E */
  int32_t num_heads;            /* H */
  int32_t intermediate_size;    /* I */
  int32_t num_layers;
  int32_t max_position;         /* rows of the position table */
  int32_t type_vocab_size;      /* T_v */
  float hidden_dropout;         /* dropout_h */
  float attention_dropout;      /* dropout_a */
  float output_dropout;         /* dropout_s (TFRBertScorer's bert_output_dropout) */
  int32_t training;             /* 1: dropout active; 0: inference */
  uint64_t seed;                /* vary per step; same value -> same draws */
  int32_t precision;            /* TFR_PREC_FP32 (default), TFR_PREC_TF32, TFR_PREC_BF16 or
                                   TFR_PREC_FP16 */
} tfr_bert_cfg;

size_t tfr_bert_param_count(const tfr_bert_cfg* cfg);
size_t tfr_bert_workspace_bytes(const tfr_bert_cfg* cfg, int S, int L);
/* scores [S].  The workspace keeps what tfr_bert_bwd needs. */
int tfr_bert_fwd(const int32_t* word_ids, const uint8_t* input_mask, const int32_t* type_ids,
                 int S, int L, const tfr_bert_cfg* cfg, const float* params, void* workspace,
                 float* scores, int* bad_ids, void* stream);
/* dscores [S] -> grads (flat, parameter layout; every element written).  Must follow a
 * tfr_bert_fwd with the same inputs, cfg, params and workspace. */
int tfr_bert_bwd(const int32_t* word_ids, const uint8_t* input_mask, const int32_t* type_ids,
                 int S, int L, const tfr_bert_cfg* cfg, const float* params,
                 const float* dscores, void* workspace, float* grads, void* stream);

/* ---------------------------------------------------------------------------
 * K12  pooled embedding bags (tf.feature_column.embedding_column over a categorical column;
 * Keras Embedding + a reduction over the token axis).  ids [R, T] int32, table [V, E] fp32.
 * Bag r holds the ids ids[r, 0..T) in [0, V); -1 marks an empty slot.  Any other id (< -1 or
 * >= V) is never read: it is skipped like -1 and counted into *bad_ids (an int device counter,
 * optional).  With c_r the number of ids in [0, V) of bag r:
 *   pooled_r = scale_r * sum_t table[ids[r, t]],  scale_r = 1 (SUM), 1 / c_r (MEAN),
 *              1 / sqrt(c_r) (SQRTN); a bag with c_r = 0 pools to zeros
 * A repeated id counts once per occurrence.
 *   tfr_embedding_fwd  writes pooled_r into rows r * rows_per_bag .. + rows_per_bag - 1 of
 *                      out (row pitch ldo >= E): a context bag repeated over its list
 *                      (rows_per_bag = list_size), or one bag per row (rows_per_bag = 1); a
 *                      column block of a wider buffer such as the tower's input.
 *   tfr_embedding_bwd  dout rows with the same layout (pitch lddo) ->
 *                      dtable[v] (=, or += when accumulate) sum over occurrences (r, t) of v
 *                      of scale_r * sum_k dout[r * rows_per_bag + k].  Rows no id hit are
 *                      written 0 (or left as they are with accumulate).  Deterministic: a
 *                      stable radix sort of the occurrences by id, then fixed-order segment
 *                      sums split into chunks of 128 occurrences; no float atomics, so two
 *                      identical calls give identical bits.
 * Limits: R * T < 2^31, V < 2^30, 1 <= E <= 1024.  workspace: tfr_embedding_workspace_bytes.
 * ------------------------------------------------------------------------- */
typedef enum {
  TFR_COMBINER_SUM = 0,
  TFR_COMBINER_MEAN = 1,
  TFR_COMBINER_SQRTN = 2
} tfr_combiner;

size_t tfr_embedding_workspace_bytes(int R, int T, int V, int E);
int tfr_embedding_fwd(const int32_t* ids, int R, int T, const float* table, int V, int E,
                      int combiner, int rows_per_bag, float* out, int ldo, int* bad_ids,
                      void* stream);
int tfr_embedding_bwd(const int32_t* ids, int R, int T, const float* dout, int lddo,
                      int rows_per_bag, int V, int E, int combiner, int accumulate,
                      void* workspace, float* dtable, int* bad_ids, void* stream);

/* ---------------------------------------------------------------------------
 * K14  Bilinear (keras/layers.py:807-890), the interaction layer of two-tower models for
 * unbiased learning to rank.  v1, v2 [M, E] fp32 row-major; for every row m
 *   y[m, k] = sum_ij v1[m, i] W[i, j, k] v2[m, j] + sum_i v1[m, i] W1[i, k]
 *             + sum_j v2[m, j] W2[j, k] + b[k]                              y [M, K]
 * Flat parameter layout (Keras get_weights() order): W `bilinear_term` [E, E, K] row-major,
 * W1 `linear_term_1` [E, K], W2 `linear_term_2` [E, K], b `const_term` [K];
 * tfr_bilinear_param_count(E, K) = E*E*K + 2*E*K + K floats.  Gradients use the same layout.
 * row_mask (uint8 [M], optional): a row whose byte is 0 gets RestoreList's ln(1e-10) in every
 * output; in the backward it contributes nothing to the parameter gradients and gets
 * dv1 = dv2 = 0.
 * The backward writes dv1, dv2 [M, E] and the six parameter gradients (=, not +=) in one pass
 * over the rows: fixed-order per-CTA partials in the workspace (tfr_bilinear_workspace_bytes),
 * then a fixed-order sum over the CTAs.  No float atomics: two identical calls give identical
 * bits.  FP32 on CUDA cores (no TF32).
 * Limits (TFR_INVALID_ARGUMENT before any CUDA call, and 0 from the size queries):
 * M >= 1, 1 <= E <= 128, 1 <= K <= 32, E * E * K <= 16384 (W and one dW partial stay in
 * shared memory); NULL v1 / v2 / params / y / dy / dv1 / dv2 / grads / workspace.
 * ------------------------------------------------------------------------- */
size_t tfr_bilinear_param_count(int E, int K);
size_t tfr_bilinear_workspace_bytes(int M, int E, int K);
int tfr_bilinear_fwd(const float* v1, const float* v2, int M, int E, int K, const float* params,
                     const uint8_t* row_mask, float* y, void* stream);
int tfr_bilinear_bwd(const float* v1, const float* v2, int M, int E, int K, const float* params,
                     const uint8_t* row_mask, const float* dy, float* dv1, float* dv2,
                     float* grads, void* workspace, void* stream);

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
/* The same engine on fp16 operands (TFR-BERT's TFR_PREC_FP16): every argument and layout as
 * tfr_tc_gemm_bf16, with fp16 in place of bf16 (a 16-bit C is fp16, rounded to nearest even;
 * magnitudes past 65504 are stored as inf). */
int tfr_tc_gemm_f16(const void* A, int lda, const void* B, int ldb, void* C, int ldc,
                    int GM, int GN, int GK, int mn, int epi, const float* bias, int act,
                    uint32_t* mask_bits_out, const uint32_t* mask_bits_in,
                    float* colsum, int colsum_stride, int* colsum_slots_out,
                    int splits, size_t split_stride, void* stream);

/* Parity helpers for TFR-BERT's bf16 attention core (csrc/din_bf16.cu; the rounding points
 * are K15's TFR_PREC_BF16 "attention" row).  Layouts as the DIN's attention core (K11):
 * qkv bf16 [B N, 3 H h] (q, k, v blocks of H heads of h columns), lmask uint8 [B N] (0 = key
 * masked with the -1e9 adder; NULL = all valid), O bf16 [B N, H h], lse fp32 [B N, H, 2] =
 * {row max, 1 / sum} (exact for a list with no valid item: 1 / sum = float(1 / N)),
 * dsum fp32 [B N, H] = dO . O over the stored bf16 values, dO bf16 [B N, H h], dqkv bf16
 * [B N, 3 H h].  Dropout of P with rate `drop` keeps element ((b H + head) N + i) N + j iff
 * u(dseed, e) >= drop, with dseed the combined site seed (seed * 0x100000001B3 + site).
 * Limits (TFR_INVALID_ARGUMENT before any CUDA call): NULL qkv / O / lse (and dO / dsum /
 * dqkv), h a multiple of 8 in [8, 128], 1 <= N <= TFR_DIN_MAX_LIST, H >= 1,
 * H h <= TFR_BERT_MAX_HIDDEN, drop in [0, 1), every buffer but lmask 16-byte aligned.
 * B = 0 launches nothing. */
int tfr_attn_bf16_fwd(const void* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                      float drop, unsigned long long dseed, void* O, float* lse, void* stream);
int tfr_attn_bf16_bwd(const void* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                      float drop, unsigned long long dseed, const void* O, const float* lse,
                      const void* dO, float* dsum, void* dqkv, void* stream);
/* The same core on fp16 (K15's TFR_PREC_FP16): arguments, layouts, limits and rounding points
 * as tfr_attn_bf16_*, with fp16 in place of bf16. */
int tfr_attn_f16_fwd(const void* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                     float drop, unsigned long long dseed, void* O, float* lse, void* stream);
int tfr_attn_f16_bwd(const void* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                     float drop, unsigned long long dseed, const void* O, const float* lse,
                     const void* dO, float* dsum, void* dqkv, void* stream);

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

/* Token features: bytes_list features mapped to ids through a vocabulary, as
 * tf.feature_column.categorical_column_with_vocabulary_file / _list do.
 *   tfr_vocab_create   tokens[i] (token_sizes[i] bytes) gets id i; a duplicate token is
 *                      TFR_INVALID_ARGUMENT.  num_oov_buckets 0: an unknown token is id -1
 *                      (ignored downstream); 1: it is id n (the table has n + 1 rows).  More
 *                      buckets (Fingerprint64 hashing) are TFR_INVALID_ARGUMENT.  The object
 *                      is a host object, read-only after creation (safe to share between
 *                      threads); free it with tfr_vocab_destroy.
 *   tfr_vocab_lookup   ids_out[i] = id of tokens[i]
 *   tfr_ranking_parse_tokens
 *                      tfr_ranking_parse plus token features: context token feature k writes
 *                      context_ids_out[k] [B, T_k], example token feature k writes
 *                      example_ids_out[k] [B, list_size, T_k] (HOST arrays of HOST pointers,
 *                      T_k = max_tokens).  A bag keeps its first T_k tokens, in record order;
 *                      the other slots hold -1, as do missing features and padded items.
 *                      dropped_out (optional, HOST int64 [n_context_tokens +
 *                      n_example_tokens], context features first) receives the number of
 *                      tokens cut by the T_k limit.  A token feature with float / int64 values
 *                      is TFR_UNSUPPORTED. */
typedef struct {
  const char* name;
  int32_t max_tokens;   /* T >= 1 */
  const void* vocab;    /* from tfr_vocab_create */
} tfr_token_spec;

int tfr_vocab_create(const char* const* tokens, const int64_t* token_sizes, int n,
                     int num_oov_buckets, void** vocab_out);
int tfr_vocab_destroy(void* vocab);
int tfr_vocab_lookup(const void* vocab, const char* const* tokens, const int64_t* token_sizes,
                     int n, int32_t* ids_out);
int tfr_ranking_parse_tokens(int format, const uint8_t* const* records,
                             const int64_t* record_sizes, int B, int list_size,
                             const tfr_feature_spec* context_spec, int n_context,
                             const tfr_feature_spec* example_spec, int n_example,
                             const tfr_token_spec* context_tokens, int n_context_tokens,
                             const tfr_token_spec* example_tokens, int n_example_tokens,
                             float* context_out, float* example_out,
                             int32_t* const* context_ids_out, int32_t* const* example_ids_out,
                             int64_t* dropped_out, int32_t* sizes_out, uint8_t* mask_out,
                             int n_threads);

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

/* AdamW, the update of tf-models-official's AdamWeightDecay (BERT's optimizer), over n floats
 * with m and v the first and second moments (zero before step 1), t = step >= 1:
 *   g *= grad_scale;  m = beta1 m + (1 - beta1) g;  v = beta2 v + (1 - beta2) g^2
 *   p -= lr * weight_decay * p                        (elements whose decay_mask byte is
 *                                                      nonzero; NULL: every element)
 *   p -= lr * sqrt(1 - beta2^t) / (1 - beta1^t) * m / (sqrt(v) + eps)   (Keras Adam form)
 * The step factor is formed on the host in double.  TFR_INVALID_ARGUMENT for NULL params /
 * grads / m / v, step < 1, or beta1 / beta2 outside [0, 1). */
int tfr_adamw_step(float* params, const float* grads, float* m, float* v,
                   const uint8_t* decay_mask, size_t n, float lr, float beta1, float beta2,
                   float eps, float weight_decay, int64_t step, float grad_scale, void* stream);

/* Global-norm gradient clipping, as tf-models' AdamWeightDecay applies it before the update
 * (gradient_clip_norm, 1.0 in BERT's fine-tuning recipe; tf.clip_by_global_norm).
 *
 * tfr_global_norm writes ||x||_2 = sqrt(sum_i x_i^2) of n floats to *norm_out (device).  The
 * squares are summed in double in a fixed order: per-block partials over fixed grid-stride
 * positions (of float4s when x is 16-byte aligned), then one ordered final sum, so two
 * identical calls give identical bits.  inf or NaN inputs give an inf or NaN norm; so does,
 * once rounded to float, a finite norm above FLT_MAX (~3.4e38).  The workspace (device, >= the bytes
 * tfr_global_norm_workspace_bytes(n) returns, 8 per block) holds the partials; n = 0 writes
 * 0.  No host synchronisation.  TFR_INVALID_ARGUMENT for NULL norm_out / workspace, NULL x
 * with n > 0, or a short workspace.
 *
 * tfr_adamw_step_clipped is tfr_adamw_step with every gradient multiplied, after grad_scale,
 * by s read from `norm` (device, the global norm of grads * grad_scale):
 *   s = 1                     norm <= clip_norm   (exactly tfr_adamw_step's bits)
 *   s = clip_norm / norm      norm >  clip_norm
 *   s = NaN                   norm inf or NaN     (every clipped gradient is NaN; with
 *                                                  tfr_global_norm's norm that includes a
 *                                                  gradient whose norm exceeds FLT_MAX)
 * The weight-decay term is not scaled.  The scale is applied inside the update kernel: no
 * extra pass over the gradient and no host synchronisation.  TFR_INVALID_ARGUMENT as
 * tfr_adamw_step, and for NULL norm or clip_norm not finite and > 0. */
size_t tfr_global_norm_workspace_bytes(size_t n);
int tfr_global_norm(const float* x, size_t n, float* norm_out, void* workspace,
                    size_t workspace_bytes, void* stream);
int tfr_adamw_step_clipped(float* params, const float* grads, float* m, float* v,
                           const uint8_t* decay_mask, size_t n, float lr, float beta1,
                           float beta2, float eps, float weight_decay, int64_t step,
                           float grad_scale, float clip_norm, const float* norm, void* stream);

/* Dynamic loss scaling, the rule of Keras' LossScaleOptimizer(dynamic=True) (Keras is not part
 * of the reference, so this is the contract).  State: the scale S (float, device; initial 2^15)
 * and a good-step counter c (int64, device; initial 0); growth_steps (Keras'
 * dynamic_growth_steps) 2000 by default.  One step, with g_s = the gradient of S * loss
 * (tfr_loss_scale_mul on dscores, then the backward) and N = tfr_global_norm(g_s):
 *   N finite       g = g_s * (1 / S)  (Keras' unscale); with clipping, the factor of
 *                  tfr_adamw_step_clipped on the unscaled norm N_u = float((double) N / S);
 *                  then the AdamW update of tfr_adamw_step.  c += 1; when c reaches
 *                  growth_steps, S = 2 S (kept only if finite) and c = 0
 *   N inf or NaN   (any inf or NaN element; also a finite gradient whose norm exceeds FLT_MAX,
 *                  which Keras would apply) params, m and v are left bit for bit as they are;
 *                  S = max(S / 2, 1), c = 0
 * The update count t (bias correction, learning-rate schedule) advances on a skipped step too:
 * Keras' skip branch increments the inner optimizer's `iterations`.  With a fixed scale S never
 * changes and c is not kept; a non-finite step is still skipped (Keras would apply it).
 * Everything runs on the device, in stream order, with no host synchronisation:
 *   tfr_loss_scale_mul     out[i] = x[i] * *scale over n floats (out may alias x)
 *   tfr_adamw_step_scaled  the update above, reading N from *norm and S from *scale; clip_norm
 *                          0 disables clipping, else it must be finite and > 0 (the
 *                          TFR_INVALID_ARGUMENT rules of tfr_adamw_step otherwise; no
 *                          grad_scale: one replica)
 *   tfr_loss_scale_update  one thread, launched after tfr_adamw_step_scaled (which must read
 *                          the old S): *unscaled_norm = float((double) N / S) (optional),
 *                          then S and c by the rule above; growth_steps 0 (a fixed scale)
 *                          leaves S and c (c may then be NULL).  TFR_INVALID_ARGUMENT for NULL
 *                          scale / norm or growth_steps < 0. */
int tfr_loss_scale_mul(const float* x, size_t n, const float* scale, float* out, void* stream);
int tfr_adamw_step_scaled(float* params, const float* grads, float* m, float* v,
                          const uint8_t* decay_mask, size_t n, float lr, float beta1,
                          float beta2, float eps, float weight_decay, int64_t step,
                          float clip_norm, const float* norm, const float* scale, void* stream);
int tfr_loss_scale_update(float* scale, int64_t* good_steps, const float* norm,
                          float* unscaled_norm, int64_t growth_steps, void* stream);

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
