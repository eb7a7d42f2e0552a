// Host-side plan of the scorer tower: parameter offsets and workspace carving.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "tfr_b200.h"

namespace tfr {

struct MlpPlan {
  int n_dense;
  int dims[TFR_MLP_MAX_LAYERS + 1];
  int activation;
  // flat parameter layout (floats)
  size_t w_off[TFR_MLP_MAX_LAYERS], b_off[TFR_MLP_MAX_LAYERS], n_params;
  // workspace layout (floats)
  size_t act_off[TFR_MLP_MAX_LAYERS];  // post-activation output of hidden layer d
  size_t bits_off[TFR_MLP_MAX_LAYERS]; // ReLU sign bits of hidden layer d: [ceil(h/32)][M] words
  size_t dz_off[2];                    // ping-pong dZ buffers
  size_t partial_off, partial_stride;  // split partials for dW / db
  int splits, rows_per_split;
  size_t whi_off, wlo_off;             // TF32 hi / lo copies of the flat parameters
  size_t wthi_off, wtlo_off;           // ... and of the per-layer transposes W^T [out, in]
                                       //   (same offsets: K-major B operand of the forward)
  // tensor-core path: per-tile column sums and the fine-grain output-layer slots
  size_t tile_off, tile_stride;        // [4 * ceil(M / 128)][tile_stride]
  int tile_slots;
  size_t oslot_off, oslot_stride;      // [ceil(M / out_rows)][oslot_stride]
  int out_rows, out_slots;
  // BatchNormalization / Dropout (create_tower options)
  int use_bn, input_bn, training;
  float bn_eps, bn_mom, dropout;
  unsigned long long seed;
  float* bn_state;                              // moving mean / variance (device)
  size_t g_off[TFR_MLP_MAX_LAYERS], be_off[TFR_MLP_MAX_LAYERS];   // gamma / beta of hidden BN d
  size_t gin_off, bein_off;                     // input BN gamma / beta
  size_t st_off[TFR_MLP_MAX_LAYERS], stin_off;  // offsets into bn_state (mean; var at +w)
  size_t n_state;
  size_t xhat_off[TFR_MLP_MAX_LAYERS];          // normalised pre-activations of hidden layer d
  size_t xin_off;                               // batch-normalised inputs
  size_t bnstat_off[TFR_MLP_MAX_LAYERS], bnstat_in_off;   // batch mean[w], rstd[w] (fwd -> bwd)
  size_t red_off, red_stride;                   // column-reduction partials [red_blocks][stride]
  int red_rows, red_blocks;
  size_t ws_floats;
  bool post() const { return use_bn || dropout > 0.f; }   // hidden layers need a post pass
};

// BatchNormalization / Dropout passes shared by both scorer paths (mlp_norm.cu).
// Forward, hidden layer d: Z (in the xhat buffer when BN) -> H (act buffer).
int mlp_hidden_post_fwd(int d, int M, const MlpPlan& p, const float* params, float* ws,
                        cudaStream_t st);
// Backward, hidden layer d: dz holds dL/dH_d on entry, dL/dZ_d on exit; writes the
// BN gamma / beta gradients.
int mlp_hidden_pre_bwd(int d, int M, const MlpPlan& p, const float* params, float* ws,
                       float* dz, float* grads, cudaStream_t st);
// Batch statistics of src [M, N] into stat (mean[N], rstd[N]) through the plan's reduction
// partials, updating the moving averages in training; the moving statistics in inference.
int mlp_bn_batch_stats(const float* src, int M, int N, const MlpPlan& p, float* ws, float* stat,
                       float* moving, cudaStream_t st);
// Input BN: X -> ws + xin_off; and its parameter gradients from dL/dXin.
int mlp_input_bn_fwd(const float* X, int M, const MlpPlan& p, const float* params, float* ws,
                     cudaStream_t st);
int mlp_input_bn_bwd(const float* X, int M, const MlpPlan& p, const float* params, float* ws,
                     const float* dxin, float* grads, cudaStream_t st);

// Loss weights of the task-major ("planar") score layout of tfr_mlp_fwd_tasks / _bwd_tasks:
// score plane o is scores[o * M + m], and the output-layer backward reads the signal
// w[o] * dscores[o * M + m], zeroed on masked rows.  Passed by value to the kernels.
struct TaskWeights {
  float w[8];
};

// Returns 0 on success and fills `p`; sets the error string otherwise.
int make_mlp_plan(const tfr_mlp_cfg* cfg, int M, MlpPlan* p);

// planar / tw: the task-major layout (TaskWeights); the defaults are tfr_mlp_fwd / _bwd's.
int mlp_simt_fwd(const float* X, int M, const MlpPlan& p, const float* params,
                 const uint8_t* mask, float* ws, float* scores, cudaStream_t st,
                 bool planar = false);
int mlp_simt_bwd(const float* X, int M, const MlpPlan& p, const float* params,
                 const float* dscores, const uint8_t* mask, float* ws, float* grads,
                 cudaStream_t st, const TaskWeights* tw = nullptr);

// tensor-core (wgmma) path; passes = 1 (TF32) or 3 (3xTF32, fp32-faithful)
int mlp_tc_fwd(const float* X, int M, const MlpPlan& p, const float* params,
               const uint8_t* mask, float* ws, float* scores, int passes, cudaStream_t st,
               bool planar = false);
int mlp_tc_bwd(const float* X, int M, const MlpPlan& p, const float* params,
               const float* dscores, const uint8_t* mask, float* ws, float* grads,
               int passes, cudaStream_t st, const TaskWeights* tw = nullptr);

// bf16 tensor-core path (wgmma bf16): X and all activations are bf16 in HBM
int mlp_bf16_fwd(const void* X, int M, const MlpPlan& p, const float* params,
                 const uint8_t* mask, float* ws, float* scores, cudaStream_t st);
int mlp_bf16_bwd(const void* X, int M, const MlpPlan& p, const float* params,
                 const float* dscores, const uint8_t* mask, float* ws, float* grads,
                 cudaStream_t st);

// partial walks of the tensor-core path (the groupwise fold supplies / consumes layer 0)
struct MlpBwdTail {
  float* dz;               // dL/dZ of Dense stop_layer - 1, [M, dims[stop_layer]]
  float* dz_other;         // the other ping-pong buffer (free)
  const float* bias_src;   // per-slot column sums of dz
  int bias_slots;
  size_t bias_stride;
};
int mlp_tc_split_params(const MlpPlan& p, const float* params, float* ws, int passes,
                        cudaStream_t st);
int mlp_tc_fwd_from(int first_layer, const float* X, int M, const MlpPlan& p,
                    const float* params, const uint8_t* mask, float* ws, float* scores,
                    int passes, cudaStream_t st, bool planar = false);
int mlp_tc_bwd_until(int stop_layer, MlpBwdTail* tail, const float* X, int M, const MlpPlan& p,
                     const float* params, const float* dscores, const uint8_t* mask,
                     float* ws, float* grads, int passes, cudaStream_t st,
                     const TaskWeights* tw = nullptr);
// Tower input gradient for columns [col0, col0 + ncols) after mlp_tc_bwd (no input BN,
// at least one hidden layer): tfr_mlp_input_grad.  After a backward that took the fused dW_0
// kernel (mlp_tc_fused_bwd_ok) it first recomputes dZ_0 into the workspace's dZ_0 region;
// nothing mlp_tc_bwd returns depends on that region.
int mlp_tc_input_grad(int M, const MlpPlan& p, const float* params, float* ws, int col0,
                      int ncols, float* dX, int ldx, int passes, cudaStream_t st);
// The three roles of Dense d's GEMMs on the TF32 engine.  Apart from the split kernel and
// the fused forward, only these know where the weight operand lives for `passes` (the
// forward and dgrad read the split parameters mlp_tc_split_params wrote for passes = 3).
// Forward: C[M, dims[d+1]] = A[M, kc] W_d[k0 : k0 + kc, :].  With a bias: bias, then `act`,
// and ReLU sign words into `bits` when it is given; without: a plain store.
int mlp_tc_dense_fwd(const MlpPlan& p, int d, int k0, int kc, const float* A, int M,
                     const float* params, const float* ws, const float* bias, int act,
                     uint32_t* bits, float* C, int passes, cudaStream_t st);
// Input side: C[M, nc] (ldc) = dZ_d[M, dims[d+1]] W_d[n0 : n0 + nc, :]^T, zeroed where the
// sign word bit is clear when `mask_bits` is given; per-CTA column sums into `colsum` when
// given (row pitch colsum_stride, slot count into *colsum_slots).
int mlp_tc_dense_dgrad(const MlpPlan& p, int d, int n0, int nc, const float* dZ, int M,
                       const float* params, const float* ws, const uint32_t* mask_bits,
                       float* colsum, size_t colsum_stride, int* colsum_slots, float* C, int ldc,
                       int passes, cudaStream_t st);
// Weight gradient: out[0 : Kin Nout) = A^T dZ for A [M, Kin] (lda), dZ [M, Nout] (ldz), then
// out[Kin Nout : + Nout) = the sums of bias_slots rows of bias_src (pitch bias_stride); no
// bias part when bias_src is null.  Split-K over `splits` row ranges into `partial` (pitch
// pstride), reduced in fixed order.  Takes the orientation with fewer tile units unless
// `direct`.
int mlp_tc_weight_grad(const float* A, int lda, int Kin, const float* dZ, int ldz, int Nout,
                       int M, int splits, float* partial, size_t pstride, const float* bias_src,
                       int bias_slots, size_t bias_stride, bool direct, float* out, int passes,
                       cudaStream_t st);
// Fused 3xTF32 forward of Dense first_layer .. L (mlp_tc_fused.cu): one persistent kernel,
// bit-identical to the per-layer walk.  _ok says whether the tower fits it: no BN / dropout /
// input BN, ReLU or no activation, Dense first_layer at most 256 wide, every later hidden
// layer at most 128, at most 8 output units, at least one hidden layer, X and the workspace
// 16-byte aligned (its operands move by TMA).  Expects the parameters already split.
bool mlp_tc_fused_fwd_ok(int first_layer, const float* X, int M, const MlpPlan& p, int passes,
                         const float* ws);
int mlp_tc_fused_fwd(int first_layer, const float* X, int M, const MlpPlan& p,
                     const float* params, const uint8_t* mask, float* ws, float* scores,
                     cudaStream_t st, bool planar = false);
// Fused 3xTF32 backward of Dense 0 (mlp_tc_fused_bwd.cu): from dZ_1, dZ_0 = (dZ_1 W_1^T) *
// relu'(H_0) and dW_0 in one kernel, into dW_0's split-K partial slots (ws + partial_off) and
// one db_0 column-sum slot per split (ws + tile_off), for mlp_reduce2; dZ_0 is not stored.
// dW_0 is bit-identical to mlp_tc_dense_dgrad(d = 1) then mlp_tc_weight_grad(d = 0).  _ok
// says whether mlp_tc_bwd takes it: 3xTF32, no BN / dropout / input BN, ReLU or no
// activation, at least two hidden layers, dims[0] <= 136 in dW_0's swapped orientation,
// dims[1] and dims[2] <= 256, a 16-byte aligned workspace.  Expects the parameters split.
bool mlp_tc_fused_bwd_ok(const MlpPlan& p, int passes, const float* ws);
int mlp_tc_fused_dw0(const float* X, const float* dz1, int M, const MlpPlan& p, float* ws,
                     cudaStream_t st);

// pieces of the CUDA-core path reused by the tensor-core path
int mlp_out_layer_fwd(const float* H, int M, int K, int O, const float* W, const float* bias,
                      const uint8_t* mask, float* scores, cudaStream_t st, bool planar = false);
int mlp_out_layer_bwd2(const float* H, int M, int K, int O, const float* W, const float* dS,
                       const uint8_t* mask, int act, int rows_per, float* dH, float* slots,
                       size_t slot_stride, cudaStream_t st);
// mlp_out_layer_bwd2's slots from the planar signal tw.w[o] * dS[o * M + m], zero on masked
// rows (every O).
int mlp_out_layer_bwd2_tasks(const float* H, int M, int K, int O, const float* W,
                             const float* dS, const TaskWeights& tw, const uint8_t* mask, int act,
                             int rows_per, float* dH, float* slots, size_t slot_stride,
                             cudaStream_t st);
int mlp_reduce2(const float* srcA, int slotsA, size_t strideA, size_t nA, const float* srcB,
                int slotsB, size_t strideB, size_t nB, float* out, cudaStream_t st);
int mlp_colsum(const float* dZ, int M, int N, int rows_per, int splits, float* partial,
               size_t pstride, size_t col_offset, cudaStream_t st);
int mlp_reduce_partials(const float* partial, int splits, size_t stride, size_t n, float* out,
                        cudaStream_t st);

}  // namespace tfr
