// K13 DASALC scorer (research/dasalc.py:116-201): a latent-cross tower over the transformed
// features X [M, D] and the DocumentInteractionAttention embedding E [M, h].
//
//   a0  = BN_in(X) + sigma g                                 stats + one normalising sweep
//   a_l = Dropout(BN_l(relu(a_{l-1} W_l + b_l)))   l = 1, 2   GEMM (bias + ReLU + sign words),
//                                                            then mlp_norm.cu's BN / dropout
//   t   = a_2 W_t + b_t,  c = BN_c(E) W_c + b_c               GEMMs with a bias epilogue
//   s   = Dropout(relu(t * c + t)) w_o + b_o                 cross forward (one warp per row)
//
// With T tasks (the _tasks entry points) w_o is [W, T] and b_o [T]: the cross forward dots each
// row's dropped vector with the T columns into T score planes, and the cross backward takes
// the combined signal sum_o w_o ds_o.  dw_o / db_o then come from a separate fixed-order
// reduction over the dropped vectors the cross backward stores, since T x W accumulators per
// thread would not fit in registers.  Both cross kernels are templated on T; T = 1 is the
// single-task path itself.
//
// Every Dense GEMM goes through the tower's three functions (mlp_tc_dense_fwd / _dgrad /
// mlp_tc_weight_grad) over parameters split by mlp_tc_split_params.  Two tower plans describe
// the Dense layers to them: `a` chains W_1, W_2, W_t (and names w_o as its output layer), `c`
// holds W_c alone.  Both index the one DASALC parameter buffer and share the split copies.
// The backward is the same walk in reverse: the cross backward writes dt, dc and fixed-order
// per-block partials of dw_o, db_o and the column sums of dt and dc (the bias gradients of
// b_t, b_c); BN + dropout backward is mlp_norm.cu's, followed by a ReLU gate from the sign
// words that also takes the bias column sums.  No float atomics anywhere.
#include <cmath>
#include <cstring>
#include <type_traits>

#include "common.cuh"
#include "mlp.h"

namespace tfr {
namespace {

constexpr int kMaxW = 4096;
constexpr int kMaxH = 128;
constexpr int kXQ = kMaxW / 4 / 256;   // column quads per thread in the cross backward
constexpr int kXRows = 32;             // rows per block of the cross backward
// random-draw sites (seed * 0x100000001B3 + site); hidden layer d's dropout is the tower's
// post pass, which draws from site d + 1 (sites 1 and 2)
constexpr int kSiteNoise = 3, kSiteCross = 4;
constexpr int kMaxTasks = 8;   // TaskWeights (mlp.h) holds 8

// f(std::integral_constant<int, T>) for the runtime task count 1 <= T <= kMaxTasks.
template <typename F>
void with_tasks(int T, F&& f) {
  switch (T) {
    case 1: f(std::integral_constant<int, 1>()); break;
    case 2: f(std::integral_constant<int, 2>()); break;
    case 3: f(std::integral_constant<int, 3>()); break;
    case 4: f(std::integral_constant<int, 4>()); break;
    case 5: f(std::integral_constant<int, 5>()); break;
    case 6: f(std::integral_constant<int, 6>()); break;
    case 7: f(std::integral_constant<int, 7>()); break;
    default: f(std::integral_constant<int, 8>()); break;
  }
}

size_t al64(size_t x) { return (x + 63) / 64 * 64; }

struct DasalcPlan {
  int D, W, h, M, T;
  float drop, noise;
  int training;
  unsigned long long seed;
  // parameter offsets
  size_t o_w1, o_b1, o_w2, o_b2, o_wt, o_bt, o_wc, o_bc, o_wo, o_bo;
  size_t o_gin, o_bein, o_g1, o_be1, o_g2, o_be2, o_gc, o_bec, n_params, n_state;
  MlpPlan a, c;   // the Dense layers as the tower functions see them
  // workspace (floats)
  size_t ec_off, t_off, cc_off, dt_off, dc_off, dh_off[2], da0_off, dyc_off;
  size_t xpart_off, xpart_stride, xdt_col;
  size_t r_off;   // T > 1: the dropped cross outputs [M, W] for the dw_o reduction
  int xblocks;
  size_t ws_floats;
};

int check_cfg(const tfr_dasalc_cfg* c) {
  TFR_REQUIRE(c != nullptr, "cfg must not be NULL");
  TFR_REQUIRE(c->input_dim >= 4 && c->input_dim % 4 == 0,
              "input_dim %d must be a positive multiple of 4", c->input_dim);
  TFR_REQUIRE(c->hidden_dim >= 4 && c->hidden_dim % 4 == 0 && c->hidden_dim <= kMaxW,
              "hidden_dim %d must be a multiple of 4 in [4, %d]", c->hidden_dim, kMaxW);
  TFR_REQUIRE(c->context_dim >= 4 && c->context_dim % 4 == 0 && c->context_dim <= kMaxH,
              "context_dim %d must be a multiple of 4 in [4, %d]", c->context_dim, kMaxH);
  TFR_REQUIRE(c->dropout >= 0.f && c->dropout < 1.f, "dropout %g must be in [0, 1)",
              (double)c->dropout);
  TFR_REQUIRE(c->input_noise_stddev >= 0.f, "input_noise_stddev must be >= 0");
  TFR_REQUIRE(c->bn_epsilon > 0.f, "bn_epsilon must be > 0");
  TFR_REQUIRE(c->bn_momentum >= 0.f && c->bn_momentum <= 1.f, "bn_momentum %g must be in [0, 1]",
              (double)c->bn_momentum);
  return TFR_OK;
}

// Only after check_cfg and every other argument check: the row splits ask for the SM count.
void make_plan(const tfr_dasalc_cfg* cfg, int M, int T, DasalcPlan* p) {
  std::memset(p, 0, sizeof(*p));
  const int D = cfg->input_dim, W = cfg->hidden_dim, h = cfg->context_dim;
  p->D = D; p->W = W; p->h = h; p->M = M; p->T = T;
  p->training = cfg->training != 0;
  p->drop = p->training ? cfg->dropout : 0.f;
  p->noise = p->training ? cfg->input_noise_stddev : 0.f;
  p->seed = cfg->seed;
  size_t o = 0;
  p->o_w1 = o; o += (size_t)D * W;
  p->o_b1 = o; o += W;
  p->o_w2 = o; o += (size_t)W * W;
  p->o_b2 = o; o += W;
  p->o_wt = o; o += (size_t)W * W;
  p->o_bt = o; o += W;
  p->o_wc = o; o += (size_t)h * W;
  p->o_bc = o; o += W;
  p->o_wo = o; o += (size_t)W * T;
  p->o_bo = o; o += T;
  p->o_gin = o; o += D;
  p->o_bein = o; o += D;
  p->o_g1 = o; o += W;
  p->o_be1 = o; o += W;
  p->o_g2 = o; o += W;
  p->o_be2 = o; o += W;
  p->o_gc = o; o += h;
  p->o_bec = o; o += h;
  p->n_params = o;
  p->n_state = 2 * ((size_t)D + 2 * (size_t)W + h);

  MlpPlan& a = p->a;
  a.n_dense = 4;
  const int dims[5] = {D, W, W, W, T};
  for (int i = 0; i < 5; ++i) a.dims[i] = dims[i];
  a.w_off[0] = p->o_w1; a.b_off[0] = p->o_b1;
  a.w_off[1] = p->o_w2; a.b_off[1] = p->o_b2;
  a.w_off[2] = p->o_wt; a.b_off[2] = p->o_bt;
  a.w_off[3] = p->o_wo; a.b_off[3] = p->o_bo;
  a.n_params = p->n_params;   // its split covers the whole buffer (W_c included)
  a.activation = TFR_ACT_NONE;   // the ReLU sits in the GEMM epilogue, before the BN
  a.use_bn = 1; a.input_bn = 1; a.training = p->training;
  a.bn_eps = cfg->bn_epsilon; a.bn_mom = cfg->bn_momentum;
  a.dropout = cfg->dropout;
  a.seed = cfg->seed;   // hidden layer d draws from site d + 1
  a.bn_state = cfg->bn_state;
  a.gin_off = p->o_gin; a.bein_off = p->o_bein;
  a.g_off[0] = p->o_g1; a.be_off[0] = p->o_be1;
  a.g_off[1] = p->o_g2; a.be_off[1] = p->o_be2;
  a.stin_off = 0;
  a.st_off[0] = 2 * (size_t)D;
  a.st_off[1] = 2 * (size_t)D + 2 * (size_t)W;
  a.n_state = p->n_state;

  const size_t Mz = (size_t)M;
  size_t w = 0;
  for (int d = 0; d < 2; ++d) {
    a.act_off[d] = w; w += al64(Mz * W);
    a.xhat_off[d] = w; w += al64(Mz * W);
    a.bits_off[d] = w; w += al64(Mz * ((W + 31) / 32));
    a.bnstat_off[d] = w; w += al64(2 * (size_t)W);
  }
  a.xin_off = w; w += al64(Mz * D);
  a.bnstat_in_off = w; w += al64(2 * (size_t)D);
  const int max_bn = D > W ? (D > h ? D : h) : (W > h ? W : h);
  a.red_rows = 256;
  a.red_blocks = M > 0 ? (M + a.red_rows - 1) / a.red_rows : 1;
  a.red_stride = al64(2 * (size_t)max_bn);
  a.red_off = w; w += (size_t)a.red_blocks * a.red_stride + al64(2 * (size_t)max_bn);
  // dW row splits: the tower's rule (about one per SM), capped so that the split-K partials
  // stay within 64 M floats at wide W.
  const int kmax = D > W ? D : W;
  const size_t per_split = (size_t)((kmax + 127) / 128 * 128) * ((W + 127) / 128 * 128);
  {
    const int sms = num_sms();
    const int per = (M + sms - 1) / sms;
    a.rows_per_split = per < 256 ? 256 : ((per + 127) / 128) * 128;
    int max_splits = (int)((size_t)(64 << 20) / per_split);
    if (max_splits < 1) max_splits = 1;
    if (M > 0 && (M + a.rows_per_split - 1) / a.rows_per_split > max_splits) {
      const int r = (M + max_splits - 1) / max_splits;
      a.rows_per_split = (r + 127) / 128 * 128;
    }
    a.splits = M > 0 ? (M + a.rows_per_split - 1) / a.rows_per_split : 1;
  }
  a.partial_stride = al64(per_split);
  a.partial_off = w; w += (size_t)a.splits * a.partial_stride;
  a.whi_off = w; w += al64(p->n_params);
  a.wlo_off = w; w += al64(p->n_params);
  a.wthi_off = w; w += al64(p->n_params);
  a.wtlo_off = w; w += al64(p->n_params);
  a.tile_stride = al64(W);
  a.tile_off = w; w += (size_t)a.splits * a.tile_stride;

  MlpPlan& c = p->c;
  c = a;   // same BN settings, reductions, row splits and split copies
  c.n_dense = 2;
  c.dims[0] = h; c.dims[1] = W; c.dims[2] = 1;
  for (int i = 3; i <= TFR_MLP_MAX_LAYERS; ++i) c.dims[i] = 0;
  c.w_off[0] = p->o_wc; c.b_off[0] = p->o_bc;
  c.n_params = 0;   // its split only writes the transpose of W_c
  c.use_bn = 0;
  c.gin_off = p->o_gc; c.bein_off = p->o_bec;
  c.stin_off = 2 * (size_t)D + 4 * (size_t)W;
  c.xin_off = w; w += al64(Mz * h);
  c.bnstat_in_off = w; w += al64(2 * (size_t)h);

  p->ec_off = w; w += al64(Mz * h);
  p->t_off = w; w += al64(Mz * W);
  p->cc_off = w; w += al64(Mz * W);
  p->dt_off = w; w += al64(Mz * W);
  p->dc_off = w; w += al64(Mz * W);
  p->dh_off[0] = w; w += al64(Mz * W);
  p->dh_off[1] = w; w += al64(Mz * W);
  p->da0_off = w; w += al64(Mz * D);
  p->dyc_off = w; w += al64(Mz * h);
  // cross backward partials per block: {dw_o [W, T], db_o [T]} then column sums of dt [W],
  // dc [W]
  p->xdt_col = ((size_t)W * T + T + 3) / 4 * 4;
  p->xpart_stride = al64(p->xdt_col + 2 * (size_t)W);
  p->xblocks = M > 0 ? (M + kXRows - 1) / kXRows : 1;
  p->xpart_off = w; w += (size_t)p->xblocks * p->xpart_stride;
  if (T > 1) {
    p->r_off = w; w += al64(Mz * W);
  }
  p->ws_floats = w;
}

__device__ __forceinline__ float uniform01(unsigned long long s, unsigned long long e) {
  unsigned long long z = s + 0x9E3779B97F4A7C15ull * (e + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (float)(z >> 40) * (1.0f / 16777216.0f);
}

__host__ __device__ inline unsigned long long site_seed(unsigned long long seed, int site) {
  return seed * 0x100000001B3ull + (unsigned long long)site;
}

unsigned blocks_for(size_t n, int per) { return (unsigned)((n + per - 1) / per); }

// a0 = gamma (X - mean) rstd + beta (+ sigma g, the DIN's Box-Muller on uniforms 2e, 2e + 1).
__global__ void __launch_bounds__(256)
input_bn_noise_kernel(const float* __restrict__ X, size_t total, int D,
                      const float* __restrict__ stat, const float* __restrict__ gamma,
                      const float* __restrict__ beta, float sigma, unsigned long long s,
                      float* __restrict__ a0) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int c = (int)(e % D);
  float v = fmaf(gamma[c], (X[e] - stat[c]) * stat[D + c], beta[c]);
  if (sigma > 0.f) {
    const float u1 = uniform01(s, 2 * e), u2 = uniform01(s, 2 * e + 1);
    v += sigma * (sqrtf(-2.f * logf(1.f - u1)) * cospif(2.f * u2));
  }
  a0[e] = v;
}

// dst [M, h] = src rows (pitch lds).
__global__ void __launch_bounds__(256)
copy_rows_kernel(const float* __restrict__ src, int lds, size_t M, int h,
                 float* __restrict__ dst) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * h) return;
  const size_t r = i / h;
  dst[i] = src[r * lds + (i - r * h)];
}

// s_u[m] = sum_j drop(relu(t c + t))_j w_o[j, u] + b_o[u] for the kT tasks u, into plane u
// (scores + u M); ln(1e-10) on every plane for masked rows; one warp per row.  w_o is [W, kT],
// so column quad q's 4 kT weights are the float4s q kT .. q kT + kT - 1.
template <int kT>
__global__ void __launch_bounds__(256)
cross_fwd_kernel(const float4* __restrict__ t, const float4* __restrict__ c,
                 const float4* __restrict__ wo, const float* __restrict__ bo,
                 const uint8_t* __restrict__ mask, int M, int W4, float drop,
                 unsigned long long s, float* __restrict__ scores) {
  const int lane = threadIdx.x & 31;
  const int m = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (m >= M) return;
  if (mask && !mask[m]) {
    if (lane < kT) scores[(size_t)lane * M + m] = kLogEpsilon;
    return;
  }
  const float ks = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  const unsigned long long e0 = (unsigned long long)m * W4 * 4;
  float acc[kT];
#pragma unroll
  for (int u = 0; u < kT; ++u) acc[u] = 0.f;
  for (int q = lane; q < W4; q += 32) {
    const float4 tv = t[(size_t)m * W4 + q], cv = c[(size_t)m * W4 + q];
    const float tt[4] = {tv.x, tv.y, tv.z, tv.w}, cc[4] = {cv.x, cv.y, cv.z, cv.w};
    float ww[4 * kT];
#pragma unroll
    for (int i = 0; i < kT; ++i) {
      const float4 w = wo[(size_t)q * kT + i];
      ww[4 * i] = w.x; ww[4 * i + 1] = w.y; ww[4 * i + 2] = w.z; ww[4 * i + 3] = w.w;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float o = fmaxf(fmaf(tt[k], cc[k], tt[k]), 0.f);
      if (drop > 0.f) o = uniform01(s, e0 + 4 * q + k) < drop ? 0.f : o * ks;
#pragma unroll
      for (int u = 0; u < kT; ++u) acc[u] = fmaf(o, ww[k * kT + u], acc[u]);
    }
  }
#pragma unroll
  for (int u = 0; u < kT; ++u) acc[u] = warp_sum(acc[u]);
  if (lane == 0) {
#pragma unroll
    for (int u = 0; u < kT; ++u) scores[(size_t)u * M + m] = acc[u] + bo[u];
  }
}

// Cross backward over rows [blockIdx.x * kXRows, ...): with ds_u = tw_u dscores_u (0 on masked
// rows) and the combined signal sw = sum_u ds_u w_o[:, u], g = sw keep / (1 - p) [t(c+1) > 0],
// dt = g (c + 1), dc = g t; this block's partials of sum dt and sum dc.  With one task also
// {dw_o = sum ds o, db_o = sum ds}; with more, the dropped outputs o go to r [M, W] for
// task_out_grad_kernel instead.  Thread (lane_r, q0) owns column quads q0 + k cw and rows
// lane_r, lane_r + rl, ...; the rl row lanes are summed in order through shared memory.
template <int kT>
__global__ void __launch_bounds__(256)
cross_bwd_kernel(const float4* __restrict__ t, const float4* __restrict__ c,
                 const float4* __restrict__ wo, const float* __restrict__ dscores,
                 TaskWeights tw, const uint8_t* __restrict__ mask, int M, int W4, int cw,
                 float drop, unsigned long long s, float4* __restrict__ dt,
                 float4* __restrict__ dc, float4* __restrict__ r, float* __restrict__ part,
                 size_t pstride, size_t dt_col) {
  constexpr bool kOne = kT == 1;
  __shared__ float red[256][13];
  const int tid = threadIdx.x;
  const int rl = 256 / cw, lane_r = tid / cw, q0 = tid % cw;
  const int mbeg = blockIdx.x * kXRows, mend = min(M, mbeg + kXRows);
  const float ks = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  float4 w[kOne ? kXQ : 1];   // one task: w_o stays in registers; more: read per row (L1)
  float aw[kOne ? kXQ : 1][4], at[kXQ][4], ac[kXQ][4];
#pragma unroll
  for (int k = 0; k < kXQ; ++k) {
    const int q = q0 + k * cw;
    if constexpr (kOne) {
      w[k] = q < W4 ? wo[q] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int j = 0; j < 4; ++j) aw[k][j] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) at[k][j] = ac[k][j] = 0.f;
  }
  float adb = 0.f;
  for (int m = mbeg + lane_r; m < mend; m += rl) {
    const bool off = mask && !mask[m];
    float ds[kT];
#pragma unroll
    for (int u = 0; u < kT; ++u) ds[u] = off ? 0.f : tw.w[u] * dscores[(size_t)u * M + m];
    adb += ds[0];
    const unsigned long long e0 = (unsigned long long)m * W4 * 4;
#pragma unroll
    for (int k = 0; k < kXQ; ++k) {
      const int q = q0 + k * cw;
      if (q >= W4) continue;
      const size_t i = (size_t)m * W4 + q;
      const float4 tv = t[i], cv = c[i];
      const float tt[4] = {tv.x, tv.y, tv.z, tv.w}, cc[4] = {cv.x, cv.y, cv.z, cv.w};
      float sw[4];   // sum_u ds_u w_o[4q + j, u]
      if constexpr (kOne) {
        const float ww[4] = {w[k].x, w[k].y, w[k].z, w[k].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) sw[j] = ds[0] * ww[j];
      } else {
        float ww[4 * kT];
#pragma unroll
        for (int u = 0; u < kT; ++u) {
          const float4 wv = wo[(size_t)q * kT + u];
          ww[4 * u] = wv.x; ww[4 * u + 1] = wv.y; ww[4 * u + 2] = wv.z; ww[4 * u + 3] = wv.w;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          sw[j] = ds[0] * ww[j * kT];
#pragma unroll
          for (int u = 1; u < kT; ++u) sw[j] = fmaf(ds[u], ww[j * kT + u], sw[j]);
        }
      }
      float dtv[4], dcv[4], ov[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float v = fmaf(tt[j], cc[j], tt[j]);
        float f = v > 0.f ? ks : 0.f;   // d o / d v
        if (drop > 0.f && uniform01(s, e0 + 4 * q + j) < drop) f = 0.f;
        const float g = sw[j] * f;
        dtv[j] = g * (cc[j] + 1.f);
        dcv[j] = g * tt[j];
        ov[j] = v * f;
        if constexpr (kOne) aw[k][j] = fmaf(ds[0], ov[j], aw[k][j]);
        at[k][j] += dtv[j];
        ac[k][j] += dcv[j];
      }
      dt[i] = make_float4(dtv[0], dtv[1], dtv[2], dtv[3]);
      dc[i] = make_float4(dcv[0], dcv[1], dcv[2], dcv[3]);
      if constexpr (!kOne) r[i] = make_float4(ov[0], ov[1], ov[2], ov[3]);
    }
  }
  float* out = part + (size_t)blockIdx.x * pstride;
  if (rl > 1) {   // then every thread owns at most one quad (W4 <= cw <= 128)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if constexpr (kOne) red[tid][j] = aw[0][j];
      red[tid][4 + j] = at[0][j];
      red[tid][8 + j] = ac[0][j];
    }
    red[tid][12] = adb;
    __syncthreads();
    if (lane_r != 0) return;
    for (int rr = 1; rr < rl; ++rr) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if constexpr (kOne) aw[0][j] += red[rr * cw + q0][j];
        at[0][j] += red[rr * cw + q0][4 + j];
        ac[0][j] += red[rr * cw + q0][8 + j];
      }
      adb += red[rr * cw + q0][12];
    }
  }
#pragma unroll
  for (int k = 0; k < kXQ; ++k) {
    const int q = q0 + k * cw;
    if (q >= W4) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if constexpr (kOne) out[4 * q + j] = aw[k][j];
      out[dt_col + 4 * q + j] = at[k][j];
      out[dt_col + 4 * (size_t)W4 + 4 * q + j] = ac[k][j];
    }
  }
  if (kOne && q0 == 0) out[4 * (size_t)W4] = adb;
}

// More than one task: this block's partials {dw_o [W, kT], db_o [kT]} over rows
// [blockIdx.x * kXRows, ...) from the dropped cross outputs r [M, W]:
// dw_o[j, u] = sum_m ds_u[m] r[m, j], db_o[u] = sum_m ds_u[m], rows ascending.
template <int kT>
__global__ void __launch_bounds__(256)
task_out_grad_kernel(const float* __restrict__ r, const float* __restrict__ dscores,
                     TaskWeights tw, const uint8_t* __restrict__ mask, int M, int W,
                     float* __restrict__ part, size_t pstride) {
  __shared__ float dss[kXRows][kT];
  const int mbeg = blockIdx.x * kXRows, rows = min(M, mbeg + kXRows) - mbeg;
  for (int i = threadIdx.x; i < kXRows * kT; i += blockDim.x) {
    const int rr = i / kT, u = i - rr * kT, m = mbeg + rr;
    dss[rr][u] = (rr < rows && !(mask && !mask[m])) ? tw.w[u] * dscores[(size_t)u * M + m]
                                                    : 0.f;
  }
  __syncthreads();
  float* out = part + (size_t)blockIdx.x * pstride;
  for (int j = threadIdx.x; j < W; j += blockDim.x) {
    float acc[kT];
#pragma unroll
    for (int u = 0; u < kT; ++u) acc[u] = 0.f;
    for (int rr = 0; rr < rows; ++rr) {
      const float v = r[(size_t)(mbeg + rr) * W + j];
#pragma unroll
      for (int u = 0; u < kT; ++u) acc[u] = fmaf(dss[rr][u], v, acc[u]);
    }
#pragma unroll
    for (int u = 0; u < kT; ++u) out[(size_t)j * kT + u] = acc[u];
  }
  if (threadIdx.x < kT) {
    float a = 0.f;
    for (int rr = 0; rr < rows; ++rr) a += dss[rr][threadIdx.x];
    out[(size_t)W * kT + threadIdx.x] = a;
  }
}

// dZ = dR [Z > 0] (sign word bit) in place, and this split's column sums of dZ (the order of
// mlp_colsum: rows ascending per column).
__global__ void __launch_bounds__(256)
relu_gate_colsum_kernel(float* __restrict__ dz, const uint32_t* __restrict__ bits, int M, int N,
                        int rows_per, float* __restrict__ partial, size_t pstride) {
  const int z = blockIdx.x;
  const int mbeg = z * rows_per, mend = min(M, mbeg + rows_per);
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    const uint32_t* bw = bits + (size_t)(n >> 5) * M;
    const uint32_t bit = 1u << (n & 31);
    float acc = 0.f;
    for (int m = mbeg; m < mend; ++m) {
      const size_t i = (size_t)m * N + n;
      const float v = (bw[m] & bit) ? dz[i] : 0.f;
      dz[i] = v;
      acc += v;
    }
    partial[(size_t)z * pstride + n] = acc;
  }
}

// Context BN input gradient: dE = gamma rstd (dY - mean dY - xhat mean(dY xhat)); the two
// means are dbeta / M and dgamma / M, zero in inference (moving statistics are constants).
__global__ void __launch_bounds__(256)
context_bn_dx_kernel(const float* __restrict__ dy, const float* __restrict__ e, size_t M, int h,
                     const float* __restrict__ stat, const float* __restrict__ gamma,
                     const float* __restrict__ dgamma, const float* __restrict__ dbeta,
                     int training, float* __restrict__ dE, int ldde) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * h) return;
  const size_t r = i / h;
  const int c = (int)(i - r * h);
  const float rs = stat[h + c];
  const float xh = (e[i] - stat[c]) * rs;
  float v = dy[i];
  if (training) v = v - dbeta[c] / (float)M - xh * (dgamma[c] / (float)M);
  dE[r * ldde + c] = gamma[c] * rs * v;
}

__global__ void __launch_bounds__(256)
log1p_clip_kernel(const float* x, size_t n, float cutoff, float* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = x[i];
  const float r = copysignf(log1pf(fabsf(v)), v);
  out[i] = fminf(fmaxf(r, -cutoff), cutoff);
}

int cross_cw(int W4) {
  int cw = 32;
  while (cw < W4 && cw < 256) cw <<= 1;
  return cw;
}

int dasalc_fwd(const float* X, const float* E, int lde, const DasalcPlan& p, const float* params,
               const uint8_t* mask, float* ws, float* scores, int passes, cudaStream_t st) {
  const int M = p.M, D = p.D, W = p.W, h = p.h;
  const MlpPlan& a = p.a;
  const MlpPlan& c = p.c;
  int rc = mlp_tc_split_params(a, params, ws, passes, st);
  if (rc) return rc;
  rc = mlp_tc_split_params(c, params, ws, passes, st);
  if (rc) return rc;
  // input BN (+ GaussianNoise)
  rc = mlp_bn_batch_stats(X, M, D, a, ws, ws + a.bnstat_in_off, a.bn_state + a.stin_off, st);
  if (rc) return rc;
  input_bn_noise_kernel<<<blocks_for((size_t)M * D, 256), 256, 0, st>>>(
      X, (size_t)M * D, D, ws + a.bnstat_in_off, params + p.o_gin, params + p.o_bein, p.noise,
      site_seed(p.seed, kSiteNoise), ws + a.xin_off);
  TFR_LAUNCH_OK();
  // two hidden layers: relu(A W + b) with sign words, then BN + dropout (sites 1, 2)
  const float* in = ws + a.xin_off;
  for (int d = 0; d < 2; ++d) {
    rc = mlp_tc_dense_fwd(a, d, 0, a.dims[d], in, M, params, ws, params + a.b_off[d],
                          TFR_ACT_RELU, reinterpret_cast<uint32_t*>(ws + a.bits_off[d]),
                          ws + a.xhat_off[d], passes, st);
    if (rc) return rc;
    rc = mlp_hidden_post_fwd(d, M, a, params, ws, st);
    if (rc) return rc;
    in = ws + a.act_off[d];
  }
  rc = mlp_tc_dense_fwd(a, 2, 0, W, in, M, params, ws, params + p.o_bt, TFR_ACT_NONE, nullptr,
                        ws + p.t_off, passes, st);
  if (rc) return rc;
  // context branch: BN_c(E) W_c + b_c
  copy_rows_kernel<<<blocks_for((size_t)M * h, 256), 256, 0, st>>>(E, lde, (size_t)M, h,
                                                                   ws + p.ec_off);
  TFR_LAUNCH_OK();
  rc = mlp_input_bn_fwd(ws + p.ec_off, M, c, params, ws, st);
  if (rc) return rc;
  rc = mlp_tc_dense_fwd(c, 0, 0, h, ws + c.xin_off, M, params, ws, params + p.o_bc, TFR_ACT_NONE,
                        nullptr, ws + p.cc_off, passes, st);
  if (rc) return rc;
  with_tasks(p.T, [&](auto kt) {
    cross_fwd_kernel<decltype(kt)::value><<<blocks_for(M, 8), 256, 0, st>>>(
        reinterpret_cast<const float4*>(ws + p.t_off),
        reinterpret_cast<const float4*>(ws + p.cc_off),
        reinterpret_cast<const float4*>(params + p.o_wo), params + p.o_bo, mask, M, W / 4, p.drop,
        site_seed(p.seed, kSiteCross), scores);
  });
  TFR_LAUNCH_OK();
  return TFR_OK;
}

// dscores: T planes [T, M]; tw: the per-task weights.
int dasalc_bwd(const float* X, const DasalcPlan& p, const float* params, const float* dscores,
               const TaskWeights& tw, const uint8_t* mask, float* ws, float* grads, float* dE,
               int ldde, int passes, cudaStream_t st) {
  const int M = p.M, W = p.W, h = p.h;
  const MlpPlan& a = p.a;
  const MlpPlan& c = p.c;
  float* xpart = ws + p.xpart_off;
  float* partial = ws + a.partial_off;
  float* dt = ws + p.dt_off;
  float* dc = ws + p.dc_off;
  const int W4 = W / 4;
  const int T = p.T;
  with_tasks(T, [&](auto kt) {
    constexpr int kT = decltype(kt)::value;
    cross_bwd_kernel<kT><<<p.xblocks, 256, 0, st>>>(
        reinterpret_cast<const float4*>(ws + p.t_off),
        reinterpret_cast<const float4*>(ws + p.cc_off),
        reinterpret_cast<const float4*>(params + p.o_wo), dscores, tw, mask, M, W4, cross_cw(W4),
        p.drop, site_seed(p.seed, kSiteCross), reinterpret_cast<float4*>(dt),
        reinterpret_cast<float4*>(dc), reinterpret_cast<float4*>(ws + p.r_off), xpart,
        p.xpart_stride, p.xdt_col);
    if (kT > 1)
      task_out_grad_kernel<kT><<<p.xblocks, 256, 0, st>>>(ws + p.r_off, dscores, tw, mask, M, W,
                                                          xpart, p.xpart_stride);
  });
  TFR_LAUNCH_OK();
  int rc = mlp_reduce_partials(xpart, p.xblocks, p.xpart_stride, (size_t)W * T + T,
                               grads + p.o_wo, st);
  if (rc) return rc;
  // t = a_2 W_t + b_t
  rc = mlp_tc_weight_grad(ws + a.act_off[1], W, W, dt, W, W, M, a.splits, partial,
                          a.partial_stride, xpart + p.xdt_col, p.xblocks, p.xpart_stride, false,
                          grads + p.o_wt, passes, st);
  if (rc) return rc;
  float* dh0 = ws + p.dh_off[0];
  float* dh1 = ws + p.dh_off[1];
  rc = mlp_tc_dense_dgrad(a, 2, 0, W, dt, M, params, ws, nullptr, nullptr, 0, nullptr, dh0, W,
                          passes, st);
  if (rc) return rc;
  // c = BN_c(E) W_c + b_c, and dE through BN_c
  rc = mlp_tc_weight_grad(ws + c.xin_off, h, h, dc, W, W, M, a.splits, partial, a.partial_stride,
                          xpart + p.xdt_col + W, p.xblocks, p.xpart_stride, false, grads + p.o_wc,
                          passes, st);
  if (rc) return rc;
  float* dyc = ws + p.dyc_off;
  rc = mlp_tc_dense_dgrad(c, 0, 0, h, dc, M, params, ws, nullptr, nullptr, 0, nullptr, dyc, h,
                          passes, st);
  if (rc) return rc;
  rc = mlp_input_bn_bwd(ws + p.ec_off, M, c, params, ws, dyc, grads, st);
  if (rc) return rc;
  context_bn_dx_kernel<<<blocks_for((size_t)M * h, 256), 256, 0, st>>>(
      dyc, ws + p.ec_off, (size_t)M, h, ws + c.bnstat_in_off, params + p.o_gc, grads + p.o_gc,
      grads + p.o_bec, p.training, dE, ldde);
  TFR_LAUNCH_OK();
  // hidden layers 2, 1: dropout + BN backward, ReLU gate, dW, input side
  float* tiles = ws + a.tile_off;
  for (int d = 1; d >= 0; --d) {
    float* dz = d == 1 ? dh0 : dh1;
    rc = mlp_hidden_pre_bwd(d, M, a, params, ws, dz, grads, st);
    if (rc) return rc;
    relu_gate_colsum_kernel<<<a.splits, 256, 0, st>>>(
        dz, reinterpret_cast<const uint32_t*>(ws + a.bits_off[d]), M, W, a.rows_per_split, tiles,
        a.tile_stride);
    TFR_LAUNCH_OK();
    const int kin = a.dims[d];
    const float* A = d == 1 ? ws + a.act_off[0] : ws + a.xin_off;
    rc = mlp_tc_weight_grad(A, kin, kin, dz, W, W, M, a.splits, partial, a.partial_stride, tiles,
                            a.splits, a.tile_stride, false, grads + a.w_off[d], passes, st);
    if (rc) return rc;
    float* dnext = d == 1 ? dh1 : ws + p.da0_off;
    rc = mlp_tc_dense_dgrad(a, d, 0, kin, dz, M, params, ws, nullptr, nullptr, 0, nullptr, dnext,
                            kin, passes, st);
    if (rc) return rc;
  }
  // input BN: gamma / beta from dL/da0 (no gradient for X)
  return mlp_input_bn_bwd(X, M, a, params, ws, ws + p.da0_off, grads, st);
}

float* ws_align(void* w) {
  uintptr_t v = reinterpret_cast<uintptr_t>(w);
  return reinterpret_cast<float*>((v + 255) & ~(uintptr_t)255);
}

int passes_of(int precision) {
  if (precision == TFR_PREC_TF32X3) return 3;
  if (precision == TFR_PREC_TF32) return 1;
  return 0;
}

int check_call(const tfr_dasalc_cfg* cfg, int M, const float* params, void* ws, int precision) {
  int rc = check_cfg(cfg);
  if (rc) return rc;
  TFR_REQUIRE(cfg->bn_state != nullptr, "bn_state must not be NULL");
  TFR_REQUIRE(params && ws, "NULL argument");
  TFR_REQUIRE(M >= 0, "M must be >= 0");
  const int widest = cfg->input_dim > cfg->hidden_dim ? cfg->input_dim : cfg->hidden_dim;
  TFR_REQUIRE((long long)M * widest < (1ll << 31), "M * max(input_dim, hidden_dim) = %lld "
              "must be < 2^31", (long long)M * widest);
  if (!passes_of(precision)) {
    set_error("DASALC runs in precision TFR_PREC_TF32X3 or TFR_PREC_TF32, got %d", precision);
    return TFR_UNSUPPORTED;
  }
  return TFR_OK;
}

}  // namespace
}  // namespace tfr

using namespace tfr;

namespace {

size_t param_count(const tfr_dasalc_cfg* cfg, int T) {
  const size_t D = cfg->input_dim, W = cfg->hidden_dim, h = cfg->context_dim;
  return D * W + W + 2 * (W * W + W) + h * W + W + W * T + T + 2 * D + 4 * W + 2 * h;
}

// The multi-task limits, after check_cfg; TFR_INVALID_ARGUMENT before any CUDA call.
int check_tasks(int T, int precision) {
  TFR_REQUIRE(T >= 1 && T <= kMaxTasks, "num_tasks %d must be in [1, %d]", T, kMaxTasks);
  TFR_REQUIRE(passes_of(precision), "DASALC runs in precision TFR_PREC_TF32X3 or TFR_PREC_TF32, "
              "got %d", precision);
  return TFR_OK;
}

size_t workspace_bytes(const tfr_dasalc_cfg* cfg, int M, int T) {
  if (M < 0) {
    set_error("M must be >= 0");
    return 0;
  }
  DasalcPlan p;
  make_plan(cfg, M, T, &p);
  return p.ws_floats * sizeof(float) + 256;
}

int fwd_tasks(const float* X, const float* E, int lde, int M, const tfr_dasalc_cfg* cfg,
              const float* params, const uint8_t* mask, void* workspace, float* scores, int T,
              int precision, cudaStream_t st) {
  int rc = check_call(cfg, M, params, workspace, precision);
  if (rc) return rc;
  TFR_REQUIRE(X && E && scores, "NULL argument");
  TFR_REQUIRE(lde >= cfg->context_dim, "lde %d must be >= context_dim %d", lde, cfg->context_dim);
  if (M == 0) return TFR_OK;
  DasalcPlan p;
  make_plan(cfg, M, T, &p);
  return dasalc_fwd(X, E, lde, p, params, mask, ws_align(workspace), scores, passes_of(precision),
                    st);
}

int bwd_tasks(const float* X, int M, const tfr_dasalc_cfg* cfg, const float* params,
              const float* dscores, const TaskWeights& tw, const uint8_t* mask, void* workspace,
              float* grads, float* dE, int ldde, int T, int precision, cudaStream_t st) {
  int rc = check_call(cfg, M, params, workspace, precision);
  if (rc) return rc;
  TFR_REQUIRE(X && dscores && grads && dE, "NULL argument");
  TFR_REQUIRE(ldde >= cfg->context_dim, "ldde %d must be >= context_dim %d", ldde,
              cfg->context_dim);
  DasalcPlan p;
  if (M == 0) {
    TFR_CUDA_OK(cudaMemsetAsync(grads, 0, param_count(cfg, T) * sizeof(float), st));
    return TFR_OK;
  }
  make_plan(cfg, M, T, &p);
  return dasalc_bwd(X, p, params, dscores, tw, mask, ws_align(workspace), grads, dE, ldde,
                    passes_of(precision), st);
}

}  // namespace

extern "C" size_t tfr_dasalc_param_count(const tfr_dasalc_cfg* cfg) {
  if (check_cfg(cfg)) return 0;
  return param_count(cfg, 1);
}

extern "C" size_t tfr_dasalc_param_count_tasks(const tfr_dasalc_cfg* cfg, int num_tasks) {
  if (check_cfg(cfg)) return 0;
  if (num_tasks < 1 || num_tasks > kMaxTasks) {
    set_error("num_tasks %d must be in [1, %d]", num_tasks, kMaxTasks);
    return 0;
  }
  return param_count(cfg, num_tasks);
}

extern "C" size_t tfr_dasalc_bn_state_count(const tfr_dasalc_cfg* cfg) {
  if (check_cfg(cfg)) return 0;
  return 2 * ((size_t)cfg->input_dim + 2 * (size_t)cfg->hidden_dim + cfg->context_dim);
}

extern "C" size_t tfr_dasalc_workspace_bytes(const tfr_dasalc_cfg* cfg, int M) {
  if (check_cfg(cfg)) return 0;
  return workspace_bytes(cfg, M, 1);
}

extern "C" size_t tfr_dasalc_workspace_bytes_tasks(const tfr_dasalc_cfg* cfg, int M,
                                                   int num_tasks) {
  if (check_cfg(cfg)) return 0;
  if (num_tasks < 1 || num_tasks > kMaxTasks) {
    set_error("num_tasks %d must be in [1, %d]", num_tasks, kMaxTasks);
    return 0;
  }
  return workspace_bytes(cfg, M, num_tasks);
}

extern "C" int tfr_dasalc_fwd(const float* X, const float* E, int lde, int M,
                              const tfr_dasalc_cfg* cfg, const float* params, const uint8_t* mask,
                              void* workspace, float* scores, int precision, void* stream) {
  return fwd_tasks(X, E, lde, M, cfg, params, mask, workspace, scores, 1, precision,
                   (cudaStream_t)stream);
}

extern "C" int tfr_dasalc_fwd_tasks(const float* X, const float* E, int lde, int M,
                                    const tfr_dasalc_cfg* cfg, const float* params,
                                    const uint8_t* mask, void* workspace, float* score_planes,
                                    int num_tasks, int precision, void* stream) {
  int rc = check_cfg(cfg);
  if (rc) return rc;
  rc = check_tasks(num_tasks, precision);
  if (rc) return rc;
  return fwd_tasks(X, E, lde, M, cfg, params, mask, workspace, score_planes, num_tasks, precision,
                   (cudaStream_t)stream);
}

extern "C" int tfr_dasalc_bwd(const float* X, int M, const tfr_dasalc_cfg* cfg,
                              const float* params, const float* dscores, const uint8_t* mask,
                              void* workspace, float* grads, float* dE, int ldde, int precision,
                              void* stream) {
  TaskWeights tw;
  tw.w[0] = 1.f;
  return bwd_tasks(X, M, cfg, params, dscores, tw, mask, workspace, grads, dE, ldde, 1, precision,
                   (cudaStream_t)stream);
}

extern "C" int tfr_dasalc_bwd_tasks(const float* X, int M, const tfr_dasalc_cfg* cfg,
                                    const float* params, const float* dscore_planes,
                                    const float* task_weights_host, const uint8_t* mask,
                                    void* workspace, float* grads, float* dE, int ldde,
                                    int num_tasks, int precision, void* stream) {
  int rc = check_cfg(cfg);
  if (rc) return rc;
  rc = check_tasks(num_tasks, precision);
  if (rc) return rc;
  TaskWeights tw;
  for (int u = 0; u < kMaxTasks; ++u) {
    tw.w[u] = (task_weights_host && u < num_tasks) ? task_weights_host[u] : 1.f;
    TFR_REQUIRE(std::isfinite(tw.w[u]), "task weight %d is %g; weights must be finite", u,
                (double)tw.w[u]);
  }
  return bwd_tasks(X, M, cfg, params, dscore_planes, tw, mask, workspace, grads, dE, ldde,
                   num_tasks, precision, (cudaStream_t)stream);
}

extern "C" int tfr_symmetric_log1p_clip(const float* X, size_t n, float cutoff, float* out,
                                        void* stream) {
  TFR_REQUIRE(X && out, "NULL argument");
  TFR_REQUIRE(cutoff > 0.f, "cutoff %g must be > 0", (double)cutoff);
  if (n == 0) return TFR_OK;
  log1p_clip_kernel<<<blocks_for(n, 256), 256, 0, (cudaStream_t)stream>>>(X, n, cutoff, out);
  TFR_LAUNCH_OK();
  return TFR_OK;
}
