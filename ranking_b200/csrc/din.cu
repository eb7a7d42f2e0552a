// K11 DocumentInteractionAttention (keras/layers.py:420-588): per-list multi-head
// self-attention over the items of every list, num_layers times, on sm_90a.
//
//   x0   = relu(X W_in + b_in)  [+ sigma g in training]      3xTF32 GEMM, bias + ReLU epilogue
//   per layer l (Keras MultiHeadAttention, key_dim = output_shape = h):
//     [q | k | v] = x_l [Wq | Wk | Wv] + [bq | bk | bv]        one 3xTF32 GEMM (packed weights)
//     o    = softmax_j(q k_j / sqrt(h) - 1e9 [j padded]) (dropped) v   attention core, FP32 SIMT
//     y    = o Wo + bo                                         3xTF32 GEMM, bias epilogue
//     x_l+1 = LayerNorm(drop(y) + x_l)                         row kernel
//   The last layer's LayerNorm writes straight into the caller's buffer (leading dimension
//   ldo), e.g. columns [D, D + h) of the scorer tower's input.
//
// The attention core is one CTA per (list, head): 64 query rows x 4 threads, each thread
// owning head dimensions t, t + 4, ...; key / value tiles of 32 items stream through shared
// memory with an online softmax; the row max and 1 / (sum of exponentials) of every query row
// are kept for the backward.
// The backward recomputes P from it in two passes over the same (list, head) grid: one owns
// the queries (dQ, and D_i = rowsum(dO * O)), one owns the keys (dK, dV), so nothing is
// accumulated with atomics and two identical calls give identical bits.  Parameter
// gradients go through the 3xTF32 engine's split-K partials and fixed-order reductions.
// The input gradient (tfr_din_input_grad) is one more 3xTF32 GEMM, dX = dZ_in W_in^T, over the
// dZ_in the backward leaves in the workspace.
// precision TFR_PREC_TF32 runs every projection GEMM above in one TF32 pass instead of three,
// and the attention core on the tensor cores (din_tc.cu); the workspace is the same.
#include <cstring>

#include "common.cuh"
#include "din.cuh"
#include "mlp.h"
#include "tc_gemm.cuh"

namespace tfr {
namespace {

constexpr int kThreads = 256;
constexpr int kRows = kThreads / 4;   // query (or key) rows per pass of a CTA
constexpr int kKT = 32;               // items per shared-memory tile
constexpr int kMaxH = 128;
constexpr float kLnEps = 1e-12f;

struct DinPlan {
  int D, h, H, L, HH, B, N, M;
  float drop, noise;
  int training;
  int passes;   // of every projection GEMM: 3 (3xTF32) or 1 (TF32)
  bool tc;      // attention core on the TF32 tensor cores (din_tc.cu) instead of FP32 SIMT
  unsigned long long seed;
  size_t layer_off[TFR_DIN_MAX_LAYERS], layer_size, n_params;
  // workspace (floats)
  size_t wqkv_off, wqkv_stride;   // packed [h, 3HH] kernel + [3HH] bias per layer
  size_t a0_off, xn_off;          // relu(X W_in + b_in); the same plus noise (training)
  size_t qkv_off[TFR_DIN_MAX_LAYERS], o_off[TFR_DIN_MAX_LAYERS], lse_off[TFR_DIN_MAX_LAYERS];
  size_t xh_off[TFR_DIN_MAX_LAYERS], rstd_off[TFR_DIN_MAX_LAYERS], xo_off[TFR_DIN_MAX_LAYERS];
  size_t dres_off, tmp_off, dy_off, do_off, dqkv_off, dsum_off;
  size_t part_off, part_stride, cs_off, cs_stride;
  int rows_per_split, splits;
  size_t ws_floats;
  bool noisy() const { return training && noise > 0.f; }
  float adrop() const { return training ? drop : 0.f; }
  // layer l parameter offsets (Keras get_weights() order); Wk / Wv follow Wq at steps of
  // h * HH + HH
  __host__ __device__ size_t wq(int l) const { return layer_off[l]; }
  size_t wo(int l) const { return layer_off[l] + 3 * ((size_t)h * HH + HH); }
  size_t bo(int l) const { return wo(l) + (size_t)HH * h; }
  size_t gamma(int l) const { return bo(l) + h; }
};

size_t al64(size_t x) { return (x + 63) / 64 * 64; }

int make_din_plan(const tfr_din_cfg* c, int B, int N, DinPlan* p) {
  TFR_REQUIRE(c != nullptr, "cfg must not be NULL");
  TFR_REQUIRE(c->input_dim >= 4 && c->input_dim % 4 == 0,
              "input_dim %d must be a positive multiple of 4", c->input_dim);
  TFR_REQUIRE(c->head_size >= 4 && c->head_size % 4 == 0 && c->head_size <= kMaxH,
              "head_size %d must be a multiple of 4 in [4, %d]", c->head_size, kMaxH);
  TFR_REQUIRE(c->num_heads >= 1 && (long long)c->num_heads * c->head_size <= TFR_DIN_MAX_HH,
              "num_heads * head_size = %lld must be in [1, %d]",
              (long long)c->num_heads * c->head_size, TFR_DIN_MAX_HH);
  TFR_REQUIRE(c->num_layers >= 1 && c->num_layers <= TFR_DIN_MAX_LAYERS,
              "num_layers %d must be in [1, %d]", c->num_layers, TFR_DIN_MAX_LAYERS);
  TFR_REQUIRE(c->dropout >= 0.f && c->dropout < 1.f, "dropout %g must be in [0, 1)",
              (double)c->dropout);
  TFR_REQUIRE(c->input_noise_stddev >= 0.f, "input_noise_stddev must be >= 0");
  TFR_REQUIRE(B >= 0 && N >= 0, "batch and list size must be >= 0");
  TFR_REQUIRE(N <= TFR_DIN_MAX_LIST, "list_size %d exceeds %d", N, TFR_DIN_MAX_LIST);
  TFR_REQUIRE(c->precision == TFR_PREC_FP32 || c->precision == TFR_PREC_TF32,
              "precision %d must be TFR_PREC_FP32 (%d) or TFR_PREC_TF32 (%d)", c->precision,
              TFR_PREC_FP32, TFR_PREC_TF32);
  std::memset(p, 0, sizeof(*p));
  p->D = c->input_dim; p->h = c->head_size; p->H = c->num_heads; p->L = c->num_layers;
  p->HH = p->H * p->h;
  p->B = B; p->N = N; p->M = B * N;
  p->drop = c->dropout; p->noise = c->input_noise_stddev;
  p->training = c->training != 0; p->seed = c->seed;
  p->tc = c->precision == TFR_PREC_TF32;
  p->passes = p->tc ? 1 : 3;
  const int h = p->h, HH = p->HH;
  const size_t M = (size_t)p->M;
  size_t off = (size_t)p->D * h + h;
  p->layer_size = 3 * ((size_t)h * HH + HH) + (size_t)HH * h + 3 * (size_t)h;
  for (int l = 0; l < p->L; ++l) {
    p->layer_off[l] = off;
    off += p->layer_size;
  }
  p->n_params = off;
  size_t w = 0;
  p->wqkv_stride = al64((size_t)h * 3 * HH + 3 * HH);
  p->wqkv_off = w; w += p->L * p->wqkv_stride;
  p->a0_off = w; w += al64(M * h);
  p->xn_off = w; w += al64(M * h);
  for (int l = 0; l < p->L; ++l) {
    p->qkv_off[l] = w; w += al64(M * 3 * HH);
    p->o_off[l] = w; w += al64(M * HH);
    p->lse_off[l] = w; w += al64(2 * M * p->H);
    p->xh_off[l] = w; w += al64(M * h);
    p->rstd_off[l] = w; w += al64(M);
    p->xo_off[l] = w; w += l + 1 < p->L ? al64(M * h) : 0;
  }
  p->dres_off = w; w += al64(M * h);
  p->tmp_off = w; w += al64(M * h);
  p->dy_off = w; w += al64(M * h);
  p->do_off = w; w += al64(M * HH);
  p->dqkv_off = w; w += al64(M * 3 * HH);
  p->dsum_off = w; w += al64(M * p->H);
  // Row splits of the dW GEMMs: about one per SM, whole 32-row k blocks each, none empty.
  const int kb = (int)((M + 31) / 32);
  const int target = num_sms();
  const int kb_per = kb > 0 ? (kb + target - 1) / target : 1;
  p->rows_per_split = kb_per * 32;
  p->splits = kb > 0 ? (kb + kb_per - 1) / kb_per : 1;
  size_t wmax = 0;
  const int shapes[3][2] = {{p->D, h}, {HH, h}, {h, HH}};   // dW_in, dWo, dWq / dWk / dWv
  for (auto& s : shapes) {
    const size_t v = (size_t)((s[0] + 127) / 128 * 128) * s[1];
    if (v > wmax) wmax = v;
  }
  p->part_stride = al64(wmax);
  p->part_off = w; w += (size_t)p->splits * p->part_stride;
  p->cs_stride = al64(3 * (size_t)HH > 2 * (size_t)h ? 3 * (size_t)HH : 2 * (size_t)h);
  p->cs_off = w; w += (size_t)p->splits * p->cs_stride;
  p->ws_floats = w;
  return TFR_OK;
}

__host__ __device__ inline unsigned long long site_seed(unsigned long long seed, int site) {
  return seed * 0x100000001B3ull + (unsigned long long)site;
}

// Packs layer l's Wq, Wk, Wv [h, HH] and biases into [h, 3HH] + [3HH]; blockIdx.y = layer.
__global__ void __launch_bounds__(256)
pack_qkv_kernel(const float* __restrict__ params, DinPlan p, float* __restrict__ ws) {
  const int l = blockIdx.y;
  const int HH = p.HH, h = p.h;
  const size_t n = (size_t)(h + 1) * 3 * HH;
  float* dst = ws + p.wqkv_off + l * p.wqkv_stride;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i / (3 * HH)), c3 = (int)(i % (3 * HH));
    const int t = c3 / HH, c = c3 % HH;
    const size_t base = p.wq(l) + (size_t)t * ((size_t)h * HH + HH);
    dst[i] = params[base + (size_t)k * HH + c];   // k == h: the bias row
  }
}

// x + sigma * g, g = sqrt(-2 ln(1 - u1)) cos(2 pi u2), u1 / u2 the uniforms 2e / 2e + 1.
__global__ void __launch_bounds__(256)
noise_kernel(const float* __restrict__ a, size_t n, float sigma, unsigned long long s,
             float* __restrict__ out) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const float u1 = din_uniform(s, 2 * e), u2 = din_uniform(s, 2 * e + 1);
  out[e] = a[e] + sigma * (sqrtf(-2.f * logf(1.f - u1)) * cospif(2.f * u2));
}

// Loads a [kKT, h] tile of items j0.. of one head (columns col0..) into shared memory.
__device__ __forceinline__ void load_tile(float (*dst)[kMaxH], const float* __restrict__ src,
                                          int ld, int j0, int n, int h) {
  for (int e = threadIdx.x; e < kKT * h; e += kThreads) {
    const int jj = e / h, c = e - jj * h;
    dst[jj][c] = jj < n ? src[(size_t)(j0 + jj) * ld + c] : 0.f;
  }
}

__device__ __forceinline__ float group_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

// Forward attention core.  qkv [M, 3HH]; O [M, HH]; lse [M, H, 2] = {row max, 1 / sum}.
template <int KD>
__global__ void __launch_bounds__(kThreads)
attn_fwd_kernel(const float* __restrict__ qkv, const uint8_t* __restrict__ lmask, int N, int H,
                int h, float scale, float drop, unsigned long long dseed, float* __restrict__ O,
                float* __restrict__ lse) {
  __shared__ float Ks[kKT][kMaxH], Vs[kKT][kMaxH];
  __shared__ uint8_t vm[kKT];
  const int b = blockIdx.x / H, hd = blockIdx.x % H;
  const int HH = H * h, ld = 3 * HH;
  const size_t row0 = (size_t)b * N;
  const float* Qg = qkv + row0 * ld + hd * h;
  const float* Kg = Qg + HH;
  const float* Vg = Qg + 2 * HH;
  const int t = threadIdx.x & 3, r = threadIdx.x >> 2;
  const float kscale = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  const unsigned long long ebase = (unsigned long long)blockIdx.x * N;   // (b * H + hd) * N
  for (int i0 = 0; i0 < N; i0 += kRows) {
    const int i = i0 + r;
    const bool active = i < N;
    float q[KD], acc[KD];
#pragma unroll
    for (int k = 0; k < KD; ++k) {
      const int c = t + 4 * k;
      q[k] = (active && c < h) ? Qg[(size_t)i * ld + c] * scale : 0.f;
      acc[k] = 0.f;
    }
    float m = -INFINITY, l = 0.f;
    for (int j0 = 0; j0 < N; j0 += kKT) {
      const int nk = min(kKT, N - j0);
      __syncthreads();
      load_tile(Ks, Kg, ld, j0, nk, h);
      load_tile(Vs, Vg, ld, j0, nk, h);
      if (threadIdx.x < kKT)
        vm[threadIdx.x] = threadIdx.x < nk ? (lmask ? lmask[row0 + j0 + threadIdx.x] : 1) : 0;
      __syncthreads();
      float s[kKT];
      float tmax = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < kKT; ++jj) {
        float d = 0.f;
#pragma unroll
        for (int k = 0; k < KD; ++k)
          if (t + 4 * k < h) d += q[k] * Ks[jj][t + 4 * k];
        d = group_sum(d);
        s[jj] = jj < nk ? (vm[jj] ? d : d + kMaskAdder) : -INFINITY;
        tmax = fmaxf(tmax, s[jj]);
      }
      const float mn = fmaxf(m, tmax);
      const float corr = expf(m - mn);
      l *= corr;
#pragma unroll
      for (int k = 0; k < KD; ++k) acc[k] *= corr;
#pragma unroll
      for (int jj = 0; jj < kKT; ++jj) {
        if (jj < nk) {
          const float pr = expf(s[jj] - mn);
          l += pr;
          float pk = pr;
          if (drop > 0.f)
            pk = din_uniform(dseed, (ebase + i) * N + j0 + jj) >= drop ? pr * kscale : 0.f;
#pragma unroll
          for (int k = 0; k < KD; ++k)
            if (t + 4 * k < h) acc[k] += pk * Vs[jj][t + 4 * k];
        }
      }
      m = mn;
    }
    if (active) {
      const float inv = 1.f / l;
      float* o = O + (row0 + i) * HH + hd * h;
#pragma unroll
      for (int k = 0; k < KD; ++k)
        if (t + 4 * k < h) o[t + 4 * k] = acc[k] * inv;
      if (t == 0) {   // max and 1 / sum: exact for a list with no valid item (all -1e9)
        lse[((row0 + i) * H + hd) * 2] = m;
        lse[((row0 + i) * H + hd) * 2 + 1] = inv;
      }
    }
  }
}

// Backward, query-owning pass: D_i = rowsum(dO_i * O_i) and
// dQ_i = scale * sum_j P_ij (dP~_ij keep_ij / (1 - rate) - D_i) k_j,  dP~_ij = dO_i . v_j.
template <int KD>
__global__ void __launch_bounds__(kThreads)
attn_bwd_dq_kernel(const float* __restrict__ qkv, const uint8_t* __restrict__ lmask, int N,
                   int H, int h, float scale, float drop, unsigned long long dseed,
                   const float* __restrict__ O, const float* __restrict__ lse,
                   const float* __restrict__ dO, float* __restrict__ dsum,
                   float* __restrict__ dqkv) {
  __shared__ float Ks[kKT][kMaxH], Vs[kKT][kMaxH];
  __shared__ uint8_t vm[kKT];
  const int b = blockIdx.x / H, hd = blockIdx.x % H;
  const int HH = H * h, ld = 3 * HH;
  const size_t row0 = (size_t)b * N;
  const float* Qg = qkv + row0 * ld + hd * h;
  const float* Kg = Qg + HH;
  const float* Vg = Qg + 2 * HH;
  const int t = threadIdx.x & 3, r = threadIdx.x >> 2;
  const float kscale = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  const unsigned long long ebase = (unsigned long long)blockIdx.x * N;
  for (int i0 = 0; i0 < N; i0 += kRows) {
    const int i = i0 + r;
    const bool active = i < N;
    const size_t ri = row0 + (active ? i : 0);
    float q[KD], g[KD], dq[KD];
    float di = 0.f;
#pragma unroll
    for (int k = 0; k < KD; ++k) {
      const int c = t + 4 * k;
      const bool ok = active && c < h;
      q[k] = ok ? Qg[(size_t)i * ld + c] * scale : 0.f;
      g[k] = ok ? dO[ri * HH + hd * h + c] : 0.f;
      di += ok ? g[k] * O[ri * HH + hd * h + c] : 0.f;
      dq[k] = 0.f;
    }
    di = group_sum(di);
    const float mi = active ? lse[(ri * H + hd) * 2] : 0.f;
    const float il = active ? lse[(ri * H + hd) * 2 + 1] : 0.f;
    if (active && t == 0) dsum[ri * H + hd] = di;
    for (int j0 = 0; j0 < N; j0 += kKT) {
      const int nk = min(kKT, N - j0);
      __syncthreads();
      load_tile(Ks, Kg, ld, j0, nk, h);
      load_tile(Vs, Vg, ld, j0, nk, h);
      if (threadIdx.x < kKT)
        vm[threadIdx.x] = threadIdx.x < nk ? (lmask ? lmask[row0 + j0 + threadIdx.x] : 1) : 0;
      __syncthreads();
#pragma unroll 4
      for (int jj = 0; jj < nk; ++jj) {
        float s = 0.f, dp = 0.f;
#pragma unroll
        for (int k = 0; k < KD; ++k)
          if (t + 4 * k < h) {
            s += q[k] * Ks[jj][t + 4 * k];
            dp += g[k] * Vs[jj][t + 4 * k];
          }
        s = group_sum(s);
        dp = group_sum(dp);
        if (!vm[jj]) s += kMaskAdder;
        const float pr = expf(s - mi) * il;
        float kf = 1.f;
        if (drop > 0.f) kf = din_uniform(dseed, (ebase + i) * N + j0 + jj) >= drop ? kscale : 0.f;
        const float ds = pr * (dp * kf - di);
#pragma unroll
        for (int k = 0; k < KD; ++k)
          if (t + 4 * k < h) dq[k] += ds * Ks[jj][t + 4 * k];
      }
    }
    if (active) {
      float* o = dqkv + ri * ld + hd * h;
#pragma unroll
      for (int k = 0; k < KD; ++k)
        if (t + 4 * k < h) o[t + 4 * k] = dq[k] * scale;
    }
  }
}

// Backward, key-owning pass: dK_j = sum_i dS_ij q_i scale, dV_j = sum_i P~_ij dO_i.
template <int KD>
__global__ void __launch_bounds__(kThreads)
attn_bwd_dkv_kernel(const float* __restrict__ qkv, const uint8_t* __restrict__ lmask, int N,
                    int H, int h, float scale, float drop, unsigned long long dseed,
                    const float* __restrict__ lse, const float* __restrict__ dsum,
                    const float* __restrict__ dO, float* __restrict__ dqkv) {
  __shared__ float Qs[kKT][kMaxH], Gs[kKT][kMaxH];
  __shared__ float ms[kKT], ls[kKT], ds_[kKT];
  const int b = blockIdx.x / H, hd = blockIdx.x % H;
  const int HH = H * h, ld = 3 * HH;
  const size_t row0 = (size_t)b * N;
  const float* Qg = qkv + row0 * ld + hd * h;
  const float* Kg = Qg + HH;
  const float* Vg = Qg + 2 * HH;
  const int t = threadIdx.x & 3, r = threadIdx.x >> 2;
  const float kscale = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  const unsigned long long ebase = (unsigned long long)blockIdx.x * N;
  for (int j0 = 0; j0 < N; j0 += kRows) {
    const int j = j0 + r;
    const bool active = j < N;
    const bool valid = active && (lmask ? lmask[row0 + j] != 0 : true);
    float kk[KD], vv[KD], dk[KD], dv[KD];
#pragma unroll
    for (int k = 0; k < KD; ++k) {
      const int c = t + 4 * k;
      const bool ok = active && c < h;
      kk[k] = ok ? Kg[(size_t)j * ld + c] : 0.f;
      vv[k] = ok ? Vg[(size_t)j * ld + c] : 0.f;
      dk[k] = dv[k] = 0.f;
    }
    for (int i0 = 0; i0 < N; i0 += kKT) {
      const int nq = min(kKT, N - i0);
      __syncthreads();
      for (int e = threadIdx.x; e < kKT * h; e += kThreads) {
        const int ii = e / h, c = e - ii * h;
        Qs[ii][c] = ii < nq ? Qg[(size_t)(i0 + ii) * ld + c] * scale : 0.f;
        Gs[ii][c] = ii < nq ? dO[(row0 + i0 + ii) * HH + hd * h + c] : 0.f;
      }
      if (threadIdx.x < kKT) {
        const bool ok = threadIdx.x < nq;
        ms[threadIdx.x] = ok ? lse[((row0 + i0 + threadIdx.x) * H + hd) * 2] : 0.f;
        ls[threadIdx.x] = ok ? lse[((row0 + i0 + threadIdx.x) * H + hd) * 2 + 1] : 0.f;
        ds_[threadIdx.x] = ok ? dsum[(row0 + i0 + threadIdx.x) * H + hd] : 0.f;
      }
      __syncthreads();
#pragma unroll 4
      for (int ii = 0; ii < nq; ++ii) {
        float s = 0.f, dp = 0.f;
#pragma unroll
        for (int k = 0; k < KD; ++k)
          if (t + 4 * k < h) {
            s += Qs[ii][t + 4 * k] * kk[k];
            dp += Gs[ii][t + 4 * k] * vv[k];
          }
        s = group_sum(s);
        dp = group_sum(dp);
        if (!valid) s += kMaskAdder;
        const float pr = expf(s - ms[ii]) * ls[ii];
        float kf = 1.f;
        if (drop > 0.f && active)
          kf = din_uniform(dseed, (ebase + i0 + ii) * N + j) >= drop ? kscale : 0.f;
        const float ds = pr * (dp * kf - ds_[ii]);
        const float pt = pr * kf;
#pragma unroll
        for (int k = 0; k < KD; ++k)
          if (t + 4 * k < h) {
            dk[k] += ds * Qs[ii][t + 4 * k];
            dv[k] += pt * Gs[ii][t + 4 * k];
          }
      }
    }
    if (active) {
      float* o = dqkv + (row0 + j) * ld + hd * h;
#pragma unroll
      for (int k = 0; k < KD; ++k)
        if (t + 4 * k < h) {
          o[HH + t + 4 * k] = dk[k];
          o[2 * HH + t + 4 * k] = dv[k];
        }
    }
  }
}

// x_l+1 = LayerNorm(drop(y) + x_l) * gamma + beta, one warp per row.  `y` and `xhat` may be
// the same buffer (each row is read completely before it is written).
__global__ void __launch_bounds__(256)
ln_fwd_kernel(const float* y, const float* __restrict__ xres, int M, int h,
              const float* __restrict__ gamma, const float* __restrict__ beta, float drop,
              unsigned long long dseed, float* xhat, float* __restrict__ rstd,
              float* __restrict__ out, int ldo) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= M) return;
  const float kscale = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  float z[4];
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int c = lane + 32 * k;
    z[k] = 0.f;
    if (c < h) {
      const size_t e = (size_t)row * h + c;
      float v = y[e];
      if (drop > 0.f) v = din_uniform(dseed, e) >= drop ? v * kscale : 0.f;
      z[k] = v + xres[e];
      sum += z[k];
    }
  }
  const float mean = warp_sum(sum) / h;
  float sq = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (lane + 32 * k < h) sq += (z[k] - mean) * (z[k] - mean);
  const float rs = rsqrtf(warp_sum(sq) / h + kLnEps);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int c = lane + 32 * k;
    if (c < h) {
      const float xh = (z[k] - mean) * rs;
      xhat[(size_t)row * h + c] = xh;
      out[(size_t)row * ldo + c] = xh * gamma[c] + beta[c];
    }
  }
  if (lane == 0) rstd[row] = rs;
}

// LayerNorm backward over rows [z * rows_per, ...) of CTA z, one warp per row:
//   dZ = rstd (g gamma - mean(g gamma) - xhat mean(g gamma xhat)) -> dres (residual branch)
//   dY = drop'(dZ)                                                -> dy
// and this CTA's partial sums of dgamma = sum g xhat, dbeta = sum g (fixed order).
// `g` may alias `dres` (ldg == h): each row is read completely before it is written.
__global__ void __launch_bounds__(256)
ln_bwd_kernel(const float* g, int ldg, const float* __restrict__ xhat,
              const float* __restrict__ rstd, const float* __restrict__ gamma, int M, int h,
              int rows_per, float drop, unsigned long long dseed, float* dres,
              float* __restrict__ dy, float* __restrict__ partial, size_t pstride) {
  __shared__ float red[8][2 * kMaxH];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int beg = blockIdx.x * rows_per, end = min(M, beg + rows_per);
  const float kscale = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  float ag[4] = {0.f, 0.f, 0.f, 0.f}, ab[4] = {0.f, 0.f, 0.f, 0.f};
  for (int row = beg + warp; row < end; row += 8) {
    float gv[4], xv[4], dx[4];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = lane + 32 * k;
      gv[k] = xv[k] = dx[k] = 0.f;
      if (c < h) {
        gv[k] = g[(size_t)row * ldg + c];
        xv[k] = xhat[(size_t)row * h + c];
        dx[k] = gv[k] * gamma[c];
        s1 += dx[k];
        s2 += dx[k] * xv[k];
      }
    }
    s1 = warp_sum(s1) / h;
    s2 = warp_sum(s2) / h;
    const float rs = rstd[row];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = lane + 32 * k;
      if (c < h) {
        const size_t e = (size_t)row * h + c;
        const float dz = rs * (dx[k] - s1 - xv[k] * s2);
        dres[e] = dz;
        dy[e] = drop > 0.f ? (din_uniform(dseed, e) >= drop ? dz * kscale : 0.f) : dz;
        ag[k] += gv[k] * xv[k];
        ab[k] += gv[k];
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int c = lane + 32 * k;
    if (c < h) {
      red[warp][c] = ag[k];
      red[warp][h + c] = ab[k];
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * h; c += blockDim.x) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][c];
    partial[(size_t)blockIdx.x * pstride + c] = s;
  }
}

// dres = tmp + dres, times [a0 > 0] when a0 is given (the input projection's ReLU).
__global__ void __launch_bounds__(256)
add_mask_kernel(const float* __restrict__ tmp, const float* __restrict__ a0, size_t n,
                float* __restrict__ dres) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = tmp[i] + dres[i];
  dres[i] = (a0 && !(a0[i] > 0.f)) ? 0.f : v;
}

unsigned blocks_for(size_t n, int per) { return (unsigned)((n + per - 1) / per); }

// grads[w .. w + Kin * Nout + Nout) = {A^T dZ, column sums of dZ} over the plan's row splits.
int weight_grad(const DinPlan& p, float* ws, const float* A, int lda, int Kin, const float* dZ,
                int ldz, int Nout, const float* colsum_src, float* grads_w, cudaStream_t st) {
  return din_weight_grad(A, lda, Kin, dZ, ldz, Nout, p.M, p.splits, ws + p.part_off,
                         p.part_stride, colsum_src, p.cs_stride, grads_w, p.passes, st);
}

template <int KD>
int attn_fwd(const float* qkv, const uint8_t* lmask, int B, int N, int H, int h, float drop,
             unsigned long long s, float* O, float* lse, cudaStream_t st) {
  attn_fwd_kernel<KD><<<B * H, kThreads, 0, st>>>(qkv, lmask, N, H, h, 1.f / sqrtf((float)h),
                                                  drop, s, O, lse);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

template <int KD>
int attn_bwd(const float* qkv, const uint8_t* lmask, int B, int N, int H, int h, float drop,
             unsigned long long s, const float* O, const float* lse, const float* dO,
             float* dsum, float* dqkv, cudaStream_t st) {
  const float scale = 1.f / sqrtf((float)h);
  attn_bwd_dq_kernel<KD><<<B * H, kThreads, 0, st>>>(qkv, lmask, N, H, h, scale, drop, s, O, lse,
                                                     dO, dsum, dqkv);
  TFR_LAUNCH_OK();
  attn_bwd_dkv_kernel<KD><<<B * H, kThreads, 0, st>>>(qkv, lmask, N, H, h, scale, drop, s, lse,
                                                      dsum, dO, dqkv);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

}  // namespace

#define TFR_DIN_DISPATCH(fn, ...)                                        \
  (h <= 16 ? fn<4>(__VA_ARGS__) : h <= 32 ? fn<8>(__VA_ARGS__)           \
   : h <= 64 ? fn<16>(__VA_ARGS__) : fn<32>(__VA_ARGS__))

int din_attn_fwd(const float* qkv, const uint8_t* lmask, int B, int N, int H, int h, float drop,
                 unsigned long long dseed, float* O, float* lse, cudaStream_t st) {
  return TFR_DIN_DISPATCH(attn_fwd, qkv, lmask, B, N, H, h, drop, dseed, O, lse, st);
}

int din_attn_bwd(const float* qkv, const uint8_t* lmask, int B, int N, int H, int h, float drop,
                 unsigned long long dseed, const float* O, const float* lse, const float* dO,
                 float* dsum, float* dqkv, cudaStream_t st) {
  return TFR_DIN_DISPATCH(attn_bwd, qkv, lmask, B, N, H, h, drop, dseed, O, lse, dO, dsum, dqkv,
                          st);
}

int din_gemm(const float* A, int lda, int a_mn, const float* B, int ldb, int b_mn, float* C,
             int ldc, int GM, int GN, int GK, const float* bias, int act, int passes,
             cudaStream_t st) {
  tc::GemmDesc g{};
  g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.B_lo = nullptr;
  g.C = C; g.ldc = ldc;
  g.GM = GM; g.GN = GN; g.GK = GK;
  g.a_mn = a_mn; g.b_mn = b_mn; g.passes = passes; g.split_b = 1;
  g.epi = bias ? tc::EPI_BIAS_ACT : tc::EPI_STORE;
  g.bias = bias; g.act = act;
  g.splits = 1;
  return tc::gemm(g, st);
}

// The tower's fewer-tile-units rule would swap the DIN's q / k / v slices at h = 64 with two
// heads, which changes their rounding: hence the direct orientation.
int din_weight_grad(const float* A, int lda, int Kin, const float* dZ, int ldz, int Nout, int M,
                    int splits, float* partial, size_t pstride, const float* colsum,
                    size_t cs_stride, float* grads_w, int passes, cudaStream_t st) {
  return mlp_tc_weight_grad(A, lda, Kin, dZ, ldz, Nout, M, splits, partial, pstride, colsum,
                            splits, cs_stride, true, grads_w, passes, st);
}

namespace {

const float* layer_input(const DinPlan& p, const float* ws, int l) {
  if (l > 0) return ws + p.xo_off[l - 1];
  return ws + (p.noisy() ? p.xn_off : p.a0_off);
}

int din_fwd(const float* X, const uint8_t* lmask, const DinPlan& p, const float* params,
            float* ws, float* out, int ldo, cudaStream_t st) {
  const int h = p.h, HH = p.HH, M = p.M;
  pack_qkv_kernel<<<dim3(32, p.L), 256, 0, st>>>(params, p, ws);
  TFR_LAUNCH_OK();
  int rc = din_gemm(X, p.D, 0, params, h, 1, ws + p.a0_off, h, M, h, p.D,
                    params + (size_t)p.D * h, TFR_ACT_RELU, p.passes, st);
  if (rc) return rc;
  if (p.noisy()) {
    noise_kernel<<<blocks_for((size_t)M * h, 256), 256, 0, st>>>(
        ws + p.a0_off, (size_t)M * h, p.noise, site_seed(p.seed, 1), ws + p.xn_off);
    TFR_LAUNCH_OK();
  }
  const float drop = p.adrop();
  for (int l = 0; l < p.L; ++l) {
    const float* xl = layer_input(p, ws, l);
    const float* wqkv = ws + p.wqkv_off + l * p.wqkv_stride;
    float* qkv = ws + p.qkv_off[l];
    rc = din_gemm(xl, h, 0, wqkv, 3 * HH, 1, qkv, 3 * HH, M, 3 * HH, h,
                  wqkv + (size_t)h * 3 * HH, TFR_ACT_NONE, p.passes, st);
    if (rc) return rc;
    rc = p.tc ? din_tc_attn_fwd(qkv, lmask, p.B, p.N, p.H, h, drop, site_seed(p.seed, 2 + 2 * l),
                                ws + p.o_off[l], ws + p.lse_off[l], st)
              : din_attn_fwd(qkv, lmask, p.B, p.N, p.H, h, drop, site_seed(p.seed, 2 + 2 * l),
                             ws + p.o_off[l], ws + p.lse_off[l], st);
    if (rc) return rc;
    float* y = ws + p.xh_off[l];
    rc = din_gemm(ws + p.o_off[l], HH, 0, params + p.wo(l), h, 1, y, h, M, h, HH,
                  params + p.bo(l), TFR_ACT_NONE, p.passes, st);
    if (rc) return rc;
    const bool last = l + 1 == p.L;
    ln_fwd_kernel<<<blocks_for(M, 8), 256, 0, st>>>(
        y, xl, M, h, params + p.gamma(l), params + p.gamma(l) + h, drop,
        site_seed(p.seed, 3 + 2 * l), y, ws + p.rstd_off[l], last ? out : ws + p.xo_off[l],
        last ? ldo : h);
    TFR_LAUNCH_OK();
  }
  return TFR_OK;
}

int din_bwd(const float* X, const uint8_t* lmask, const DinPlan& p, const float* params,
            const float* dout, int lddo, float* ws, float* grads, cudaStream_t st) {
  const int h = p.h, HH = p.HH, M = p.M;
  const float drop = p.adrop();
  float* dres = ws + p.dres_off;
  float* tmp = ws + p.tmp_off;
  float* dy = ws + p.dy_off;
  float* dO = ws + p.do_off;
  float* dqkv = ws + p.dqkv_off;
  float* cs = ws + p.cs_off;
  int rc;
  for (int l = p.L - 1; l >= 0; --l) {
    const bool last = l + 1 == p.L;
    ln_bwd_kernel<<<p.splits, 256, 0, st>>>(
        last ? dout : dres, last ? lddo : h, ws + p.xh_off[l], ws + p.rstd_off[l],
        params + p.gamma(l), M, h, p.rows_per_split, drop, site_seed(p.seed, 3 + 2 * l), dres, dy,
        ws + p.part_off, p.part_stride);
    TFR_LAUNCH_OK();
    rc = mlp_reduce_partials(ws + p.part_off, p.splits, p.part_stride, 2 * (size_t)h,
                             grads + p.gamma(l), st);
    if (rc) return rc;
    // output projection: dWo, dbo, dO = dY Wo^T
    rc = mlp_colsum(dy, M, h, p.rows_per_split, p.splits, cs, p.cs_stride, 0, st);
    if (rc) return rc;
    rc = weight_grad(p, ws, ws + p.o_off[l], HH, HH, dy, h, h, cs, grads + p.wo(l), st);
    if (rc) return rc;
    rc = din_gemm(dy, h, 0, params + p.wo(l), h, 0, dO, HH, M, HH, h, nullptr, TFR_ACT_NONE,
                  p.passes, st);
    if (rc) return rc;
    const float* qkv = ws + p.qkv_off[l];
    rc = p.tc ? din_tc_attn_bwd(qkv, lmask, p.B, p.N, p.H, h, drop, site_seed(p.seed, 2 + 2 * l),
                                ws + p.o_off[l], ws + p.lse_off[l], dO, ws + p.dsum_off, dqkv,
                                st)
              : din_attn_bwd(qkv, lmask, p.B, p.N, p.H, h, drop, site_seed(p.seed, 2 + 2 * l),
                             ws + p.o_off[l], ws + p.lse_off[l], dO, ws + p.dsum_off, dqkv, st);
    if (rc) return rc;
    // Q / K / V projections: one dW GEMM each (the flat layout keeps them apart)
    const float* xl = layer_input(p, ws, l);
    rc = mlp_colsum(dqkv, M, 3 * HH, p.rows_per_split, p.splits, cs, p.cs_stride, 0, st);
    if (rc) return rc;
    for (int t = 0; t < 3; ++t) {
      rc = weight_grad(p, ws, xl, h, h, dqkv + (size_t)t * HH, 3 * HH, HH, cs + (size_t)t * HH,
                       grads + p.wq(l) + (size_t)t * ((size_t)h * HH + HH), st);
      if (rc) return rc;
    }
    // dX_l = dQKV [Wq | Wk | Wv]^T + residual branch (+ ReLU mask of the input projection)
    const float* wqkv = ws + p.wqkv_off + l * p.wqkv_stride;
    rc = din_gemm(dqkv, 3 * HH, 0, wqkv, 3 * HH, 0, tmp, h, M, h, 3 * HH, nullptr, TFR_ACT_NONE,
                  p.passes, st);
    if (rc) return rc;
    add_mask_kernel<<<blocks_for((size_t)M * h, 256), 256, 0, st>>>(
        tmp, l == 0 ? ws + p.a0_off : nullptr, (size_t)M * h, dres);
    TFR_LAUNCH_OK();
  }
  rc = mlp_colsum(dres, M, h, p.rows_per_split, p.splits, cs, p.cs_stride, 0, st);
  if (rc) return rc;
  return weight_grad(p, ws, X, p.D, p.D, dres, h, h, cs, grads, st);
}

// dst[r, c] (row pitch ldd) += src[r, c] (row pitch nc), r < M, c < nc.
__global__ void __launch_bounds__(256)
add_cols_kernel(const float* __restrict__ src, size_t M, int nc, float* __restrict__ dst,
                int ldd) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * nc) return;
  const size_t r = i / nc;
  const int c = (int)(i - r * nc);
  dst[r * ldd + c] += src[i];
}

// dX[:, 0 : ncols) (pitch ldx) = or += dres W_in[col0 : col0 + ncols, :]^T, where dres is the
// dZ_in that din_bwd left in the workspace.  The GEMM runs in column chunks of at most 3 HH
// in both modes, so the two launch the same GEMMs and += adds exactly the = result.  When
// accumulating, a chunk lands in the dqkv scratch (dead after din_bwd) and is then added.
int din_input_grad(const DinPlan& p, const float* params, float* ws, int col0, int ncols,
                   float* dX, int ldx, bool accumulate, cudaStream_t st) {
  const int h = p.h, chunk = 3 * p.HH;
  const float* dres = ws + p.dres_off;
  float* scratch = ws + p.dqkv_off;
  for (int c0 = 0; c0 < ncols; c0 += chunk) {
    const int nc = ncols - c0 < chunk ? ncols - c0 : chunk;
    float* out = accumulate ? scratch : dX + c0;
    int rc = din_gemm(dres, h, 0, params + (size_t)(col0 + c0) * h, h, 0, out,
                      accumulate ? nc : ldx, p.M, nc, h, nullptr, TFR_ACT_NONE, p.passes, st);
    if (rc) return rc;
    if (accumulate) {
      add_cols_kernel<<<blocks_for((size_t)p.M * nc, 256), 256, 0, st>>>(scratch, (size_t)p.M,
                                                                          nc, dX + c0, ldx);
      TFR_LAUNCH_OK();
    }
  }
  return TFR_OK;
}

float* ws_align(void* w) {
  uintptr_t a = reinterpret_cast<uintptr_t>(w);
  return reinterpret_cast<float*>((a + 255) & ~(uintptr_t)255);
}

}  // namespace
}  // namespace tfr

using namespace tfr;

extern "C" size_t tfr_din_param_count(const tfr_din_cfg* cfg) {
  DinPlan p;
  if (make_din_plan(cfg, 0, 0, &p)) return 0;
  return p.n_params;
}

extern "C" size_t tfr_din_workspace_bytes(const tfr_din_cfg* cfg, int B, int N) {
  DinPlan p;
  if (make_din_plan(cfg, B, N, &p)) return 0;
  return p.ws_floats * sizeof(float) + 256;
}

extern "C" int tfr_din_fwd(const float* X, const uint8_t* list_mask, int B, int N,
                           const tfr_din_cfg* cfg, const float* params, void* workspace,
                           float* out, int ldo, void* stream) {
  DinPlan p;
  int rc = make_din_plan(cfg, B, N, &p);
  if (rc) return rc;
  TFR_REQUIRE(X && params && workspace && out, "NULL argument");
  TFR_REQUIRE(ldo >= p.h, "ldo %d must be >= head_size %d", ldo, p.h);
  if (p.M == 0) return TFR_OK;
  return din_fwd(X, list_mask, p, params, ws_align(workspace), out, ldo, (cudaStream_t)stream);
}

extern "C" int tfr_din_bwd(const float* X, const uint8_t* list_mask, int B, int N,
                           const tfr_din_cfg* cfg, const float* params, const float* dout,
                           int lddo, void* workspace, float* grads, void* stream) {
  DinPlan p;
  int rc = make_din_plan(cfg, B, N, &p);
  if (rc) return rc;
  TFR_REQUIRE(X && params && workspace && dout && grads, "NULL argument");
  TFR_REQUIRE(lddo >= p.h, "lddo %d must be >= head_size %d", lddo, p.h);
  if (p.M == 0) {
    TFR_CUDA_OK(cudaMemsetAsync(grads, 0, p.n_params * sizeof(float), (cudaStream_t)stream));
    return TFR_OK;
  }
  return din_bwd(X, list_mask, p, params, dout, lddo, ws_align(workspace), grads,
                 (cudaStream_t)stream);
}

extern "C" int tfr_din_input_grad(const tfr_din_cfg* cfg, int B, int N, const float* params,
                                  void* workspace, int col0, int ncols, float* dX, int ldx,
                                  int accumulate, void* stream) {
  // every argument check comes before make_din_plan, whose SM-count query is a CUDA call
  TFR_REQUIRE(cfg != nullptr, "cfg must not be NULL");
  TFR_REQUIRE(params && workspace && dX, "NULL argument");
  TFR_REQUIRE(col0 >= 0 && ncols >= 1 && (long long)col0 + ncols <= cfg->input_dim,
              "columns [%d, %lld) outside the DIN input [0, %d)", col0,
              (long long)col0 + ncols, cfg->input_dim);
  TFR_REQUIRE(ldx >= ncols, "ldx %d must be >= ncols %d", ldx, ncols);
  TFR_REQUIRE(accumulate == 0 || accumulate == 1, "accumulate must be 0 or 1, got %d",
              accumulate);
  DinPlan p;
  int rc = make_din_plan(cfg, B, N, &p);
  if (rc) return rc;
  if (p.M == 0) return TFR_OK;
  return din_input_grad(p, params, ws_align(workspace), col0, ncols, dX, ldx, accumulate != 0,
                        (cudaStream_t)stream);
}
