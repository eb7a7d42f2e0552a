// K10: neural additive ranking model (GAMLayer, keras/layers.py:591-803).
//
// F example towers create_tower(hidden, 1) over one feature each, plus optional context
// towers create_tower(context_hidden, F) + softmax.  The example towers are block-diagonal:
// as one Dense stack they would multiply mostly zeros or write [M, F * h] activations per
// layer (1.8 GB for the first hidden layer of the canned-GAM recipe at B = 1024, N = 200).
// Here one thread evaluates one (row, feature) tower in registers with fp32 FFMA, and every
// pass ("sweep") recomputes the towers from X, so no per-feature hidden activation reaches
// HBM.  A CTA owns `nw` consecutive features (one warp each) and a range of rows; a warp
// walks its rows 32 at a time (lane = row), so every parameter read is a shared-memory
// broadcast of the warp's own padded parameter copy.
//
// Sweeps of one training step with BatchNormalization (L hidden layers):
//   forward   STATS(0) .. STATS(L-1)  batch mean / M2 of layer l's pre-BN values (Chan merge
//                                     of per-tile statistics, per-CTA partials merged in
//                                     split order), each followed by a finalize kernel
//             FWD                     sublogits [M, F]; then the combine kernel writes logits
//   backward  RED(L-1) .. RED(0)      sum dY and sum dY * xhat of BN layer l (the mean terms
//                                     of the BN backward), each followed by a finalize kernel
//             GRAD                    full backward; per-warp gradients are reduced over the
//                                     32 rows of a tile through shared memory into a
//                                     per-warp accumulator; per-CTA partials are summed in
//                                     split order by one more kernel (no float atomics)
// Without BN (or in inference) the forward is one sweep and the backward one sweep.
// Context towers run on the fp32 tower path (mlp_simt) over their own buffer slices.
#include <cstring>

#include "common.cuh"
#include "mlp.h"

namespace tfr {

namespace {

constexpr int kMaxF = TFR_GAM_MAX_FEATURES;
constexpr int kMaxL = TFR_GAM_MAX_HIDDEN;
constexpr int kMaxH = 64;
constexpr int kMaxDf = 32;
constexpr size_t kSmemBudget = 227 * 1024;

enum GamMode { GAM_STATS = 0, GAM_FWD = 1, GAM_RED = 2, GAM_GRAD = 3 };

struct GamArgs {
  const float* X;
  const float* params;
  const uint8_t* mask;
  const float* dlogits;   // upstream gradient per row (no context) ...
  const float* ds;        // ... or per (row, feature) [M, F] (context weighting)
  float* sub;             // GAM_FWD: sublogits [M, F]
  const float* bnstat;    // per BN layer d at bnst_off[d]: mean [F * h_d], rstd [F * h_d]
  const float* coef;      // same layout: mean(dY), mean(dY * xhat)
  float* part;            // STATS / RED: [split][F * h_l][2];  GRAD: [split][ex_params]
  size_t ex_params;
  int M, D, F, L, layer, act, use_bn, training, nw, rows_per;
  int h[kMaxL + 1];       // hidden widths; h[L] = 1 (the output Dense)
  float drop, scale;
  unsigned long long seed;
  int pconst;             // parameters of one example tower except W_0
  int bnst_off[kMaxL];
  // padded per-warp parameter copy: Dense d is a (K_d + 1) x pcols[d] block at prow[d]
  // (bias = last row; K_0 = dfmax), then BN gamma / beta at pg / pb
  int pp, dfmax;
  int prow[kMaxL + 1], pcols[kMaxL + 1], pg[kMaxL], pb[kMaxL];
  // per-row stash (backward): I_d = [input of Dense d, 1] at sin[d], xhat_d at sxh[d],
  // dZ of the current layer at sdz, dY at sdy; row stride ss (ss / 4 odd)
  int ss, sin[kMaxL + 1], sxh[kMaxL], sdz, sdy;
  int foff[kMaxF + 1];
};

__device__ __forceinline__ float uniform01(unsigned long long seed, unsigned long long idx) {
  unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (idx + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (float)(z >> 40) * (1.0f / 16777216.0f);
}

// Padded position of element i of a tower's tfr_mlp parameter slice (input width df).
__device__ int gam_pidx(const GamArgs& a, int i, int df) {
  const int n0 = a.h[0];
  if (i < (df + 1) * n0) {
    const int k = i / n0, u = i - k * n0;
    return a.prow[0] + (k < df ? k : a.dfmax) * a.pcols[0] + u;
  }
  i -= (df + 1) * n0;
  for (int d = 1; d <= a.L; ++d) {
    const int n = a.h[d], sz = (a.h[d - 1] + 1) * n;
    if (i < sz) {
      const int k = i / n;
      return a.prow[d] + k * a.pcols[d] + (i - k * n);
    }
    i -= sz;
  }
  for (int d = 0; d < a.L; ++d) {
    if (i < a.h[d]) return a.pg[d] + i;
    i -= a.h[d];
    if (i < a.h[d]) return a.pb[d] + i;
    i -= a.h[d];
  }
  return 0;
}

__device__ __forceinline__ float keep_mask(float h, int act, bool drop) {
  if (act == TFR_ACT_RELU) return h > 0.f ? 1.f : 0.f;
  if (drop) return h != 0.f ? 1.f : 0.f;
  return 1.f;
}

template <int WM, int MODE>
__global__ void __launch_bounds__(256, 1)
gam_sweep_kernel(const __grid_constant__ GamArgs a) {
  constexpr bool BWD = MODE >= GAM_RED;
  constexpr bool GRAD = MODE == GAM_GRAD;
  extern __shared__ float4 gam_smem4[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int f = blockIdx.x * a.nw + warp;
  if (f >= a.F) return;   // warps are independent: no block-wide barrier below
  const int per_warp = a.pp * (GRAD ? 2 : 1) + (BWD ? 32 * a.ss : 0);
  float* prm = reinterpret_cast<float*>(gam_smem4) + (size_t)warp * per_warp;
  float* acc = prm + a.pp;
  float* stash = prm + a.pp * (GRAD ? 2 : 1);
  float* my = stash + lane * a.ss;
  const int c0 = a.foff[f], df = a.foff[f + 1] - c0;
  const int L = a.L;
  const int P = df * a.h[0] + a.pconst;
  const size_t base = (size_t)c0 * a.h[0] + (size_t)f * a.pconst;
  for (int i = lane; i < a.pp; i += 32) {
    prm[i] = 0.f;
    if (GRAD) acc[i] = 0.f;
  }
  __syncwarp();
  for (int i = lane; i < P; i += 32) prm[gam_pidx(a, i, df)] = a.params[base + i];
  if (BWD) {
    for (int i = 0; i < a.ss; ++i) my[i] = 0.f;
    for (int d = 0; d <= L; ++d) my[a.sin[d] + (d == 0 ? a.dfmax : a.h[d - 1])] = 1.f;
  }
  __syncwarp();

  const bool drop = a.training && a.drop > 0.f;
  const unsigned long long F64 = (unsigned long long)a.F;
  // per-lane statistics of layer `layer` (units lane and lane + 32)
  double st_a0 = 0.0, st_a1 = 0.0, st_b0 = 0.0, st_b1 = 0.0;
  int n_run = 0;
  const int hl = (MODE == GAM_STATS || MODE == GAM_RED) ? a.h[a.layer] : 0;

  const int rbeg = blockIdx.y * a.rows_per, rend = min(a.M, rbeg + a.rows_per);
  for (int t0 = rbeg; t0 < rend; t0 += 32) {
    const int m = t0 + lane;
    const bool live = m < rend;
    const int nt = min(32, rend - t0);
    float hc[WM], z[WM];
    // ---- Dense 0 from X
    {
      const int n0 = a.h[0];
      const float* W = prm + a.prow[0];
      const int pc = a.pcols[0];
#pragma unroll
      for (int u = 0; u < WM; ++u) z[u] = u < n0 ? W[a.dfmax * pc + u] : 0.f;
      const float* xr = a.X + (size_t)(live ? m : rbeg) * a.D + c0;
      for (int k = 0; k < df; ++k) {
        const float xk = live ? __ldg(xr + k) : 0.f;
        if (BWD) my[a.sin[0] + k] = xk;
        const float* w = W + k * pc;
#pragma unroll
        for (int u4 = 0; u4 < WM / 4; ++u4) {
          if (4 * u4 < n0) {
            const float4 wv = *reinterpret_cast<const float4*>(w + 4 * u4);
            z[4 * u4 + 0] = fmaf(xk, wv.x, z[4 * u4 + 0]);
            z[4 * u4 + 1] = fmaf(xk, wv.y, z[4 * u4 + 1]);
            z[4 * u4 + 2] = fmaf(xk, wv.z, z[4 * u4 + 2]);
            z[4 * u4 + 3] = fmaf(xk, wv.w, z[4 * u4 + 3]);
          }
        }
      }
    }
    // ---- hidden layers: [BN] -> act -> [dropout] -> Dense d + 1
    bool stop = false;
    for (int d = 0; d < L; ++d) {
      const int n = a.h[d];
      if (MODE == GAM_STATS && d == a.layer) {
        // tile statistics, then Chan's merge into the running (n, mean, M2) of lane u % 32
#pragma unroll
        for (int u = 0; u < WM; ++u) {
          if (u < n) {
            const float v = live ? z[u] : 0.f;
            const float tmean = warp_sum(v) / (float)nt;
            const float dv = live ? z[u] - tmean : 0.f;
            const float tm2 = warp_sum(dv * dv);
            if ((u & 31) == lane) {
              double& ma = u < 32 ? st_a0 : st_a1;
              double& mb = u < 32 ? st_b0 : st_b1;
              const double na = (double)n_run, nb = (double)nt, nn = na + nb;
              const double delta = (double)tmean - ma;
              ma += delta * (nb / nn);
              mb += tm2 + delta * delta * (na * nb / nn);
            }
          }
        }
        n_run += nt;
        stop = true;
        break;
      }
      const float* mean = a.bnstat + a.bnst_off[d] + (size_t)f * n;
      const float* rstd = mean + (size_t)a.F * n;
      const unsigned long long sd = a.seed * 0x100000001B3ull + (unsigned long long)(d + 1);
      const unsigned long long ebase = ((unsigned long long)(live ? m : 0) * F64 + f) * n;
#pragma unroll
      for (int u = 0; u < WM; ++u) {
        if (u < n) {
          float v = z[u];
          if (a.use_bn) {
            const float xh = (v - __ldg(mean + u)) * __ldg(rstd + u);
            if (BWD) my[a.sxh[d] + u] = xh;
            v = fmaf(prm[a.pg[d] + u], xh, prm[a.pb[d] + u]);
          }
          if (a.act == TFR_ACT_RELU) v = fmaxf(v, 0.f);
          if (drop) v = uniform01(sd, ebase + u) < a.drop ? 0.f : v * a.scale;
          hc[u] = v;
          if (BWD) my[a.sin[d + 1] + u] = v;
        } else {
          hc[u] = 0.f;
        }
      }
      const int nn = a.h[d + 1];
      const float* W = prm + a.prow[d + 1];
      const int pc = a.pcols[d + 1];
#pragma unroll
      for (int v = 0; v < WM; ++v) z[v] = v < nn ? W[n * pc + v] : 0.f;
#pragma unroll
      for (int k = 0; k < WM; ++k) {
        if (k < n) {
          const float hk = hc[k];
          const float* w = W + k * pc;
#pragma unroll
          for (int v4 = 0; v4 < WM / 4; ++v4) {
            if (4 * v4 < nn) {
              const float4 wv = *reinterpret_cast<const float4*>(w + 4 * v4);
              z[4 * v4 + 0] = fmaf(hk, wv.x, z[4 * v4 + 0]);
              z[4 * v4 + 1] = fmaf(hk, wv.y, z[4 * v4 + 1]);
              z[4 * v4 + 2] = fmaf(hk, wv.z, z[4 * v4 + 2]);
              z[4 * v4 + 3] = fmaf(hk, wv.w, z[4 * v4 + 3]);
            }
          }
        }
      }
    }
    if (stop) continue;
    if (MODE == GAM_FWD) {
      if (live) a.sub[(size_t)m * a.F + f] = z[0];
      continue;
    }
    if (!BWD) continue;

    // ---- backward: upstream gradient of s_f for this row
    float g = 0.f;
    if (live)
      g = a.ds ? a.ds[(size_t)m * a.F + f] : ((a.mask && !a.mask[m]) ? 0.f : a.dlogits[m]);
    float (&dh)[WM] = hc;
    float (&dz)[WM] = z;
    // Dense L (one output): dW_L = I_L * g, dh = g * W_L
    if (GRAD) my[a.sdz] = g;
    int dcur = L;   // Dense layer whose dZ sits in the stash (GRAD)
    for (;;) {
      if (GRAD) {
        // reduce dW_dcur / db_dcur over the tile's 32 rows: output (k, 4-column chunk c)
        __syncwarp();
        const int K = dcur == 0 ? df : a.h[dcur - 1];
        const int N = a.h[dcur];
        const int nc = (N + 3) >> 2;
        const int ss = a.ss;
        for (int idx = lane; idx < (K + 1) * nc; idx += 32) {
          const int k = idx / nc, c = idx - k * nc;
          const int ks = (dcur == 0 && k == K) ? a.dfmax : k;
          const float* ip = stash + a.sin[dcur] + ks;
          const float* dp = stash + a.sdz + 4 * c;
          float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 8
          for (int r = 0; r < 32; ++r) {
            const float iv = ip[r * ss];
            const float4 dv = *reinterpret_cast<const float4*>(dp + r * ss);
            s.x = fmaf(iv, dv.x, s.x);
            s.y = fmaf(iv, dv.y, s.y);
            s.z = fmaf(iv, dv.z, s.z);
            s.w = fmaf(iv, dv.w, s.w);
          }
          float4* ac = reinterpret_cast<float4*>(acc + a.prow[dcur] + ks * a.pcols[dcur] + 4 * c);
          float4 o = *ac;
          o.x += s.x; o.y += s.y; o.z += s.z; o.w += s.w;
          *ac = o;
        }
        if (dcur < L && a.use_bn) {
          for (int u = lane; u < N; u += 32) {
            float sg = 0.f, sb = 0.f;
#pragma unroll 8
            for (int r = 0; r < 32; ++r) {
              const float dy = stash[r * ss + a.sdy + u];
              sg = fmaf(dy, stash[r * ss + a.sxh[dcur] + u], sg);
              sb += dy;
            }
            acc[a.pg[dcur] + u] += sg;
            acc[a.pb[dcur] + u] += sb;
          }
        }
        __syncwarp();
      }
      if (dcur == 0) break;
      // dh = dZ_dcur W_dcur^T  (input width K = h[dcur - 1])
      {
        const int K = a.h[dcur - 1], N = a.h[dcur];
        const float* W = prm + a.prow[dcur];
        const int pc = a.pcols[dcur];
        float gz[WM];
        if (dcur == L) {
#pragma unroll
          for (int k = 0; k < WM; ++k) dh[k] = k < K ? g * W[k * pc] : 0.f;
        } else {
#pragma unroll
          for (int u = 0; u < WM; ++u) gz[u] = dz[u];
#pragma unroll
          for (int k = 0; k < WM; ++k) {
            float t = 0.f;
            if (k < K) {
              const float* w = W + k * pc;
#pragma unroll
              for (int u4 = 0; u4 < WM / 4; ++u4) {
                if (4 * u4 < N) {
                  const float4 wv = *reinterpret_cast<const float4*>(w + 4 * u4);
                  t = fmaf(gz[4 * u4 + 0], wv.x, t);
                  t = fmaf(gz[4 * u4 + 1], wv.y, t);
                  t = fmaf(gz[4 * u4 + 2], wv.z, t);
                  t = fmaf(gz[4 * u4 + 3], wv.w, t);
                }
              }
            }
            dh[k] = t;
          }
        }
      }
      // hidden layer d = dcur - 1: dY = dH * dropout / act mask; BN backward -> dZ_d
      const int d = dcur - 1;
      const int n = a.h[d];
      const bool red_here = MODE == GAM_RED && d == a.layer;
      const float* c1 = a.coef + a.bnst_off[d] + (size_t)f * n;
      const float* c2 = c1 + (size_t)a.F * n;
      const float* rstd = a.bnstat + a.bnst_off[d] + (size_t)a.F * n + (size_t)f * n;
#pragma unroll
      for (int u = 0; u < WM; ++u) {
        float out = 0.f;
        if (u < n) {
          const float hv = my[a.sin[d + 1] + u];
          const float dy = dh[u] * (drop ? a.scale : 1.f) * keep_mask(hv, a.act, drop);
          out = dy;
          if (a.use_bn) {
            const float xh = my[a.sxh[d] + u];
            if (red_here) {
              const float s1 = warp_sum(dy), s2 = warp_sum(dy * xh);
              if ((u & 31) == lane) {
                (u < 32 ? st_a0 : st_a1) += s1;
                (u < 32 ? st_b0 : st_b1) += s2;
              }
            } else {
              if (GRAD) my[a.sdy + u] = dy;
              const float m1 = a.training ? __ldg(c1 + u) : 0.f;
              const float m2 = a.training ? __ldg(c2 + u) : 0.f;
              out = prm[a.pg[d] + u] * __ldg(rstd + u) * (dy - m1 - xh * m2);
            }
          }
        }
        // rows past the end of the range carry no gradient (the BN mean terms would
        // otherwise make theirs nonzero)
        dz[u] = live ? out : 0.f;
      }
      if (red_here) break;
      if (GRAD) {
#pragma unroll
        for (int u = 0; u < WM; ++u)
          if (u < n) my[a.sdz + u] = dz[u];
      }
      dcur = d;
    }
  }

  // ---- per-CTA partials
  if (MODE == GAM_STATS || MODE == GAM_RED) {
    float* out = a.part + ((size_t)blockIdx.y * a.F + f) * hl * 2;
    if (lane < hl) {
      out[2 * lane] = (float)st_a0;
      out[2 * lane + 1] = (float)st_b0;
    }
    if (lane + 32 < hl) {
      out[2 * lane + 64] = (float)st_a1;
      out[2 * lane + 65] = (float)st_b1;
    }
  }
  if (GRAD) {
    __syncwarp();
    float* out = a.part + (size_t)blockIdx.y * a.ex_params + base;
    for (int i = lane; i < P; i += 32) out[i] = acc[gam_pidx(a, i, df)];
  }
}

// Merge the per-split (mean, M2) of one BN layer in split order (fp64); mean / rstd; moving
// update.
__global__ void __launch_bounds__(256)
gam_stats_finalize_kernel(const float* __restrict__ part, int splits, int rows_per, int M,
                          int F, int n, float eps, float mom, float* __restrict__ stat,
                          float* __restrict__ bn_state, int state_stride, int state_off) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F * n) return;
  double cnt = 0.0, dmean = 0.0, m2 = 0.0;
  for (int s = 0; s < splits; ++s) {
    const double nb = (double)(min(M, (s + 1) * rows_per) - s * rows_per);
    const double mb = part[((size_t)s * F * n + i) * 2], qb = part[((size_t)s * F * n + i) * 2 + 1];
    const double nn = cnt + nb, delta = mb - dmean;
    dmean += delta * (nb / nn);
    m2 += qb + delta * delta * (cnt * nb / nn);
    cnt = nn;
  }
  const float mean = (float)dmean, var = (float)(m2 / (double)M);
  stat[i] = mean;
  stat[(size_t)F * n + i] = rsqrtf(var + eps);
  const int f = i / n, u = i - f * n;
  float* mv = bn_state + (size_t)f * state_stride + state_off;
  mv[u] = mv[u] * mom + mean * (1.f - mom);
  mv[n + u] = mv[n + u] * mom + var * (1.f - mom);
}

__global__ void __launch_bounds__(256)
gam_stats_from_moving_kernel(const float* __restrict__ bn_state, int F, int n, float eps,
                             int state_stride, int state_off, float* __restrict__ stat) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F * n) return;
  const int f = i / n, u = i - f * n;
  const float* mv = bn_state + (size_t)f * state_stride + state_off;
  stat[i] = mv[u];
  stat[(size_t)F * n + i] = rsqrtf(mv[n + u] + eps);
}

// coef = (sum dY, sum dY * xhat) / M, summed in split order.
__global__ void __launch_bounds__(256)
gam_red_finalize_kernel(const float* __restrict__ part, int splits, int M, int F, int n,
                        float* __restrict__ coef) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F * n) return;
  double s1 = 0.0, s2 = 0.0;
  for (int s = 0; s < splits; ++s) {
    s1 += part[((size_t)s * F * n + i) * 2];
    s2 += part[((size_t)s * F * n + i) * 2 + 1];
  }
  coef[i] = (float)(s1 / M);
  coef[(size_t)F * n + i] = (float)(s2 / M);
}

// Softmax over the F outputs of context tower j for row m (one warp, lane = feature, F <= 32).
__device__ __forceinline__ float ctx_softmax(const float* ctx, int m, int F, int lane) {
  const float c = lane < F ? ctx[(size_t)m * F + lane] : -INFINITY;
  const float mx = warp_max(c);
  const float e = lane < F ? __expf(c - mx) : 0.f;
  return e / warp_sum(e);
}

// logits[m] = sum_f s_f (no context) or sum_f s_f w_f; RestoreList fill.  One warp per row.
__global__ void __launch_bounds__(256)
gam_combine_fwd_kernel(const float* __restrict__ sub, const float* __restrict__ ctx, int C,
                       int M, int F, const uint8_t* __restrict__ mask,
                       float* __restrict__ logits, float* __restrict__ subweights) {
  const int lane = threadIdx.x & 31;
  const int m = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (m >= M) return;
  float t = 0.f;
  if (C == 0) {
    for (int f = lane; f < F; f += 32) t += sub[(size_t)m * F + f];
  } else {
    float w = 0.f;
    for (int j = 0; j < C; ++j) {
      const float p = ctx_softmax(ctx + (size_t)j * M * F, m, F, lane);
      if (subweights && lane < F) subweights[((size_t)j * M + m) * F + lane] = p;
      w += p;
    }
    if (lane < F) t = sub[(size_t)m * F + lane] * w;
  }
  t = warp_sum(t);
  if (lane == 0) logits[m] = (mask && !mask[m]) ? kLogEpsilon : t;
}

// ds[m, f] = g w_f; dctx_j[m, f] = p_jf (g s_f - sum_f' p_jf' g s_f').
__global__ void __launch_bounds__(256)
gam_combine_bwd_kernel(const float* __restrict__ sub, const float* __restrict__ ctx, int C,
                       int M, int F, const uint8_t* __restrict__ mask,
                       const float* __restrict__ dlogits, float* __restrict__ ds,
                       float* __restrict__ dctx) {
  const int lane = threadIdx.x & 31;
  const int m = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (m >= M) return;
  const float g = (mask && !mask[m]) ? 0.f : dlogits[m];
  const float s = lane < F ? sub[(size_t)m * F + lane] : 0.f;
  const float gs = g * s;
  float w = 0.f;
  for (int j = 0; j < C; ++j) {
    const float p = ctx_softmax(ctx + (size_t)j * M * F, m, F, lane);
    w += p;
    const float dot = warp_sum(p * gs);
    if (lane < F) dctx[((size_t)j * M + m) * F + lane] = p * (gs - dot);
  }
  if (lane < F) ds[(size_t)m * F + lane] = g * w;
}

size_t al64(size_t x) { return (x + 63) / 64 * 64; }
int pad4(int x) { return (x + 3) & ~3; }

struct GamPlan {
  GamArgs a;            // geometry part of the kernel arguments
  int F, L, C, wmax;
  size_t ex_params, n_params, ex_state, n_state, tower_state;
  int splits;
  size_t smem_fwd, smem_bwd, smem_grad;
  MlpPlan ctx[TFR_GAM_MAX_CONTEXT];
  size_t ctx_param_off[TFR_GAM_MAX_CONTEXT];
  // workspace (floats)
  size_t sub_off, ds_off, cout_off, dctx_off, cws_off[TFR_GAM_MAX_CONTEXT];
  size_t bnstat_off, coef_off, spart_off, gpart_off, ws_floats;
};

int make_gam_plan(const tfr_gam_cfg* cfg, int M, GamPlan* p) {
  TFR_REQUIRE(cfg != nullptr, "cfg must not be NULL");
  TFR_REQUIRE(M >= 0, "M must be >= 0");
  const int F = cfg->n_features, L = cfg->n_hidden, C = cfg->n_context;
  TFR_REQUIRE(F >= 1 && F <= kMaxF, "n_features %d must be in [1, %d]", F, kMaxF);
  TFR_REQUIRE(L >= 0 && L <= kMaxL, "n_hidden %d must be in [0, %d]", L, kMaxL);
  TFR_REQUIRE(C >= 0 && C <= TFR_GAM_MAX_CONTEXT, "n_context %d must be in [0, %d]", C,
              TFR_GAM_MAX_CONTEXT);
  TFR_REQUIRE(cfg->activation == TFR_ACT_NONE || cfg->activation == TFR_ACT_RELU,
              "activation %d unsupported", cfg->activation);
  TFR_REQUIRE(cfg->dropout >= 0.f && cfg->dropout < 1.f, "dropout %g must be in [0, 1)",
              (double)cfg->dropout);
  TFR_REQUIRE(cfg->feature_offsets[0] == 0, "feature_offsets[0] must be 0");
  std::memset(p, 0, sizeof(*p));
  GamArgs& a = p->a;
  int dfmax = 1;
  for (int f = 0; f < F; ++f) {
    const int df = cfg->feature_offsets[f + 1] - cfg->feature_offsets[f];
    TFR_REQUIRE(df >= 1 && df <= kMaxDf, "feature %d has width %d, must be in [1, %d]", f, df,
                kMaxDf);
    if (df > dfmax) dfmax = df;
  }
  for (int f = 0; f <= F; ++f) a.foff[f] = cfg->feature_offsets[f];
  int wmax = 1;
  for (int d = 0; d < L; ++d) {
    TFR_REQUIRE(cfg->hidden[d] >= 1 && cfg->hidden[d] <= kMaxH,
                "hidden width %d must be in [1, %d]", cfg->hidden[d], kMaxH);
    a.h[d] = cfg->hidden[d];
    if (a.h[d] > wmax) wmax = a.h[d];
  }
  a.h[L] = 1;
  const bool bn = cfg->use_batch_norm != 0 && L > 0;
  if (bn) {
    TFR_REQUIRE(cfg->bn_epsilon > 0.f, "bn_epsilon must be > 0");
    TFR_REQUIRE(cfg->bn_momentum >= 0.f && cfg->bn_momentum <= 1.f,
                "bn_momentum %g must be in [0, 1]", (double)cfg->bn_momentum);
  }
  p->F = F; p->L = L; p->C = C;
  p->wmax = wmax <= 16 ? 16 : wmax <= 32 ? 32 : 64;
  a.M = M; a.D = a.foff[F]; a.F = F; a.L = L;
  a.act = cfg->activation; a.use_bn = bn; a.training = cfg->training != 0;
  a.drop = L > 0 ? cfg->dropout : 0.f;
  a.scale = a.drop > 0.f ? 1.f / (1.f - a.drop) : 1.f;
  a.seed = cfg->dropout_seed;
  // parameter counts (tfr_mlp layout per tower)
  size_t rest = 0;                 // Dense 1..L
  for (int d = 1; d <= L; ++d) rest += (size_t)(a.h[d - 1] + 1) * a.h[d];
  int hsum = 0;
  for (int d = 0; d < L; ++d) hsum += a.h[d];
  a.pconst = (int)(a.h[0] + rest + (bn ? 2 * hsum : 0));
  p->ex_params = (size_t)a.foff[F] * a.h[0] + (size_t)F * a.pconst;
  a.ex_params = p->ex_params;
  p->tower_state = bn ? 2 * (size_t)hsum : 0;
  p->ex_state = (size_t)F * p->tower_state;
  {
    size_t o = 0;
    for (int d = 0; d < L; ++d) { a.bnst_off[d] = (int)o; o += 2 * (size_t)F * a.h[d]; }
  }
  // padded per-warp layout
  a.dfmax = dfmax;
  {
    int o = 0;
    for (int d = 0; d <= L; ++d) {
      const int K = d == 0 ? dfmax : a.h[d - 1];
      a.prow[d] = o;
      a.pcols[d] = pad4(a.h[d]);
      o += (K + 1) * a.pcols[d];
    }
    for (int d = 0; d < L; ++d) {
      a.pg[d] = o; o += pad4(a.h[d]);
      a.pb[d] = o; o += pad4(a.h[d]);
    }
    a.pp = pad4(o);
    int s = 0, nmax = 1;
    for (int d = 0; d <= L; ++d) {
      const int K = d == 0 ? dfmax : a.h[d - 1];
      a.sin[d] = s; s += pad4(K + 1);
      if (a.h[d] > nmax) nmax = a.h[d];
    }
    for (int d = 0; d < L; ++d)
      if (bn) { a.sxh[d] = s; s += pad4(a.h[d]); }
    a.sdz = s; s += pad4(nmax);
    a.sdy = s; s += bn ? pad4(nmax) : 0;
    if ((s / 4) % 2 == 0) s += 4;    // row stride = 4 * odd: conflict-free float4 rows
    a.ss = s;
  }
  // warps (= features) per CTA: as many as fit, up to 8
  int nw = 8;
  auto smem = [&](int w, int mode) {
    return (size_t)w * sizeof(float) *
           ((size_t)a.pp * (mode == GAM_GRAD ? 2 : 1) + (mode >= GAM_RED ? 32 * (size_t)a.ss : 0));
  };
  while (nw > 1 && smem(nw, GAM_GRAD) > kSmemBudget) --nw;
  TFR_REQUIRE(smem(nw, GAM_GRAD) <= kSmemBudget, "GAM towers too large for shared memory");
  a.nw = nw;
  p->smem_fwd = smem(nw, GAM_FWD);
  p->smem_bwd = smem(nw, GAM_RED);
  p->smem_grad = smem(nw, GAM_GRAD);
  {
    const int chunks = (F + nw - 1) / nw;
    const int target = (8 * num_sms() + chunks - 1) / chunks;
    int per = M > 0 ? (M + target - 1) / target : 32;
    per = (per + 31) / 32 * 32;
    a.rows_per = per;
    p->splits = M > 0 ? (M + per - 1) / per : 1;
  }
  // context towers
  size_t poff = p->ex_params, soff = p->ex_state;
  if (C > 0) {
    TFR_REQUIRE(F <= 8, "context towers need n_features <= 8 (got %d)", F);
    TFR_REQUIRE(cfg->n_context_hidden >= 0 && cfg->n_context_hidden < TFR_MLP_MAX_LAYERS,
                "n_context_hidden %d must be in [0, %d]", cfg->n_context_hidden,
                TFR_MLP_MAX_LAYERS - 1);
  }
  for (int j = 0; j < C; ++j) {
    tfr_mlp_cfg mc;
    std::memset(&mc, 0, sizeof(mc));
    mc.n_dense = cfg->n_context_hidden + 1;
    mc.dims[0] = cfg->context_dims[j];
    for (int d = 0; d < cfg->n_context_hidden; ++d) mc.dims[d + 1] = cfg->context_hidden[d];
    mc.dims[mc.n_dense] = F;
    mc.activation = cfg->activation;
    mc.use_batch_norm = cfg->use_batch_norm;
    mc.bn_epsilon = cfg->bn_epsilon;
    mc.bn_momentum = cfg->bn_momentum;
    mc.dropout = cfg->dropout;
    mc.training = cfg->training;
    mc.dropout_seed = cfg->dropout_seed + (unsigned long long)(j + 1) * 0xD1B54A32D192ED03ull;
    mc.bn_state = cfg->bn_state ? cfg->bn_state + soff : nullptr;
    int rc = make_mlp_plan(&mc, M, &p->ctx[j]);
    if (rc) return rc;
    p->ctx_param_off[j] = poff;
    poff += p->ctx[j].n_params;
    soff += p->ctx[j].n_state;
  }
  p->n_params = poff;
  p->n_state = soff;
  // workspace
  size_t w = 0;
  const size_t mf = (size_t)M * F;
  p->sub_off = w; w += al64(mf);
  p->ds_off = w; w += C ? al64(mf) : 0;
  p->cout_off = w; w += al64((size_t)C * mf);
  p->dctx_off = w; w += al64((size_t)C * mf);
  for (int j = 0; j < C; ++j) { p->cws_off[j] = w; w += al64(p->ctx[j].ws_floats); }
  p->bnstat_off = w; w += al64(2 * (size_t)F * hsum);
  p->coef_off = w; w += al64(2 * (size_t)F * hsum);
  p->spart_off = w; w += al64((size_t)p->splits * F * 2 * (size_t)(L ? wmax : 1));
  p->gpart_off = w; w += al64((size_t)p->splits * p->ex_params);
  p->ws_floats = w;
  return TFR_OK;
}

float* ws_base(void* workspace) {
  uintptr_t x = reinterpret_cast<uintptr_t>(workspace);
  x = (x + 255) & ~(uintptr_t)255;
  return reinterpret_cast<float*>(x);
}

template <int MODE>
int launch_sweep(const GamPlan& p, const GamArgs& a, cudaStream_t st) {
  const size_t smem = MODE == GAM_GRAD ? p.smem_grad : MODE == GAM_RED ? p.smem_bwd : p.smem_fwd;
  dim3 grid((p.F + a.nw - 1) / a.nw, p.splits);
  const int threads = 32 * a.nw;
#define TFR_GAM_LAUNCH(WM_)                                                               \
  {                                                                                       \
    TFR_CUDA_OK(cudaFuncSetAttribute(gam_sweep_kernel<WM_, MODE>,                         \
                                     cudaFuncAttributeMaxDynamicSharedMemorySize,         \
                                     (int)smem));                                         \
    gam_sweep_kernel<WM_, MODE><<<grid, threads, smem, st>>>(a);                          \
  }
  if (p.wmax == 16) TFR_GAM_LAUNCH(16)
  else if (p.wmax == 32) TFR_GAM_LAUNCH(32)
  else TFR_GAM_LAUNCH(64)
#undef TFR_GAM_LAUNCH
  TFR_LAUNCH_OK();
  return TFR_OK;
}

int check_call(const GamPlan& p, const tfr_gam_cfg* cfg, const float* const* ctx_host) {
  TFR_REQUIRE(!(p.a.use_bn || (p.C && cfg->use_batch_norm && cfg->n_context_hidden > 0)) ||
                  cfg->bn_state,
              "cfg->bn_state must be set with BN");
  if (ctx_host)
    for (int j = 0; j < p.C; ++j) TFR_REQUIRE(ctx_host[j], "context input %d is NULL", j);
  return TFR_OK;
}

}  // namespace

}  // namespace tfr

using namespace tfr;

extern "C" size_t tfr_gam_param_count(const tfr_gam_cfg* cfg) {
  static thread_local GamPlan p;
  if (make_gam_plan(cfg, 0, &p)) return 0;
  return p.n_params;
}

extern "C" size_t tfr_gam_bn_state_count(const tfr_gam_cfg* cfg) {
  static thread_local GamPlan p;
  if (make_gam_plan(cfg, 0, &p)) return 0;
  return p.n_state;
}

extern "C" size_t tfr_gam_workspace_bytes(const tfr_gam_cfg* cfg, int M) {
  static thread_local GamPlan p;
  if (make_gam_plan(cfg, M, &p)) return 0;
  return p.ws_floats * sizeof(float) + 256;
}

extern "C" int tfr_gam_fwd(const float* X, const float* const* ctx_host, int M,
                           const tfr_gam_cfg* cfg, const float* params, const uint8_t* mask,
                           void* workspace, float* logits, float* sublogits, float* subweights,
                           void* stream) {
  static thread_local GamPlan p;
  int rc = make_gam_plan(cfg, M, &p);
  if (rc) return rc;
  TFR_REQUIRE(X && params && workspace && logits, "NULL argument");
  rc = check_call(p, cfg, ctx_host);
  if (rc) return rc;
  if (M == 0) return TFR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = ws_base(workspace);
  const int C = ctx_host ? p.C : 0;
  GamArgs a = p.a;
  a.X = X;
  a.params = params;
  a.bnstat = ws + p.bnstat_off;
  a.part = ws + p.spart_off;
  for (int d = 0; d < p.L && a.use_bn; ++d) {
    const int n = a.h[d], total = p.F * n;
    float* stat = ws + p.bnstat_off + a.bnst_off[d];
    const int state_off = 2 * (int)(a.bnst_off[d] / (2 * p.F));   // 2 * sum_{e<d} h_e
    if (a.training) {
      a.layer = d;
      rc = launch_sweep<GAM_STATS>(p, a, st);
      if (rc) return rc;
      gam_stats_finalize_kernel<<<(total + 255) / 256, 256, 0, st>>>(
          a.part, p.splits, a.rows_per, M, p.F, n, cfg->bn_epsilon, cfg->bn_momentum, stat,
          cfg->bn_state, (int)p.tower_state, state_off);
    } else {
      gam_stats_from_moving_kernel<<<(total + 255) / 256, 256, 0, st>>>(
          cfg->bn_state, p.F, n, cfg->bn_epsilon, (int)p.tower_state, state_off, stat);
    }
    TFR_LAUNCH_OK();
  }
  a.sub = ws + p.sub_off;
  rc = launch_sweep<GAM_FWD>(p, a, st);
  if (rc) return rc;
  for (int j = 0; j < C; ++j) {
    rc = mlp_simt_fwd(ctx_host[j], M, p.ctx[j], params + p.ctx_param_off[j], nullptr,
                      ws + p.cws_off[j], ws + p.cout_off + (size_t)j * M * p.F, st);
    if (rc) return rc;
  }
  gam_combine_fwd_kernel<<<(M + 7) / 8, 256, 0, st>>>(ws + p.sub_off, ws + p.cout_off, C, M,
                                                      p.F, mask, logits, subweights);
  TFR_LAUNCH_OK();
  if (sublogits)
    TFR_CUDA_OK(cudaMemcpyAsync(sublogits, ws + p.sub_off, (size_t)M * p.F * sizeof(float),
                                cudaMemcpyDeviceToDevice, st));
  return TFR_OK;
}

extern "C" int tfr_gam_bwd(const float* X, const float* const* ctx_host, int M,
                           const tfr_gam_cfg* cfg, const float* params, const float* dlogits,
                           const uint8_t* mask, void* workspace, float* grads, void* stream) {
  static thread_local GamPlan p;
  int rc = make_gam_plan(cfg, M, &p);
  if (rc) return rc;
  TFR_REQUIRE(X && params && workspace && dlogits && grads, "NULL argument");
  rc = check_call(p, cfg, ctx_host);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (M == 0) {
    TFR_CUDA_OK(cudaMemsetAsync(grads, 0, p.n_params * sizeof(float), st));
    return TFR_OK;
  }
  float* ws = ws_base(workspace);
  const int C = ctx_host ? p.C : 0;
  GamArgs a = p.a;
  a.X = X;
  a.params = params;
  a.mask = mask;
  a.dlogits = dlogits;
  a.bnstat = ws + p.bnstat_off;
  a.coef = ws + p.coef_off;
  if (C > 0) {
    gam_combine_bwd_kernel<<<(M + 7) / 8, 256, 0, st>>>(ws + p.sub_off, ws + p.cout_off, C, M,
                                                        p.F, mask, dlogits, ws + p.ds_off,
                                                        ws + p.dctx_off);
    TFR_LAUNCH_OK();
    a.ds = ws + p.ds_off;
  }
  if (a.use_bn && a.training) {
    a.part = ws + p.spart_off;
    for (int d = p.L - 1; d >= 0; --d) {
      const int n = a.h[d], total = p.F * n;
      a.layer = d;
      rc = launch_sweep<GAM_RED>(p, a, st);
      if (rc) return rc;
      gam_red_finalize_kernel<<<(total + 255) / 256, 256, 0, st>>>(
          a.part, p.splits, M, p.F, n, ws + p.coef_off + a.bnst_off[d]);
      TFR_LAUNCH_OK();
    }
  }
  a.part = ws + p.gpart_off;
  rc = launch_sweep<GAM_GRAD>(p, a, st);
  if (rc) return rc;
  rc = mlp_reduce_partials(a.part, p.splits, p.ex_params, p.ex_params, grads, st);
  if (rc) return rc;
  for (int j = 0; j < p.C; ++j) {
    float* gj = grads + p.ctx_param_off[j];
    if (C == 0) {
      TFR_CUDA_OK(cudaMemsetAsync(gj, 0, p.ctx[j].n_params * sizeof(float), st));
      continue;
    }
    rc = mlp_simt_bwd(ctx_host[j], M, p.ctx[j], params + p.ctx_param_off[j],
                      ws + p.dctx_off + (size_t)j * M * p.F, nullptr, ws + p.cws_off[j], gj,
                      st);
    if (rc) return rc;
  }
  return TFR_OK;
}
