// K3c  Listwise losses outside RankingLossKey's Keras subset that SURVEY.md §8(f1) names:
//   CircleLoss                  losses_impl.py:1036-1116   O(N^2) pair exponentials + log1p
//   NeuralSortCrossEntropyLoss  losses_impl.py:1635-1675   N x N softmax rows (NeuralSort)
//   NeuralSortNDCGLoss          losses_impl.py:1678-1708   PiRank NDCG on the same rows
// One CTA per list, a thread per item / per relaxed-permutation row; the N x N matrices of
// the reference (pair logits, permutation matrices) are never formed: rows are re-evaluated
// from O(N) per-row statistics kept in shared memory.
#include "common.cuh"
#include "loss_common.cuh"

namespace tfr {

namespace {

__device__ __forceinline__ float sgn(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); }

// ---------------------------------------------------------------------------
// Circle:  L = log1p( sum_{i, j valid, l_i > l_j} exp(gamma (a_i + c_j)) ),
//   s = clip(score, 0, 1), a_i = relu(1 - s_i + m)(1 - s_i - m), c_j = relu(s_j + m)(s_j - m);
//   the relu factors carry no gradient (stop_gradient, :1090-1093).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kLossThreads)
circle_loss_kernel(const float* __restrict__ scores, const float* __restrict__ labels,
                   const float* __restrict__ item_w, int w_per_item,
                   const uint8_t* __restrict__ mask, int N, float gamma, float margin,
                   float grad_scale, float* __restrict__ grad, float* __restrict__ loss,
                   float* __restrict__ weight) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const ListView v = carve(smem_raw, N);
  const int b = blockIdx.x, tid = threadIdx.x;
  load_list(v, scores, labels, item_w, w_per_item, mask, b, N, 1.f);
  const size_t off = (size_t)b * N;
  float* a = v.g;        // positive-side exponent / gamma
  float* c = v.disc;     // negative-side exponent / gamma
  float wl = 0.f, lvsum = 0.f;
  for (int i = tid; i < N; i += blockDim.x) {
    const float s = fminf(fmaxf(v.z[i], 0.f), 1.f);
    a[i] = fmaxf(1.f - s + margin, 0.f) * (1.f - s - margin);
    c[i] = fmaxf(s + margin, 0.f) * (s - margin);
    const float lv = v.lv[i] ? v.l[i] : 0.f;
    wl += v.w[i] * lv;
    lvsum += lv;
  }
  wl = block_sum(wl, v.red);
  lvsum = block_sum(lvsum, v.red);   // (barriers publish a / c)
  const float list_w = item_w ? (lvsum != 0.f ? wl / lvsum : 0.f) : 1.f;
  float S = 0.f, pairs = 0.f;
  float* spos = v.w;                               // free after list_w
  float* sneg = reinterpret_cast<float*>(v.rank);
  for (int i = tid; i < N; i += blockDim.x) {
    const float li = v.l[i], ai = a[i], ci = c[i];
    const bool vi = v.mv[i];
    float sp = 0.f, sn = 0.f, cnt = 0.f;
    for (int j = 0; j < N; ++j) {
      const bool vj = vi && v.mv[j];
      const float lj = v.l[j];
      if (vj && li > lj) {
        sp += expf(gamma * (ai + c[j]));
        cnt += 1.f;
      } else if (vj && lj > li) {
        sn += expf(gamma * (a[j] + ci));
      }
    }
    spos[i] = sp;
    sneg[i] = sn;
    S += sp;
    pairs += cnt;
  }
  S = block_sum(S, v.red);
  pairs = block_sum(pairs, v.red);
  if (grad) {
    const float inv = grad_scale * gamma / (1.f + S);
    for (int i = tid; i < N; i += blockDim.x) {
      const float raw = v.z[i];
      const float s = fminf(fmaxf(raw, 0.f), 1.f);
      const bool pass = raw >= 0.f && raw <= 1.f;   // clip_by_value passes the closed interval
      const float g = -fmaxf(1.f - s + margin, 0.f) * spos[i] + fmaxf(s + margin, 0.f) * sneg[i];
      grad[off + i] = (pass && v.mv[i]) ? g * inv : 0.f;
    }
  }
  if (tid == 0) {
    loss[b] = log1pf(S);
    // :1108-1110  sum(w) / count(w > 0): 0 / 0 = NaN for a list without a pair, as the reference
    if (weight) weight[b] = list_w * (pairs / pairs);
  }
}

// ---------------------------------------------------------------------------
// NeuralSort.  Row of the relaxed permutation that belongs to the r-th valid item (in list
// order): u_k = c_r x_k - D_k over valid k, c_r = n_valid - 1 - 2 r, D_k = sum_j |x_k - x_j|;
// P[r, :] = softmax(u).  MODE 0: cross entropy against the same construction on the labels;
// MODE 1: - sum_r disc(r + 1) sum_k P[r, k] gain_k / maxDCG.
// c_r x_k and D_k grow with N (to ~4e4 at N = 4000 for unit-scale scores) while the softmax
// only sees u_k - max_k u_k, which is O(1) where P is not 0 or 1: in fp32 the exponent would
// carry ~1 ulp(4e4) = 4e-3 of rounding error.  D is therefore accumulated in fp64 and every
// exponent c_r x_k - D_k - max is formed in fp64 (exact product and difference of fp32 inputs)
// before the fp32 expf.
// ---------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(kLossThreads)
neural_sort_loss_kernel(const float* __restrict__ scores, const float* __restrict__ labels,
                        const float* __restrict__ item_w, int w_per_item,
                        const uint8_t* __restrict__ mask, int N, float temperature,
                        float grad_scale, float* __restrict__ grad, float* __restrict__ loss,
                        float* __restrict__ weight) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const ListView v = carve(smem_raw, N);
  float* ext = reinterpret_cast<float*>(smem_raw + ((list_smem_bytes(N) + 15) & ~(size_t)15));
  double* D = reinterpret_cast<double*>(ext);   // [N] sum_j |s_k - s_j| (fp64: see above)
  float* DL = ext + 2 * N;   // [N] same on the labels (MODE 0) / gains (MODE 1)
  float* rmx = ext + 3 * N;  // [N] row max of u
  float* rZ = ext + 4 * N;   // [N] row sum of exp(u - max)
  float* tmx = ext + 5 * N;  // [N] (MODE 0) the same for the label rows
  float* tZ = ext + 6 * N;
  float* rA = ext + 7 * N;   // [N] sum_k g[r, k] P[r, k]
  float* H = v.g;            // [N] column sums of G
  float* C = v.disc;         // [N] column sums of c_r G
  int* cum = v.rank;         // [N] 1-based index among the valid items
  const int b = blockIdx.x, tid = threadIdx.x;
  load_list(v, scores, labels, item_w, w_per_item, mask, b, N, temperature);
  const size_t off = (size_t)b * N;

  // cleaned labels / logits, list weight (:1004-1015), label sum, label max
  float wl = 0.f, lvsum = 0.f, lsum = 0.f, lmax = -CUDART_INF_F;
  for (int i = tid; i < N; i += blockDim.x) {
    const bool ok = v.mv[i];
    const float lv = v.lv[i] ? v.l[i] : 0.f;
    wl += v.w[i] * lv;
    lvsum += lv;
    if (!ok) {
      v.z[i] = 0.f;
      v.l[i] = 0.f;
    }
    lsum += v.l[i];
    lmax = fmaxf(lmax, v.l[i]);
  }
  wl = block_sum(wl, v.red);
  lvsum = block_sum(lvsum, v.red);
  lsum = block_sum(lsum, v.red);
  lmax = block_max(lmax, v.red);
  const float list_w = item_w ? (lvsum != 0.f ? wl / lvsum : 0.f) : 1.f;
  const bool nonzero = lsum > 0.f;
  // valid-item index (serial prefix count: N <= 8192 byte reads from smem)
  for (int i = tid; i < N; i += blockDim.x) {
    int cnt = 0;
    for (int j = 0; j <= i; ++j) cnt += v.mv[j];
    cum[i] = cnt;
  }
  __syncthreads();
  int nv = 0;
  if (N > 0) nv = cum[N - 1];
  if (nv == 0 || (MODE == 1 && !nonzero)) {
    // MODE 1 without a positive label: every gain is 2^0 - 2^-1e-10 = 0 in fp32
    for (int i = tid; i < N; i += blockDim.x)
      if (grad) grad[off + i] = 0.f;
    if (tid == 0) {
      loss[b] = 0.f;
      if (weight) weight[b] = nonzero ? list_w : 0.f;
    }
    return;
  }
  float* gain = DL;   // MODE 1: safe default gains (losses_impl.py:33-49)
  for (int k = tid; k < N; k += blockDim.x) {
    const float sk = v.z[k], lk = v.l[k];
    double d = 0.0;
    float dl = 0.f;
    if (v.mv[k]) {
      for (int j = 0; j < N; ++j)
        if (v.mv[j]) {
          d += fabs((double)sk - (double)v.z[j]);
          dl += fabsf(lk - v.l[j]);
        }
    }
    D[k] = d;
    if (MODE == 0) DL[k] = dl;
    else gain[k] = exp2f(lk - lmax) - exp2f(-lmax);
  }
  __syncthreads();
  // c_r of the row owned by item i, and the fp64 exponent of entry (row c, column k)
  auto rc = [&](int i) { return (float)(nv + 1 - 2 * cum[i]); };
  auto u_of = [&](float c, int k, float mx) {
    return (float)((double)c * (double)v.z[k] - D[k] - (double)mx);
  };
  auto t_of = [&](float c, int k, float mt) {
    return (float)((double)c * (double)v.l[k] - (double)DL[k] - (double)mt);
  };
  float inv_max_dcg = 0.f;
  if (MODE == 1) {
    // ideal DCG of the safe gains (all N cleaned labels, discount 1 / log1p(rank))
    const float ideal = ideal_dcg(v.l, gain, N, N, v.red,
                                  [](int r) { return 1.f / log1pf((float)r); });
    inv_max_dcg = ideal > 0.f ? 1.f / ideal : 0.f;
  }
  const float inv_nv = 1.f / (float)nv;

  // pass 1 (thread per row): softmax statistics of the score row (and the label row)
  for (int i = tid; i < N; i += blockDim.x) {
    if (!v.mv[i]) continue;
    const float c = rc(i);
    float mx = -CUDART_INF_F, mt = -CUDART_INF_F;
    for (int k = 0; k < N; ++k)
      if (v.mv[k]) {
        mx = fmaxf(mx, u_of(c, k, 0.f));
        if (MODE == 0) mt = fmaxf(mt, t_of(c, k, 0.f));
      }
    float Z = 0.f, Zt = 0.f;
    for (int k = 0; k < N; ++k)
      if (v.mv[k]) {
        Z += expf(u_of(c, k, mx));
        if (MODE == 0) Zt += expf(t_of(c, k, mt));
      }
    rmx[i] = mx;
    rZ[i] = Z;
    if (MODE == 0) {
      tmx[i] = mt;
      tZ[i] = Zt;
    }
  }
  __syncthreads();
  // pass 2 (thread per row): the row's loss term and A_r = sum_k g[r, k] P[r, k], where
  // g = d loss / d P:  MODE 0: -T / (n_valid (1e-20 + P));  MODE 1: -disc_r gain_k / maxDCG
  float part = 0.f;
  for (int i = tid; i < N; i += blockDim.x) {
    if (!v.mv[i]) continue;
    const float c = rc(i), mx = rmx[i], iz = 1.f / rZ[i];
    float A = 0.f, term = 0.f;
    if (MODE == 0) {
      const float mt = tmx[i], izt = 1.f / tZ[i];
      for (int k = 0; k < N; ++k)
        if (v.mv[k]) {
          const float P = expf(u_of(c, k, mx)) * iz;
          const float T = expf(t_of(c, k, mt)) * izt;
          term -= T * logf(1e-20f + P);
          A -= T * P / (1e-20f + P);
        }
      // log_softmax of log(1e-20 + P) over ALL N columns subtracts log(1 + N 1e-20) = 0 in fp32
      part += term * inv_nv;
      A *= inv_nv;
    } else {
      const float disc = 1.f / log1pf((float)cum[i]);
      float gs = 0.f;
      for (int k = 0; k < N; ++k)
        if (v.mv[k]) gs += expf(u_of(c, k, mx)) * iz * gain[k];
      part -= disc * gs * inv_max_dcg;
      A = -disc * inv_max_dcg * gs;
    }
    rA[i] = A;
  }
  part = block_sum(part, v.red);   // barrier publishes rA
  if (grad) {
    // pass 3 (thread per column): H_k = sum_r G[r, k], C_k = sum_r c_r G[r, k],
    //   G = P (g - A_r)   (softmax backward)
    for (int k = tid; k < N; k += blockDim.x) {
      float h = 0.f, cc = 0.f;
      if (v.mv[k]) {
        for (int i = 0; i < N; ++i) {
          if (!v.mv[i]) continue;
          const float c = rc(i);
          const float P = expf(u_of(c, k, rmx[i])) / rZ[i];
          float g;
          if (MODE == 0) {
            const float T = expf(t_of(c, k, tmx[i])) / tZ[i];
            g = -T * inv_nv / (1e-20f + P);
          } else {
            g = -inv_max_dcg * gain[k] / log1pf((float)cum[i]);
          }
          const float G = P * (g - rA[i]);
          h += G;
          cc += c * G;
        }
      }
      H[k] = h;
      C[k] = cc;
    }
    __syncthreads();
    // pass 4: u[r, k] = c_r s_k - D_k, dD_k / ds_m = [k == m] sum_j sign(s_k - s_j) - sign(s_k - s_m)
    const float gs = grad_scale / temperature;
    for (int m = tid; m < N; m += blockDim.x) {
      float g = 0.f;
      if (v.mv[m]) {
        const float sm_ = v.z[m];
        float sg = 0.f, cross = 0.f;
        for (int j = 0; j < N; ++j)
          if (v.mv[j]) {
            const float sd = sgn(sm_ - v.z[j]);
            sg += sd;
            cross -= H[j] * sd;       // H_j sign(s_j - s_m)
          }
        g = C[m] - H[m] * sg + cross;
      }
      grad[off + m] = g * gs;
    }
  }
  if (tid == 0) {
    loss[b] = part;
    if (weight) weight[b] = nonzero ? list_w : 0.f;
  }
}

}  // namespace

}  // namespace tfr

using namespace tfr;

extern "C" int tfr_extra_loss_fwd_bwd(const float* scores, const float* labels,
                                      const float* item_w, int w_per_item, const uint8_t* mask,
                                      int B, int N, float temperature, int kind, float p0,
                                      float p1, float grad_scale, float* grad, float* loss,
                                      float* weight, void* stream) {
  TFR_REQUIRE(scores && labels && loss, "scores / labels / loss must not be NULL");
  TFR_REQUIRE(B >= 0 && N >= 1 && N <= kMaxListSize, "bad shape B=%d N=%d", B, N);
  TFR_REQUIRE(temperature > 0.f, "temperature must be positive");
  TFR_REQUIRE(kind >= TFR_EXTRA_CIRCLE && kind <= TFR_EXTRA_NEURAL_SORT_NDCG,
              "kind %d is not a tfr_extra_loss", kind);
  if (B == 0) return TFR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t base = (list_smem_bytes(N) + 15) & ~(size_t)15;
  if (kind == TFR_EXTRA_CIRCLE) {
    TFR_CUDA_OK(cudaFuncSetAttribute(circle_loss_kernel,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)base));
    circle_loss_kernel<<<B, kLossThreads, base, st>>>(scores, labels, item_w, w_per_item, mask, N,
                                                      p0, p1, grad_scale, grad, loss, weight);
  } else {
    auto bytes_for = [](int n) {
      return ((list_smem_bytes(n) + 15) & ~(size_t)15) + (size_t)8 * n * sizeof(float);
    };
    const size_t smem = bytes_for(N), limit = smem_optin_limit();
    if (smem > limit) {
      int n_max = N;
      while (n_max >= 1 && bytes_for(n_max) > limit) --n_max;
      TFR_REQUIRE(false,
                  "NeuralSort: list_size %d needs %zu bytes of shared memory per block but the "
                  "device allows %zu; the largest list_size accepted is %d",
                  N, smem, limit, n_max);
    }
    if (kind == TFR_EXTRA_NEURAL_SORT_CE) {
      TFR_CUDA_OK(cudaFuncSetAttribute(neural_sort_loss_kernel<0>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      neural_sort_loss_kernel<0><<<B, kLossThreads, smem, st>>>(
          scores, labels, item_w, w_per_item, mask, N, temperature, grad_scale, grad, loss, weight);
    } else {
      TFR_CUDA_OK(cudaFuncSetAttribute(neural_sort_loss_kernel<1>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      neural_sort_loss_kernel<1><<<B, kLossThreads, smem, st>>>(
          scores, labels, item_w, w_per_item, mask, N, temperature, grad_scale, grad, loss, weight);
    }
  }
  TFR_LAUNCH_OK();
  return TFR_OK;
}
