// K3d  Click-model losses (losses_impl.py:1324-1422, 1472-1538):
//   ClickEMLoss    examination x relevance click model (Wang et al. 2018), pointwise
//   MixtureEMLoss  mixture of click models (Yan et al. 2022), listwise
// One CTA per list, forward and backward in the same launch; every sum runs in a fixed
// order (no float atomics), so two identical calls give identical bits.
#include "common.cuh"
#include "loss_common.cuh"

namespace tfr {

namespace {

// Stable forms: no exp of a positive argument, so logits of +-1e4 stay finite.
__device__ __forceinline__ float log1p_exp_neg_abs(float x) { return log1pf(expf(-fabsf(x))); }
__device__ __forceinline__ float softplus(float x) { return fmaxf(x, 0.f) + log1p_exp_neg_abs(x); }
__device__ __forceinline__ float sigmoid(float x) {
  const float e = expf(-fabsf(x));
  return x >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
}
// tf.nn.sigmoid_cross_entropy_with_logits(labels = z, logits = x)
__device__ __forceinline__ float sce(float z, float x) {
  return fmaxf(x, 0.f) - x * z + log1p_exp_neg_abs(x);
}

// ---------------------------------------------------------------------------
// Click EM.  Item i of list b reads e = exam[(b N + i) stride], r = rel[(b N + i) stride]
// and writes its gradients at the same offsets of d_exam / d_rel.  The posteriors
//   pe = P(exam | no click) = sigmoid(e - softplus(r)),  pr = sigmoid(r - softplus(e))
// are 1 for a clicked item and carry no gradient (stop_gradient, :1390-1391).
// ---------------------------------------------------------------------------
__global__ void click_em_kernel(const float* __restrict__ exam, const float* __restrict__ rel,
                                int stride, const float* __restrict__ labels,
                                const float* __restrict__ item_w, int w_per_item,
                                const uint8_t* __restrict__ mask, int N, float inv_t,
                                float exam_w, float rel_w, float gs, float* __restrict__ d_exam,
                                float* __restrict__ d_rel, float* __restrict__ row,
                                float* __restrict__ loss, float* __restrict__ weight,
                                float* __restrict__ nonzero) {
  __shared__ float red[32];
  const int b = blockIdx.x, tid = threadIdx.x;
  const size_t off = (size_t)b * N;
  float sl = 0.f, sw = 0.f, nz = 0.f;
  for (int i = tid; i < N; i += blockDim.x) {
    const size_t k = off + i;
    const float lab = labels[k];
    const bool lvalid = lab >= 0.f;
    const bool mvalid = mask ? (mask[k] != 0) : lvalid;
    float wv = 1.f;
    if (item_w) wv = w_per_item ? item_w[k] : item_w[b];
    // normalised item weight (:1287-1293) x the loss weight, which is the mask (:1422)
    const float w = (lvalid && mvalid) ? wv : 0.f;
    const bool clicked = mvalid && lab >= 1.f;
    const float e = mvalid ? exam[k * stride] * inv_t : 0.f;
    const float r = mvalid ? rel[k * stride] * inv_t : 0.f;
    const float pe = clicked ? 1.f : sigmoid(e - softplus(r));
    const float pr = clicked ? 1.f : sigmoid(r - softplus(e));
    const float f = exam_w * sce(pe, e) + rel_w * sce(pr, r);
    if (row) row[k] = f * w;
    if (d_exam) {
      const float gw = w * gs;   // w = 0 on invalid items: an exact 0 gradient
      d_exam[k * stride] = gw != 0.f ? exam_w * (sigmoid(e) - pe) * gw : 0.f;
      d_rel[k * stride] = gw != 0.f ? rel_w * (sigmoid(r) - pr) * gw : 0.f;
    }
    sl += f * w;
    sw += w;
    nz += w != 0.f ? 1.f : 0.f;
  }
  sl = block_sum(sl, red);
  sw = block_sum(sw, red);
  nz = block_sum(nz, red);
  if (tid == 0) {
    loss[b] = sl;
    if (weight) weight[b] = sw;
    if (nonzero) nonzero[b] = nz;
  }
}

// ---------------------------------------------------------------------------
// Mixture EM.  scores [B, N, M]; per list
//   L_m = sum_i sce(l_i, s_im / T) over valid items (l_i = 0 elsewhere),
//   q_m = exp(-alpha (L_m - min_k L_k)) (no gradient), loss = sum_m q_m L_m / sum_m q_m,
//   weight = list weight (:1004-1015) x [sum of the valid labels > 0].
// A warp step covers P = 32 / M whole items with lane l on model l % M, so the [N, M] rows
// are read coalesced for every M and each lane only ever sums one model's terms.  L_m is
// accumulated in fp64: q_m depends on differences of L that grow with N, and alpha scales
// their rounding error into the exponent.
// ---------------------------------------------------------------------------
constexpr int kMixThreads = 256;

__global__ void __launch_bounds__(kMixThreads)
mixture_em_kernel(const float* __restrict__ scores, const float* __restrict__ labels,
                  const float* __restrict__ item_w, int w_per_item,
                  const uint8_t* __restrict__ mask, int N, int M, float inv_t, float alpha,
                  float gs, float* __restrict__ grad, float* __restrict__ loss,
                  float* __restrict__ weight) {
  __shared__ double part[kMixThreads];
  __shared__ double Ls[32];
  __shared__ float qn[32];
  __shared__ float red[32];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const size_t off = (size_t)b * N;

  // list weight (sum w l / sum l over label-valid items) and the sum of the valid labels
  float wl = 0.f, lvsum = 0.f, lsum = 0.f;
  for (int i = tid; i < N; i += blockDim.x) {
    const float lab = labels[off + i];
    const bool lvalid = lab >= 0.f;
    const bool mvalid = mask ? (mask[off + i] != 0) : lvalid;
    const float lv = lvalid ? lab : 0.f;
    float wv = 1.f;
    if (item_w) wv = w_per_item ? item_w[off + i] : item_w[b];
    wl += wv * lv;
    lvsum += lv;
    lsum += mvalid ? lab : 0.f;
  }
  wl = block_sum(wl, red);
  lvsum = block_sum(lvsum, red);
  lsum = block_sum(lsum, red);
  const float list_w = item_w ? (lvsum != 0.f ? wl / lvsum : 0.f) : 1.f;

  const int P = 32 / M;
  double acc = 0.0;
  if (lane < P * M) {
    const int sub = lane / M, m = lane - sub * M;
    for (int i = warp * P + sub; i < N; i += nwarps * P) {
      const float lab = labels[off + i];
      const bool mvalid = mask ? (mask[off + i] != 0) : lab >= 0.f;
      if (mvalid) acc += (double)sce(lab, scores[(off + i) * M + m] * inv_t);
    }
  }
  part[tid] = acc;
  __syncthreads();
  if (tid < M) {
    double L = 0.0;
    for (int w = 0; w < nwarps; ++w)
      for (int s = 0; s < P; ++s) L += part[w * 32 + s * M + tid];
    Ls[tid] = L;
  }
  __syncthreads();
  if (warp == 0) {
    double mn = lane < M ? Ls[lane] : INFINITY;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    const float L = lane < M ? (float)Ls[lane] : 0.f;
    const float q = lane < M ? expf(-alpha * (float)(Ls[lane] - mn)) : 0.f;
    // lane 0's butterfly result is the one every lane uses
    const float sq = __shfl_sync(0xffffffffu, warp_sum(q), 0);
    const float sql = __shfl_sync(0xffffffffu, warp_sum(q * L), 0);
    if (lane < M) qn[lane] = q / sq;
    if (lane == 0) {
      loss[b] = sql / sq;
      if (weight) weight[b] = lsum > 0.f ? list_w : 0.f;
    }
  }
  __syncthreads();
  if (grad) {
    const int nm = N * M;
    for (int e = tid; e < nm; e += blockDim.x) {
      const int i = e / M, m = e - i * M;
      const float lab = labels[off + i];
      const bool mvalid = mask ? (mask[off + i] != 0) : lab >= 0.f;
      float g = 0.f;
      if (mvalid) g = qn[m] * (sigmoid(scores[off * M + e] * inv_t) - lab) * gs;
      grad[off * M + e] = g;
    }
  }
}

}  // namespace

}  // namespace tfr

using namespace tfr;

extern "C" int tfr_click_em_loss_fwd_bwd(const float* exam, const float* rel, int stride,
                                         const float* labels, const float* item_w,
                                         int w_per_item, const uint8_t* mask, int B, int N,
                                         float temperature, float exam_weight, float rel_weight,
                                         float grad_scale, float* d_exam, float* d_rel,
                                         float* row, float* loss, float* weight, float* nonzero,
                                         void* stream) {
  TFR_REQUIRE(exam && rel && labels && loss, "exam / rel / labels / loss must not be NULL");
  TFR_REQUIRE((d_exam == nullptr) == (d_rel == nullptr),
              "d_exam and d_rel are both given or both NULL");
  TFR_REQUIRE(stride == 1 || stride == 2, "stride %d must be 1 or 2", stride);
  TFR_REQUIRE(B >= 0 && N >= 1 && N <= kMaxListSize, "bad shape B=%d N=%d (1 <= N <= %d)", B,
              N, kMaxListSize);
  TFR_REQUIRE(temperature > 0.f, "temperature must be positive");
  if (B == 0) return TFR_OK;
  const int threads = N >= kLossThreads ? kLossThreads : ((N + 31) / 32) * 32;
  click_em_kernel<<<B, threads, 0, (cudaStream_t)stream>>>(
      exam, rel, stride, labels, item_w, w_per_item, mask, N, 1.f / temperature, exam_weight,
      rel_weight, grad_scale / temperature, d_exam, d_rel, row, loss, weight, nonzero);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

extern "C" int tfr_mixture_em_loss_fwd_bwd(const float* scores, const float* labels,
                                           const float* item_w, int w_per_item,
                                           const uint8_t* mask, int B, int N, int M,
                                           float temperature, float alpha, float grad_scale,
                                           float* grad, float* loss, float* weight,
                                           void* stream) {
  TFR_REQUIRE(scores && labels && loss, "scores / labels / loss must not be NULL");
  TFR_REQUIRE(B >= 0 && N >= 1 && N <= kMaxListSize, "bad shape B=%d N=%d (1 <= N <= %d)", B,
              N, kMaxListSize);
  TFR_REQUIRE(M >= 1 && M <= 32, "model_num %d must be in 1..32", M);
  TFR_REQUIRE(temperature > 0.f, "temperature must be positive");
  if (B == 0) return TFR_OK;
  mixture_em_kernel<<<B, kMixThreads, 0, (cudaStream_t)stream>>>(
      scores, labels, item_w, w_per_item, mask, N, M, 1.f / temperature, alpha,
      grad_scale / temperature, grad, loss, weight);
  TFR_LAUNCH_OK();
  return TFR_OK;
}
