// K4: NDCG@k / MRR@k for several cut-offs in one launch.
//
// One CTA per list.  The list is ordered with an in-shared-memory bitonic sort of
// 64-bit keys (valid-first | score descending | original index), which makes the
// order exactly "valid items by score, ties by index, invalid last" — the
// reference's sort_by_scores(..., mask) with shuffle_ties=False (utils.py:115-164).
// A second sort by weight*gain gives the ideal ordering (metrics_impl.py:660-665).
#include <math_constants.h>

#include "common.cuh"

namespace tfr {

constexpr int kMetricThreads = 256;
constexpr int kMaxMetricListSize = 8192;
constexpr int kMaxTopn = 16;

struct TopnList {
  int n;
  int v[kMaxTopn];
};

__device__ __forceinline__ uint32_t desc_bits(float x) {
  if (x == 0.f) x = 0.f;  // -0 == +0
  uint32_t u = __float_as_uint(x);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // ascending-order preserving
  return ~u;                                        // descending
}

__device__ __forceinline__ float sc_clean(bool ok, float s, float pmin) {
  return ok ? s : (-1e-6f + pmin);   // metrics_impl.py:262-265
}

__device__ inline void bitonic_sort(unsigned long long* keys, int P) {
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int idx = threadIdx.x; idx < P; idx += blockDim.x) {
        const int ixj = idx ^ j;
        if (ixj > idx) {
          const bool asc = (idx & k) == 0;
          const unsigned long long a = keys[idx], c = keys[ixj];
          if ((a > c) == asc) {
            keys[idx] = c;
            keys[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  }
}

struct MetricExt {   // device copy of tfr_metric_ext (all optional)
  float *dcg, *precision, *recall, *map, *hits, *arp, *opa, *bpref, *bpref_alt;
  __host__ __device__ bool any() const {
    return dcg || precision || recall || map || hits || arp || opa || bpref || bpref_alt;
  }
};

// Inclusive prefix sums of a[0..N) in place (chunk per thread + serial chunk totals).
__device__ inline void block_inclusive_scan(float* a, int N, float* scratch /*[blockDim.x]*/) {
  const int tid = threadIdx.x, nt = blockDim.x;
  const int per = (N + nt - 1) / nt;
  const int beg = min(N, tid * per), end = min(N, beg + per);
  float s = 0.f;
  for (int i = beg; i < end; ++i) s += a[i];
  scratch[tid] = s;
  __syncthreads();
  if (tid == 0) {
    float run = 0.f;
    for (int t = 0; t < nt; ++t) {
      const float x = scratch[t];
      scratch[t] = run;
      run += x;
    }
  }
  __syncthreads();
  float run = scratch[tid];
  for (int i = beg; i < end; ++i) {
    run += a[i];
    a[i] = run;
  }
  __syncthreads();
}

// raw[b, 0..4] = {sum w, sum w*gain, sum gain, sum w*rel, sum rel}, rel = [label >= 1]
__global__ void __launch_bounds__(kMetricThreads)
rank_metrics_kernel(const float* __restrict__ scores, const float* __restrict__ labels,
                    const float* __restrict__ item_w, int w_per_item,
                    const uint8_t* __restrict__ mask, int N, int P, TopnList topns,
                    int gain_fn, int disc_fn, const float* __restrict__ gain_table,
                    const float* __restrict__ disc_table, float* __restrict__ ndcg,
                    float* __restrict__ mrr, float* __restrict__ raw, MetricExt ext) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw);
  float* cl = reinterpret_cast<float*>(keys + P);  // cleaned labels
  float* w = cl + N;                                // example weights
  float* wg = w + N;                                // weight * gain
  float* term = wg + N;                             // per-position DCG terms
  float* red = term + N;                            // [32]
  unsigned char* valid = reinterpret_cast<unsigned char*>(red + 32);
  // extended metrics only: scan scratch.  Sorted relevance and weights are read through the
  // sort keys, and OPA's cleaned scores go to `term` once it is free, so that every output
  // fits shared memory up to kMaxMetricListSize (rank_metrics_smem_bytes).
  float* scratch = reinterpret_cast<float*>(
      smem_raw + (((size_t)P * 8 + (size_t)(4 * N + 32) * 4 + N + 15) & ~(size_t)15));
  const bool want_ext = ext.any();

  const int b = blockIdx.x, tid = threadIdx.x;
  const size_t off = (size_t)b * N;

  // metrics_impl.py:228-266: mask &= w > 0; labels := 0, preds := min - 1e-6 where masked out
  float pmin = CUDART_INF_F;
  for (int i = tid; i < N; i += blockDim.x) pmin = fminf(pmin, scores[off + i]);
  pmin = block_min(pmin, red);
  float s_w = 0.f, s_wg = 0.f, s_g = 0.f, s_wr = 0.f, s_r = 0.f;
  for (int i = tid; i < N; i += blockDim.x) {
    const float lab = labels[off + i];
    float wv = 1.f;
    if (item_w) wv = w_per_item ? item_w[off + i] : item_w[b];
    bool ok = mask ? (mask[off + i] != 0) : (lab >= 0.f);
    ok = ok && (wv > 0.f);
    const float c = ok ? lab : 0.f;
    const float g = gain_fn == TFR_GAIN_TABLE ? gain_table[off + i] : gain_of(gain_fn, c);
    const float sc_i = sc_clean(ok, scores[off + i], pmin);
    cl[i] = c;
    w[i] = wv;
    wg[i] = wv * g;
    valid[i] = ok;
    keys[i] = ((unsigned long long)(ok ? 0 : 1) << 45) |
              ((unsigned long long)desc_bits(sc_i) << 13) | (unsigned long long)i;
    const float rel = c >= 1.f ? 1.f : 0.f;
    s_w += wv;
    s_wg += wv * g;
    s_g += g;
    s_wr += wv * rel;
    s_r += rel;
  }
  for (int i = N + tid; i < P; i += blockDim.x) keys[i] = ~0ull;
  s_w = block_sum(s_w, red);
  s_wg = block_sum(s_wg, red);
  s_g = block_sum(s_g, red);
  s_wr = block_sum(s_wr, red);
  s_r = block_sum(s_r, red);
  if (tid == 0 && raw) {
    raw[b * 5 + 0] = s_w;
    raw[b * 5 + 1] = s_wg;
    raw[b * 5 + 2] = s_g;
    raw[b * 5 + 3] = s_wr;
    raw[b * 5 + 4] = s_r;
  }
  __syncthreads();
  bitonic_sort(keys, P);

  // DCG terms by position and first relevant position (MRR).
  int first_rel = 0x7fffffff;
  for (int k = tid; k < N; k += blockDim.x) {
    const int idx = (int)(keys[k] & 0x1fffull);
    const float d = disc_fn == TFR_DISC_TABLE ? disc_table[k + 1] : disc_of(disc_fn, (float)(k + 1));
    term[k] = wg[idx] * d;
    if (cl[idx] >= 1.f) first_rel = min(first_rel, k);
  }
  {
    float fr = block_min((float)min(first_rel, 1 << 24), red);
    first_rel = (int)fr;
  }
  float dcg[kMaxTopn];
  for (int t = 0; t < topns.n; ++t) {
    const int cut = topns.v[t] > 0 ? min(topns.v[t], N) : N;
    float acc = 0.f;
    for (int k = tid; k < cut; k += blockDim.x) acc += term[k];
    dcg[t] = block_sum(acc, red);
    if (tid == 0 && mrr)
      mrr[(size_t)b * topns.n + t] = first_rel < cut ? 1.f / (float)(first_rel + 1) : 0.f;
  }
  if (want_ext) {
    // ---- metrics that share the score order (metrics_impl.py:154-207, 462-744) ----
    __syncthreads();
    float nv = 0.f, a_num = 0.f, a_den = 0.f;
    for (int k = tid; k < N; k += blockDim.x) {
      const int idx = (int)(keys[k] & 0x1fffull);
      const float c = cl[idx];
      term[k] = c >= 1.f ? 1.f : 0.f;    // -> cumulative relevant count
      nv += valid[k] ? 1.f : 0.f;
      a_num += (float)(k + 1) * w[idx] * c;      // ARP (:524-536)
      a_den += w[idx] * c;
    }
    nv = block_sum(nv, red);
    a_num = block_sum(a_num, red);
    a_den = block_sum(a_den, red);
    if (tid == 0 && ext.arp) {
      ext.arp[b * 2 + 0] = a_den != 0.f ? a_num / a_den : 0.f;
      ext.arp[b * 2 + 1] = a_den;
    }
    block_inclusive_scan(term, N, scratch);
    for (int t = 0; t < topns.n; ++t) {
      const int cut = topns.v[t] > 0 ? min(topns.v[t], N) : N;
      float rsum = 0.f, msum = 0.f, bsum = 0.f, bsum_alt = 0.f;
      // BPref (:868-893): irrelevant = valid - relevant; the valid items lead the order, so
      // #irrelevant in the first k + 1 positions = min(k + 1, #valid) - #relevant there
      const float n_irr = nv - s_r;
      const float den_trec = fminf(n_irr, s_r);
      for (int k = tid; k < cut; k += blockDim.x) {
        const int idx = (int)(keys[k] & 0x1fffull);
        const float relk = cl[idx] >= 1.f ? 1.f : 0.f;
        rsum += relk;
        msum += term[k] / (float)(k + 1) * w[idx] * relk;   // precision@k at relevant k
        const float num = fminf(fminf((float)(k + 1), nv) - term[k], s_r);
        bsum += relk * (1.f - (den_trec != 0.f ? num / den_trec : 0.f));
        bsum_alt += relk * (1.f - (s_r != 0.f ? num / s_r : 0.f));
      }
      rsum = block_sum(rsum, red);
      msum = block_sum(msum, red);
      if (ext.bpref) bsum = block_sum(bsum, red);
      if (ext.bpref_alt) bsum_alt = block_sum(bsum_alt, red);
      if (tid == 0) {
        const size_t o = (size_t)b * topns.n + t;
        const float vt = fminf((float)cut, nv);
        if (ext.dcg) ext.dcg[o] = dcg[t];
        if (ext.precision) ext.precision[o] = vt > 0.f ? rsum / vt : 0.f;
        if (ext.recall) ext.recall[o] = s_r != 0.f ? rsum / s_r : 0.f;
        if (ext.hits) ext.hits[o] = rsum > 0.f ? 1.f : 0.f;
        if (ext.map) ext.map[o] = s_wr != 0.f ? msum / s_wr : 0.f;
        if (ext.bpref) ext.bpref[o] = s_r != 0.f ? bsum / s_r : 0.f;
        if (ext.bpref_alt) ext.bpref_alt[o] = s_r != 0.f ? bsum_alt / s_r : 0.f;
      }
    }
    if (ext.opa) {
      // ordered pair accuracy (:721-743): pairs (i, j) with l_i > l_j, weight w_i.  The
      // cleaned scores go to `term` (free again: dcg[] holds what it was needed for).
      __syncthreads();
      float* sc = term;
      for (int i = tid; i < N; i += blockDim.x) sc[i] = sc_clean(valid[i], scores[off + i], pmin);
      __syncthreads();
      float num = 0.f, den = 0.f;
      for (int i = tid; i < N; i += blockDim.x) {
        if (!valid[i]) continue;
        const float li = cl[i], si = sc[i], wi = w[i];
        float n_i = 0.f, d_i = 0.f;
        for (int j = 0; j < N; ++j) {
          const bool pair = valid[j] && li > cl[j];
          d_i += pair ? 1.f : 0.f;
          n_i += (pair && si > sc[j]) ? 1.f : 0.f;
        }
        num += wi * n_i;
        den += wi * d_i;
      }
      num = block_sum(num, red);
      den = block_sum(den, red);
      if (tid == 0) {
        ext.opa[b * 2 + 0] = den != 0.f ? num / den : 0.f;
        ext.opa[b * 2 + 1] = den;
      }
    }
  }
  if (ndcg == nullptr) return;
  __syncthreads();

  // ideal ordering: sort by weight * gain (metrics_impl.py:660-662), same mask.
  for (int i = tid; i < N; i += blockDim.x) {
    keys[i] = ((unsigned long long)(valid[i] ? 0 : 1) << 45) |
              ((unsigned long long)desc_bits(valid[i] ? wg[i] : 0.f) << 13) |
              (unsigned long long)i;
  }
  for (int i = N + tid; i < P; i += blockDim.x) keys[i] = ~0ull;
  __syncthreads();
  bitonic_sort(keys, P);
  for (int k = tid; k < N; k += blockDim.x) {
    const int idx = (int)(keys[k] & 0x1fffull);
    const float d = disc_fn == TFR_DISC_TABLE ? disc_table[k + 1] : disc_of(disc_fn, (float)(k + 1));
    term[k] = wg[idx] * d;
  }
  __syncthreads();
  for (int t = 0; t < topns.n; ++t) {
    const int cut = topns.v[t] > 0 ? min(topns.v[t], N) : N;
    float acc = 0.f;
    for (int k = tid; k < cut; k += blockDim.x) acc += term[k];
    const float ideal = block_sum(acc, red);
    if (tid == 0) ndcg[(size_t)b * topns.n + t] = ideal != 0.f ? dcg[t] / ideal : 0.f;
  }
}


// ---------------------------------------------------------------------------
// Diversity metrics (metrics_impl.py:36-60, 313-427, 746-823): labels [B, N, S] are
// per-subtopic relevances; one CTA per list, the same 64-bit key sort as K4.
//   PrecisionIA@k = sum_{r < k} #{t: l_(r)t >= 1} / (min(k, #valid) * #{t with a relevant doc})
//   alphaDCG@k    = sum_{r < k} w_(r) disc(r + 1) sum_t l_(r)t (1 - alpha)^(sum_{r' < r} l_(r')t)
// raw[b] = {sum w, -, -, sum w rel, sum rel} with rel_i = [any_t l_it >= 1] feeds the
// per-list weight rule (the same finalise kernel as MRR's weights).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kMetricThreads)
div_metrics_kernel(const float* __restrict__ scores, const float* __restrict__ labels,
                   const float* __restrict__ item_w, int w_per_item,
                   const uint8_t* __restrict__ mask, int N, int S, int P, TopnList topns,
                   float alpha, int disc_fn, const float* __restrict__ disc_table,
                   float* __restrict__ precision_ia, float* __restrict__ alpha_dcg,
                   float* __restrict__ raw) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw);
  float* w = reinterpret_cast<float*>(keys + P);   // [N] example weights
  float* relcnt = w + N;                            // [N] #subtopics with l >= 1, by position
  float* term = relcnt + N;                         // [N] alphaDCG terms by position
  float* red = term + N;                            // [32]
  float* topic_any = red + 32;                               // [S]
  float* cum = topic_any + S;                                // [N] scan buffer
  float* scratch = cum + N;                                  // [blockDim.x]
  unsigned char* valid = reinterpret_cast<unsigned char*>(scratch + kMetricThreads);

  const int b = blockIdx.x, tid = threadIdx.x;
  const size_t off = (size_t)b * N;
  const float* lab = labels + off * S;
  float pmin = CUDART_INF_F;
  for (int i = tid; i < N; i += blockDim.x) pmin = fminf(pmin, scores[off + i]);
  pmin = block_min(pmin, red);
  float s_w = 0.f, s_wr = 0.f, s_r = 0.f, nv = 0.f;
  for (int i = tid; i < N; i += blockDim.x) {
    bool ok;
    if (mask) {
      ok = mask[off + i] != 0;
    } else {                          // is_label_valid reduced over the subtopics (:352-357)
      ok = false;
      for (int t = 0; t < S; ++t) ok = ok || lab[(size_t)i * S + t] >= 0.f;
    }
    float wv = 1.f;
    if (item_w) wv = w_per_item ? item_w[off + i] : item_w[b];
    bool rel = false;
    for (int t = 0; t < S; ++t) rel = rel || (ok && lab[(size_t)i * S + t] >= 1.f);
    w[i] = wv;
    valid[i] = ok;
    keys[i] = ((unsigned long long)(ok ? 0 : 1) << 45) |
              ((unsigned long long)desc_bits(sc_clean(ok, scores[off + i], pmin)) << 13) |
              (unsigned long long)i;
    s_w += wv;
    s_wr += rel ? wv : 0.f;
    s_r += rel ? 1.f : 0.f;
    nv += ok ? 1.f : 0.f;
  }
  for (int i = N + tid; i < P; i += blockDim.x) keys[i] = ~0ull;
  s_w = block_sum(s_w, red);
  s_wr = block_sum(s_wr, red);
  s_r = block_sum(s_r, red);
  nv = block_sum(nv, red);
  if (tid == 0 && raw) {
    raw[b * 5 + 0] = s_w;
    raw[b * 5 + 1] = 0.f;
    raw[b * 5 + 2] = 0.f;
    raw[b * 5 + 3] = s_wr;
    raw[b * 5 + 4] = s_r;
  }
  __syncthreads();
  bitonic_sort(keys, P);
  // the item at position k is keys[k] & 0x1fff: the sorted keys stay put for the rest
  auto order = [keys](int k) { return (int)(keys[k] & 0x1fffull); };
  for (int k = tid; k < N; k += blockDim.x) {
    term[k] = 0.f;
    relcnt[k] = 0.f;
  }
  __syncthreads();
  // subtopic by subtopic (fixed order => deterministic sums): the running coverage along
  // the ranking is a block scan of that subtopic's sorted labels
  const float base = 1.f - alpha;
  for (int t = 0; t < S; ++t) {
    float any = 0.f;
    for (int k = tid; k < N; k += blockDim.x) {
      const int idx = order(k);
      const float l = valid[idx] ? lab[(size_t)idx * S + t] : 0.f;
      cum[k] = l;
      any = fmaxf(any, l >= 1.f ? 1.f : 0.f);
    }
    any = block_max(any, red);
    if (tid == 0) topic_any[t] = any;
    __syncthreads();
    block_inclusive_scan(cum, N, scratch);
    for (int k = tid; k < N; k += blockDim.x) {
      const int idx = order(k);
      const float l = valid[idx] ? lab[(size_t)idx * S + t] : 0.f;
      if (l != 0.f) term[k] += l * powf(base, cum[k] - l);   // exclusive coverage
      if (l >= 1.f) relcnt[k] += 1.f;
    }
    __syncthreads();
  }
  float nt = 0.f;
  for (int t = tid; t < S; t += blockDim.x) nt += topic_any[t];
  nt = block_sum(nt, red);
  for (int k = tid; k < N; k += blockDim.x) {
    const float d = disc_fn == TFR_DISC_TABLE ? disc_table[k + 1] : disc_of(disc_fn, (float)(k + 1));
    term[k] *= w[order(k)] * d;
  }
  __syncthreads();
  for (int t = 0; t < topns.n; ++t) {
    const int cut = topns.v[t] > 0 ? min(topns.v[t], N) : N;
    float a = 0.f, r = 0.f;
    for (int k = tid; k < cut; k += blockDim.x) {
      a += term[k];
      r += relcnt[k];
    }
    a = block_sum(a, red);
    r = block_sum(r, red);
    if (tid == 0) {
      const size_t o = (size_t)b * topns.n + t;
      const float den = fminf((float)cut, nv) * nt;
      if (precision_ia) precision_ia[o] = den != 0.f ? r / den : 0.f;
      if (alpha_dcg) alpha_dcg[o] = a;
    }
  }
}

// metrics_impl.py:63-119 over one (single-process) batch.
__global__ void __launch_bounds__(1024)
metric_list_weights_kernel(const float* __restrict__ raw, int B, float* __restrict__ ndcg_w,
                           float* __restrict__ mrr_w) {
  __shared__ float red[32];
  for (int m = 0; m < 2; ++m) {
    float* out = m == 0 ? ndcg_w : mrr_w;
    if (out == nullptr) continue;
    float cnt = 0.f, sw = 0.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
      const float sum_w = raw[b * 5 + 0];
      const float wr = raw[b * 5 + 1 + 2 * m], r = raw[b * 5 + 2 + 2 * m];
      cnt += (sum_w > 0.f && r > 0.f) ? 1.f : 0.f;
      sw += r != 0.f ? wr / r : 0.f;
    }
    cnt = block_sum(cnt, red);
    sw = block_sum(sw, red);
    const float avg = cnt > 0.f ? sw / cnt : 1.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
      const float sum_w = raw[b * 5 + 0];
      const float wr = raw[b * 5 + 1 + 2 * m], r = raw[b * 5 + 2 + 2 * m];
      out[b] = sum_w > 0.f ? (r > 0.f ? wr / r : avg) : 0.f;
    }
  }
}

static int next_pow2(int n) {
  int p = 1;
  while (p < n) p <<= 1;
  return p;
}

// Dynamic shared memory of one CTA, as carved by the kernels above.  At N = 8192 the rank
// kernel needs 204,944 bytes (205,968 with extended outputs) and the diversity kernel
// 205,968 + 4 S bytes: all fit the 232,448-byte opt-in limit of an H100 for every S <= 4096.
static size_t rank_metrics_smem_bytes(int N, bool ext) {
  const size_t P = (size_t)next_pow2(N);
  return ((P * 8 + (size_t)(4 * N + 32) * 4 + N + 15) & ~(size_t)15) +
         (ext ? (size_t)kMetricThreads * 4 : 0) + 16;
}

static size_t div_metrics_smem_bytes(int N, int S) {
  return (size_t)next_pow2(N) * 8 + (size_t)(4 * N + 32 + S + kMetricThreads) * 4 + N + 16;
}

// Largest list size whose launch fits `limit` bytes (0 if none does).
template <typename F>
static int largest_fitting_list(F bytes_for, size_t limit) {
  int n = kMaxMetricListSize;
  while (n >= 1 && bytes_for(n) > limit) --n;
  return n;
}

// Checks the launch's shared memory against the device's opt-in limit before any CUDA call,
// then raises the kernel's limit when it needs more than the default 48 KB.
template <typename K, typename F>
static int prep_metric_smem(K kernel, int N, F bytes_for, const char* what) {
  const size_t smem = bytes_for(N), limit = smem_optin_limit();
  TFR_REQUIRE(smem <= limit,
              "%s: list_size %d needs %zu bytes of shared memory per block but the device "
              "allows %zu; the largest list_size accepted for this call is %d",
              what, N, smem, limit, largest_fitting_list(bytes_for, limit));
  if (smem > 48 * 1024)
    TFR_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)smem));
  return TFR_OK;
}

}  // namespace tfr

using namespace tfr;

extern "C" int tfr_rank_metrics_ext(const float* scores, const float* labels,
                                const float* item_w, int w_per_item, const uint8_t* mask,
                                int B, int N, const int32_t* topns_host, int n_topn,
                                int gain_fn, int disc_fn, const float* gain_table,
                                const float* disc_table, float* ndcg, float* ndcg_w,
                                    float* mrr, float* mrr_w, float* raw,
                                    const tfr_metric_ext* ext_host, void* stream) {
  TFR_REQUIRE(scores && labels, "scores/labels must not be NULL");
  TFR_REQUIRE(B >= 0 && N >= 1 && N <= kMaxMetricListSize,
              "need 1 <= list_size <= %d (got %d)", kMaxMetricListSize, N);
  TFR_REQUIRE(n_topn >= 1 && n_topn <= kMaxTopn && topns_host, "need 1..%d cut-offs", kMaxTopn);
  TFR_REQUIRE(gain_fn >= 0 && gain_fn <= TFR_GAIN_TABLE && disc_fn >= 0 && disc_fn <= TFR_DISC_TABLE,
              "bad gain_fn/disc_fn");
  TFR_REQUIRE(gain_fn != TFR_GAIN_TABLE || gain_table, "gain_fn TABLE needs gain_table");
  TFR_REQUIRE(disc_fn != TFR_DISC_TABLE || disc_table, "disc_fn TABLE needs disc_table");
  TFR_REQUIRE(raw != nullptr, "raw [B,5] workspace must not be NULL");
  if (B == 0) return TFR_OK;
  TopnList t;
  t.n = n_topn;
  for (int i = 0; i < n_topn; ++i) t.v[i] = topns_host[i];
  const int P = next_pow2(N);
  MetricExt ext{};
  if (ext_host)
    ext = MetricExt{ext_host->dcg, ext_host->precision, ext_host->recall, ext_host->map,
                    ext_host->hits, ext_host->arp, ext_host->opa, ext_host->bpref,
                    ext_host->bpref_alt};
  const bool want_ext = ext.any();
  auto bytes_for = [want_ext](int n) { return rank_metrics_smem_bytes(n, want_ext); };
  int rc = prep_metric_smem(rank_metrics_kernel, N, bytes_for, "tfr_rank_metrics");
  if (rc) return rc;
  const size_t smem = bytes_for(N);
  cudaStream_t st = (cudaStream_t)stream;
  rank_metrics_kernel<<<B, kMetricThreads, smem, st>>>(scores, labels, item_w, w_per_item, mask,
                                                      N, P, t, gain_fn, disc_fn, gain_table,
                                                      disc_table, ndcg, mrr, raw, ext);
  TFR_LAUNCH_OK();
  if (ndcg_w || mrr_w) {
    metric_list_weights_kernel<<<1, 1024, 0, st>>>(raw, B, ndcg_w, mrr_w);
    TFR_LAUNCH_OK();
  }
  return TFR_OK;
}

extern "C" int tfr_rank_metrics(const float* scores, const float* labels,
                                const float* item_w, int w_per_item, const uint8_t* mask,
                                int B, int N, const int32_t* topns_host, int n_topn,
                                int gain_fn, int disc_fn, const float* gain_table,
                                const float* disc_table, float* ndcg, float* ndcg_w,
                                float* mrr, float* mrr_w, float* raw, void* stream) {
  return tfr_rank_metrics_ext(scores, labels, item_w, w_per_item, mask, B, N, topns_host,
                              n_topn, gain_fn, disc_fn, gain_table, disc_table, ndcg, ndcg_w,
                              mrr, mrr_w, raw, nullptr, stream);
}

extern "C" int tfr_div_metrics(const float* scores, const float* labels, const float* item_w,
                               int w_per_item, const uint8_t* mask, int B, int N, int S,
                               const int32_t* topns_host, int n_topn, float alpha, int disc_fn,
                               const float* disc_table, float* precision_ia, float* alpha_dcg,
                               float* list_w, float* raw, void* stream) {
  TFR_REQUIRE(scores && labels, "scores/labels must not be NULL");
  TFR_REQUIRE(B >= 0 && N >= 1 && N <= kMaxMetricListSize,
              "need 1 <= list_size <= %d (got %d)", kMaxMetricListSize, N);
  TFR_REQUIRE(S >= 1 && S <= 4096, "subtopic_size %d out of range", S);
  TFR_REQUIRE(n_topn >= 1 && n_topn <= kMaxTopn && topns_host, "need 1..%d cut-offs", kMaxTopn);
  TFR_REQUIRE(disc_fn >= 0 && disc_fn <= TFR_DISC_TABLE, "bad disc_fn");
  TFR_REQUIRE(disc_fn != TFR_DISC_TABLE || disc_table, "disc_fn TABLE needs disc_table");
  TFR_REQUIRE(raw != nullptr, "raw [B,5] workspace must not be NULL");
  if (B == 0) return TFR_OK;
  TopnList t;
  t.n = n_topn;
  for (int i = 0; i < n_topn; ++i) t.v[i] = topns_host[i];
  const int P = next_pow2(N);
  auto bytes_for = [S](int n) { return div_metrics_smem_bytes(n, S); };
  int rc = prep_metric_smem(div_metrics_kernel, N, bytes_for, "tfr_div_metrics");
  if (rc) return rc;
  const size_t smem = bytes_for(N);
  cudaStream_t st = (cudaStream_t)stream;
  div_metrics_kernel<<<B, kMetricThreads, smem, st>>>(scores, labels, item_w, w_per_item, mask, N,
                                                     S, P, t, alpha, disc_fn, disc_table,
                                                     precision_ia, alpha_dcg, raw);
  TFR_LAUNCH_OK();
  if (list_w) {
    metric_list_weights_kernel<<<1, 1024, 0, st>>>(raw, B, nullptr, list_w);
    TFR_LAUNCH_OK();
  }
  return TFR_OK;
}
