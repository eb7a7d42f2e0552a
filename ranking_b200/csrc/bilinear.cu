// K14  Bilinear (keras/layers.py:807-890): for every row m of v1, v2 [M, E]
//   y[m, k] = sum_ij v1[m, i] W[i, j, k] v2[m, j] + sum_i v1[m, i] W1[i, k]
//             + sum_j v2[m, j] W2[j, k] + b[k]
// FP32 on CUDA cores.  Both kernels fold the linear and constant terms into one augmented
// bilinear form: with a = [v1, 1] and c = [v2, 1] (length E1 = E + 1) and
//   W'[i, j, k] = W[i, j, k] (i, j < E),  W'[i, E, k] = W1[i, k],  W'[E, j, k] = W2[j, k],
//   W'[E, E, k] = b[k],
// y[m, k] = sum_ij a_i W'[i, j, k] c_j, and the six gradients are one augmented outer product
// dW'[i, j, k] = sum_m dy[m, k] a_i c_j plus two contractions of W' for dv1 and dv2.
//
// A CTA keeps W' in shared memory (k-major, rows padded to EP = roundup(E1, 4) floats so a
// thread reads four columns with one 16-byte load) and walks tiles of R consecutive rows:
// a tile of v1 / v2 is one contiguous run of R * E floats, read with coalesced 16-byte loads
// into shared memory, so rows of 64 bytes (E = 16) cost no more than wide ones.
//   forward   one thread per (row, k); the tile rows sit at an odd pitch so that the 32 lanes
//             of a warp, which hold 32 different rows, read them without bank conflicts.
//   backward  per-thread dW' accumulators over a fixed row slice, added into a per-CTA
//             partial in shared memory after every tile; at the end the CTA writes its
//             partial to the workspace and a second kernel sums the G partials in a fixed order.
//             The row -> CTA assignment depends on (M, E, K) only, so two identical calls give
//             identical bits.  No float atomics.
#include "common.cuh"

namespace tfr {

namespace {

constexpr int kThreads = 256;
constexpr int kMaxE = 128;
constexpr int kMaxK = 32;
constexpr int kMaxEEK = 16384;
constexpr int kMaxCtas = 528;                     // backward partials (4 per SM on an H100)
constexpr size_t kSmemBudget = 232448 - 1024;     // H100 opt-in limit, with some headroom

struct Geo {
  int E, K, E1, EP, Q;   // Q = EP / 4 column quads
  int LD;                // odd pitch of the row tiles (>= EP)
  int LDK;               // odd pitch of the dy tile (>= K)
  int LDO;               // odd pitch of the dv staging tile (>= E)
  int R;                 // rows per tile
  int NG, S;             // backward: dW' quads, row slices per quad
  size_t P;              // parameter count
};

__host__ __device__ inline int odd_at_least(int x) { return x | 1; }

Geo make_geo(int E, int K) {
  Geo g;
  g.E = E;
  g.K = K;
  g.E1 = E + 1;
  g.EP = (g.E1 + 3) & ~3;
  g.Q = g.EP / 4;
  g.LD = odd_at_least(g.EP);
  g.LDK = odd_at_least(K);
  g.LDO = odd_at_least(E);
  g.NG = g.E1 * K * g.Q;
  g.S = g.NG >= kThreads ? 1 : kThreads / g.NG;
  g.P = (size_t)E * E * K + 2 * (size_t)E * K + K;
  g.R = 0;
  return g;
}

size_t fwd_smem_floats(const Geo& g, int R) {
  return (size_t)g.K * g.E1 * g.EP + 2 * (size_t)R * g.LD;
}

// W' (in both orientations when `transposed`), the dW' partial, a / c at the odd pitch, c again
// at pitch EP (the dW' pass reads four columns of one row at a time), dy and the dv staging tile.
size_t bwd_smem_floats(const Geo& g, int R, bool transposed) {
  return (transposed ? 2 : 1) * (size_t)g.K * g.E1 * g.EP + (size_t)g.S * g.NG * 4 +
         2 * (size_t)R * g.LD + (size_t)R * g.EP + (size_t)R * g.LDK + (size_t)R * g.LDO;
}

// Rows per tile: the largest that fits.  The backward keeps a second, transposed copy of W' for
// 16-byte loads in the dv1 pass when that fits with R >= 8 rows, and reads the one copy with
// scalar loads otherwise (*transposed = false; only a few shapes near E^2 K = 16384).  Every
// (E, K) within the limits fits one of the two with R >= 8.
int pick_rows(const Geo& g, bool bwd, bool* transposed) {
  for (int t = 1; t >= 0; --t) {
    for (int R = bwd ? 128 : 256; R >= 8; R >>= 1) {
      const size_t f = bwd ? bwd_smem_floats(g, R, t) : fwd_smem_floats(g, R);
      if (f * sizeof(float) <= kSmemBudget) {
        if (transposed) *transposed = t;
        return R;
      }
    }
    if (!bwd) break;
  }
  return 0;
}

int bwd_ctas(const Geo& g, int M) {
  const int tiles = (M + g.R - 1) / g.R;
  return tiles < kMaxCtas ? tiles : kMaxCtas;
}

// sW[(k * E1 + i) * EP + j] = W'[i, j, k] (transposed = 0), or W'[j, i, k] (transposed = 1);
// zero in the padding columns.
__device__ void load_augmented(const float* __restrict__ params, const Geo& g, int transposed,
                               float* __restrict__ sW) {
  const int E = g.E, K = g.K;
  const float* W1 = params + (size_t)E * E * K;
  const float* W2 = W1 + (size_t)E * K;
  const float* b = W2 + (size_t)E * K;
  const int n = K * g.E1 * g.EP;
  for (int e = threadIdx.x; e < n; e += blockDim.x) {
    const int col = e % g.EP;
    const int row = (e / g.EP) % g.E1;
    const int k = e / (g.EP * g.E1);
    const int i = transposed ? col : row, j = transposed ? row : col;
    float v = 0.f;
    if (i < E && j < E) v = __ldg(params + ((size_t)i * E + j) * K + k);
    else if (i < E && j == E) v = __ldg(W1 + (size_t)i * K + k);
    else if (i == E && j < E) v = __ldg(W2 + (size_t)j * K + k);
    else if (i == E && j == E) v = __ldg(b + k);
    sW[e] = v;
  }
}

// Rows [row0, row0 + rows) of v [M, E] into s[r * ld + 0..E1): the row, then the constant 1;
// masked rows and rows past `rows` are zero (constant included), so they contribute nothing.
// A second copy at pitch EP (s2, optional) serves the backward's dW' pass.
__device__ void load_tile(const float* __restrict__ v, const uint8_t* __restrict__ mask,
                          int row0, int rows, const Geo& g, int R, float* __restrict__ s,
                          float* __restrict__ s2) {
  const int E = g.E;
  const int n = rows * E;
  const float* src = v + (size_t)row0 * E;
  const bool vec = (E & 3) == 0 && (reinterpret_cast<uintptr_t>(v) & 15) == 0;
  if (vec) {
    const float4* src4 = reinterpret_cast<const float4*>(src);
    for (int e4 = threadIdx.x; e4 < n / 4; e4 += blockDim.x) {
      const float4 x = __ldg(src4 + e4);
      const int r = (4 * e4) / E, j = 4 * e4 - r * E;
      const bool live = !mask || mask[row0 + r];
      const float xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float val = live ? xs[q] : 0.f;
        s[r * g.LD + j + q] = val;
        if (s2) s2[r * g.EP + j + q] = val;
      }
    }
  } else {
    for (int e = threadIdx.x; e < n; e += blockDim.x) {
      const int r = e / E, j = e - r * E;
      const bool live = !mask || mask[row0 + r];
      const float val = live ? __ldg(src + e) : 0.f;
      s[r * g.LD + j] = val;
      if (s2) s2[r * g.EP + j] = val;
    }
  }
  // the constant column, the padding columns, and whole rows past the tile's end
  const int pad = g.EP - E;
  for (int e = threadIdx.x; e < R * pad; e += blockDim.x) {
    const int r = e / pad, j = E + (e - r * pad);
    const float val = (j == E && r < rows && (!mask || mask[row0 + r])) ? 1.f : 0.f;
    s[r * g.LD + j] = val;
    if (s2) s2[r * g.EP + j] = val;
  }
  for (int e = threadIdx.x; e < (R - rows) * E; e += blockDim.x) {
    const int r = rows + e / E, j = e % E;
    s[r * g.LD + j] = 0.f;
    if (s2) s2[r * g.EP + j] = 0.f;
  }
}

// out4[q] += sum_i x[i] * sW[(k * E1 + i) * EP + 4 jq + q] over i < E1: four columns of the
// contraction of W' (in the orientation of sW) with the row x.
__device__ __forceinline__ float4 contract4(const float* __restrict__ x,
                                            const float* __restrict__ sW, int k, int jq,
                                            const Geo& g) {
  const float4* w4 = reinterpret_cast<const float4*>(sW + (size_t)k * g.E1 * g.EP) + jq;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int i = 0; i < g.E1; ++i) {
    const float a = x[i];
    const float4 w = w4[i * g.Q];
    s.x = fmaf(a, w.x, s.x);
    s.y = fmaf(a, w.y, s.y);
    s.z = fmaf(a, w.z, s.z);
    s.w = fmaf(a, w.w, s.w);
  }
  return s;
}

__global__ void __launch_bounds__(kThreads)
bilinear_fwd_kernel(const float* __restrict__ v1, const float* __restrict__ v2, int M,
                    Geo g, const float* __restrict__ params,
                    const uint8_t* __restrict__ mask, float* __restrict__ y) {
  extern __shared__ float4 smem4[];
  float* sW = reinterpret_cast<float*>(smem4);
  float* sa = sW + (size_t)g.K * g.E1 * g.EP;
  float* sc = sa + (size_t)g.R * g.LD;
  load_augmented(params, g, 0, sW);
  const int R = g.R, K = g.K;
  const int tiles = (M + R - 1) / R;
  for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int row0 = t * R, rows = min(R, M - row0);
    __syncthreads();   // the previous tile's rows are no longer read (first pass: sW written)
    load_tile(v1, mask, row0, rows, g, R, sa, nullptr);
    load_tile(v2, mask, row0, rows, g, R, sc, nullptr);
    __syncthreads();
    for (int it = threadIdx.x; it < rows * K; it += blockDim.x) {
      const int k = it / rows, r = it - k * rows;
      const float* ar = sa + r * g.LD;
      const float* cr = sc + r * g.LD;
      float acc = 0.f;
      for (int jq = 0; jq < g.Q; ++jq) {
        // s_j = sum_i a_i W'[i, j, k]: with a_E = 1 it carries W2 (j < E) and b (j = E)
        const float4 s = contract4(ar, sW, k, jq, g);
        acc = fmaf(cr[4 * jq + 0], s.x, acc);
        acc = fmaf(cr[4 * jq + 1], s.y, acc);
        acc = fmaf(cr[4 * jq + 2], s.z, acc);
        acc = fmaf(cr[4 * jq + 3], s.w, acc);
      }
      const int m = row0 + r;
      y[(size_t)m * K + k] = (mask && !mask[m]) ? kLogEpsilon : acc;
    }
  }
}

// Four rows 4 iq .. 4 iq + 3 of the contraction sum_j W'[i, j, k] c_j from the one copy of W',
// with scalar loads (every lane of a warp reads the same W' entries: broadcasts).
__device__ __forceinline__ float4 contract4_rows(const float* __restrict__ c,
                                                 const float* __restrict__ sW, int k, int iq,
                                                 const Geo& g) {
  const float* w = sW + (size_t)k * g.E1 * g.EP;
  float s[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = 4 * iq + q;
    if (i >= g.E1) break;
    for (int j = 0; j < g.E1; ++j) s[q] = fmaf(c[j], w[i * g.EP + j], s[q]);
  }
  return make_float4(s[0], s[1], s[2], s[3]);
}

template <bool kTransposed>
__global__ void __launch_bounds__(kThreads)
bilinear_bwd_kernel(const float* __restrict__ v1, const float* __restrict__ v2, int M,
                    Geo g, const float* __restrict__ params,
                    const uint8_t* __restrict__ mask, const float* __restrict__ dy,
                    float* __restrict__ dv1, float* __restrict__ dv2,
                    float* __restrict__ partials) {
  extern __shared__ float4 smem4[];
  const int R = g.R, K = g.K, E = g.E, E1 = g.E1, EP = g.EP, Q = g.Q;
  const size_t wsz = (size_t)K * E1 * EP;
  float* sW = reinterpret_cast<float*>(smem4);      // W'[i, j, k] at (k E1 + i) EP + j
  float* sWt = sW + wsz;                            // W'[i, j, k] at (k E1 + j) EP + i
  float* part = sW + (kTransposed ? 2 : 1) * wsz;   // [S][NG][4]
  float* sa = part + (size_t)g.S * g.NG * 4;        // a rows, pitch LD
  float* sc = sa + (size_t)R * g.LD;                // c rows, pitch LD
  float* sc4 = sc + (size_t)R * g.LD;               // c rows, pitch EP
  float* sdy = sc4 + (size_t)R * EP;                // dy rows, pitch LDK (0 where masked)
  float* sdv = sdy + (size_t)R * g.LDK;             // dv1 / dv2 staging, pitch LDO
  load_augmented(params, g, 0, sW);
  if (kTransposed) load_augmented(params, g, 1, sWt);
  const int nitems = g.S * g.NG;
  for (int w = threadIdx.x; w < nitems * 4; w += blockDim.x) part[w] = 0.f;
  const int tiles = (M + R - 1) / R;
  const bool vec_out = (E & 3) == 0 && (reinterpret_cast<uintptr_t>(dv1) & 15) == 0 &&
                       (reinterpret_cast<uintptr_t>(dv2) & 15) == 0;
  for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int row0 = t * R, rows = min(R, M - row0);
    __syncthreads();
    load_tile(v1, mask, row0, rows, g, R, sa, nullptr);
    load_tile(v2, mask, row0, rows, g, R, sc, sc4);
    for (int e = threadIdx.x; e < R * K; e += blockDim.x) {
      const int r = e / K, k = e - r * K;
      const bool live = r < rows && (!mask || mask[row0 + r]);
      sdy[r * g.LDK + k] = live ? __ldg(dy + (size_t)(row0 + r) * K + k) : 0.f;
    }
    __syncthreads();
    // dW' quads: item w = s * NG + (i * K + k) * Q + jq sums rows s, s + S, ... of the tile
    for (int w = threadIdx.x; w < nitems; w += blockDim.x) {
      const int s = w / g.NG, gq = w - s * g.NG;
      const int jq = gq % Q, ik = gq / Q;
      const int k = ik % K, i = ik / K;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int r = s; r < rows; r += g.S) {
        const float u = sdy[r * g.LDK + k] * sa[r * g.LD + i];
        const float4 c = *reinterpret_cast<const float4*>(sc4 + r * EP + 4 * jq);
        acc.x = fmaf(u, c.x, acc.x);
        acc.y = fmaf(u, c.y, acc.y);
        acc.z = fmaf(u, c.z, acc.z);
        acc.w = fmaf(u, c.w, acc.w);
      }
      float4* p = reinterpret_cast<float4*>(part) + w;
      float4 cur = *p;
      cur.x += acc.x; cur.y += acc.y; cur.z += acc.z; cur.w += acc.w;
      *p = cur;
    }
    // dv1[m, i] = sum_k dy_k sum_j W'[i, j, k] c_j  (c_E = 1 brings in W1)
    for (int it = threadIdx.x; it < rows * Q; it += blockDim.x) {
      const int iq = it / rows, r = it - iq * rows;
      float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int k = 0; k < K; ++k) {
        const float dk = sdy[r * g.LDK + k];
        const float4 s = kTransposed ? contract4(sc + r * g.LD, sWt, k, iq, g)
                                     : contract4_rows(sc + r * g.LD, sW, k, iq, g);
        d.x = fmaf(dk, s.x, d.x);
        d.y = fmaf(dk, s.y, d.y);
        d.z = fmaf(dk, s.z, d.z);
        d.w = fmaf(dk, s.w, d.w);
      }
      const float ds[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (4 * iq + q < E) sdv[r * g.LDO + 4 * iq + q] = ds[q];
    }
    for (int pass = 0; pass < 2; ++pass) {
      __syncthreads();
      float* out = (pass == 0 ? dv1 : dv2) + (size_t)row0 * E;
      const int n = rows * E;
      if (vec_out) {
        for (int e4 = threadIdx.x; e4 < n / 4; e4 += blockDim.x) {
          const int r = (4 * e4) / E, j = 4 * e4 - r * E;
          const float* src = sdv + r * g.LDO + j;
          reinterpret_cast<float4*>(out)[e4] = make_float4(src[0], src[1], src[2], src[3]);
        }
      } else {
        for (int e = threadIdx.x; e < n; e += blockDim.x) {
          const int r = e / E, j = e - r * E;
          out[e] = sdv[r * g.LDO + j];
        }
      }
      if (pass == 1) break;
      __syncthreads();
      // dv2[m, j] = sum_k dy_k sum_i a_i W'[i, j, k]  (a_E = 1 brings in W2)
      for (int it = threadIdx.x; it < rows * Q; it += blockDim.x) {
        const int jq = it / rows, r = it - jq * rows;
        float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int k = 0; k < K; ++k) {
          const float dk = sdy[r * g.LDK + k];
          const float4 s = contract4(sa + r * g.LD, sW, k, jq, g);
          d.x = fmaf(dk, s.x, d.x);
          d.y = fmaf(dk, s.y, d.y);
          d.z = fmaf(dk, s.z, d.z);
          d.w = fmaf(dk, s.w, d.w);
        }
        const float ds[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (4 * jq + q < E) sdv[r * g.LDO + 4 * jq + q] = ds[q];
      }
    }
  }
  __syncthreads();
  // this CTA's partial in the parameter layout: W, W1, W2, b; slices summed in order
  float* out = partials + (size_t)blockIdx.x * g.P;
  const size_t nW = (size_t)E * E * K, nL = (size_t)E * K;
  for (size_t p = threadIdx.x; p < g.P; p += blockDim.x) {
    int i, j, k;
    if (p < nW) {
      k = (int)(p % K);
      j = (int)((p / K) % E);
      i = (int)(p / ((size_t)K * E));
    } else if (p < nW + nL) {
      k = (int)((p - nW) % K); i = (int)((p - nW) / K); j = E;
    } else if (p < nW + 2 * nL) {
      k = (int)((p - nW - nL) % K); j = (int)((p - nW - nL) / K); i = E;
    } else {
      k = (int)(p - nW - 2 * nL); i = E; j = E;
    }
    const int gq = (i * K + k) * Q + j / 4, q = j & 3;
    float acc = 0.f;
    for (int s = 0; s < g.S; ++s) acc += part[((size_t)s * g.NG + gq) * 4 + q];
    out[p] = acc;
  }
}

// grads[p] = sum over the G CTA partials of partials[c][p]: one block per p, thread t sums
// c = t, t + 256, ... in order, then block_sum's fixed tree.
__global__ void __launch_bounds__(256)
bilinear_reduce_kernel(const float* __restrict__ partials, int G, size_t P,
                       float* __restrict__ grads) {
  __shared__ float red[32];
  const size_t p = blockIdx.x;
  float acc = 0.f;
  for (int c = threadIdx.x; c < G; c += blockDim.x) acc += partials[(size_t)c * P + p];
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) grads[p] = acc;
}

int check_sizes(int M, int E, int K) {
  TFR_REQUIRE(M >= 1, "bilinear: M = %d must be >= 1", M);
  TFR_REQUIRE(E >= 1 && E <= kMaxE, "bilinear: embedding_dim %d must be in [1, %d]", E, kMaxE);
  TFR_REQUIRE(K >= 1 && K <= kMaxK, "bilinear: output_dim %d must be in [1, %d]", K, kMaxK);
  TFR_REQUIRE((long long)E * E * K <= kMaxEEK,
              "bilinear: embedding_dim^2 * output_dim = %lld exceeds %d", (long long)E * E * K,
              kMaxEEK);
  TFR_REQUIRE((long long)M * (E > K ? E : K) < (1ll << 31), "bilinear: M = %d too large", M);
  return TFR_OK;
}

int set_smem(const void* fn, size_t bytes) {
  if (bytes > 48 * 1024)
    TFR_CUDA_OK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)bytes));
  return TFR_OK;
}

}  // namespace

}  // namespace tfr

using namespace tfr;

extern "C" size_t tfr_bilinear_param_count(int E, int K) {
  if (check_sizes(1, E, K) != TFR_OK) return 0;
  return make_geo(E, K).P;
}

extern "C" size_t tfr_bilinear_workspace_bytes(int M, int E, int K) {
  if (check_sizes(M, E, K) != TFR_OK) return 0;
  Geo g = make_geo(E, K);
  g.R = pick_rows(g, true, nullptr);
  return (size_t)bwd_ctas(g, M) * g.P * sizeof(float);
}

extern "C" int tfr_bilinear_fwd(const float* v1, const float* v2, int M, int E, int K,
                                const float* params, const uint8_t* row_mask, float* y,
                                void* stream) {
  TFR_REQUIRE(v1 && v2 && params && y, "bilinear: NULL argument");
  int rc = check_sizes(M, E, K);
  if (rc) return rc;
  Geo g = make_geo(E, K);
  g.R = pick_rows(g, false, nullptr);
  const size_t smem = fwd_smem_floats(g, g.R) * sizeof(float);
  rc = set_smem((const void*)bilinear_fwd_kernel, smem);
  if (rc) return rc;
  int per_sm = 0;
  TFR_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bilinear_fwd_kernel,
                                                            kThreads, smem));
  const int tiles = (M + g.R - 1) / g.R;
  const int cap = num_sms() * (per_sm > 0 ? per_sm : 1);
  bilinear_fwd_kernel<<<tiles < cap ? tiles : cap, kThreads, smem, (cudaStream_t)stream>>>(
      v1, v2, M, g, params, row_mask, y);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

extern "C" int tfr_bilinear_bwd(const float* v1, const float* v2, int M, int E, int K,
                                const float* params, const uint8_t* row_mask, const float* dy,
                                float* dv1, float* dv2, float* grads, void* workspace,
                                void* stream) {
  TFR_REQUIRE(v1 && v2 && params && dy && dv1 && dv2 && grads && workspace,
              "bilinear: NULL argument");
  int rc = check_sizes(M, E, K);
  if (rc) return rc;
  Geo g = make_geo(E, K);
  bool transposed = true;
  g.R = pick_rows(g, true, &transposed);
  const size_t smem = bwd_smem_floats(g, g.R, transposed) * sizeof(float);
  auto kernel = transposed ? bilinear_bwd_kernel<true> : bilinear_bwd_kernel<false>;
  rc = set_smem((const void*)kernel, smem);
  if (rc) return rc;
  const int G = bwd_ctas(g, M);
  cudaStream_t st = (cudaStream_t)stream;
  float* partials = static_cast<float*>(workspace);
  kernel<<<G, kThreads, smem, st>>>(v1, v2, M, g, params, row_mask, dy, dv1, dv2, partials);
  TFR_LAUNCH_OK();
  bilinear_reduce_kernel<<<(unsigned)g.P, 256, 0, st>>>(partials, G, g.P, grads);
  TFR_LAUNCH_OK();
  return TFR_OK;
}
