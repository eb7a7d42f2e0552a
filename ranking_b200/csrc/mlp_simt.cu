// K5/K6 (fp32 CUDA-core path): create_tower forward/backward over the flattened
// [M, D] matrix with register-tiled SGEMMs.  This is the exact-fp32 path
// (TFR_PREC_FP32); the tensor-core paths live in mlp_tc.cu.
//
// Layout: activations row-major [M, units]; Dense kernels [in, out] row-major
// (Keras layout, keras/layers.py:70); all parameters / gradients in one flat
// buffer: W_0, b_0, W_1, b_1, ...
#include "common.cuh"
#include "mlp.h"

namespace tfr {

// ------------------------------------------------------------------ SGEMM ---
// C[M, N] = epi(opA(A) * opB(B)); 128x128x8 tile, 256 threads, 8x8 per thread.
constexpr int BM = 128, BN = 128, BK = 8, GEMM_THREADS = 256;

enum Epilogue { EPI_NONE = 0, EPI_BIAS_ACT = 1, EPI_MASK_POS = 2 };

struct GemmArgs {
  const float* A; int lda;
  const float* B; int ldb;
  float* C; int ldc;
  int M, N, K;
  const float* bias;   // EPI_BIAS_ACT: [N]
  const float* aux;    // EPI_MASK_POS: [M, N] (ld = ldc); C *= (aux > 0)
  int act;
  // split-K (over the K dimension): each blockIdx.z handles k_per_split of K and
  // writes to C + z * split_stride.
  int k_per_split;
  size_t split_stride;
};

template <bool TA, bool TB, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS)
sgemm_kernel(GemmArgs g) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kbeg = blockIdx.z * g.k_per_split;
  const int kend = min(g.K, kbeg + g.k_per_split);
  float* C = g.C + (size_t)blockIdx.z * g.split_stride;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  for (int k0 = kbeg; k0 < kend; k0 += BK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = tid + i * GEMM_THREADS;  // 0 .. 1023
      int m, k;
      if (TA) { m = e & (BM - 1); k = e >> 7; } else { k = e & (BK - 1); m = e >> 3; }
      const int gm = m0 + m, gk = k0 + k;
      float v = 0.f;
      if (gm < g.M && gk < kend)
        v = TA ? g.A[(size_t)gk * g.lda + gm] : g.A[(size_t)gm * g.lda + gk];
      As[k][m] = v;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = tid + i * GEMM_THREADS;
      int n, k;
      if (TB) { k = e & (BK - 1); n = e >> 3; } else { n = e & (BN - 1); k = e >> 7; }
      const int gn = n0 + n, gk = k0 + k;
      float v = 0.f;
      if (gn < g.N && gk < kend)
        v = TB ? g.B[(size_t)gn * g.ldb + gk] : g.B[(size_t)gk * g.ldb + gn];
      Bs[k][n] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[8], b[8];
      *reinterpret_cast<float4*>(&a[0]) = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      *reinterpret_cast<float4*>(&a[4]) = *reinterpret_cast<const float4*>(&As[kk][64 + ty * 4]);
      *reinterpret_cast<float4*>(&b[0]) = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      *reinterpret_cast<float4*>(&b[4]) = *reinterpret_cast<const float4*>(&Bs[kk][64 + tx * 4]);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int gm = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (gm >= g.M) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int gn = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
      if (gn >= g.N) continue;
      float v = acc[i][j];
      if (EPI == EPI_BIAS_ACT) {
        v += g.bias[gn];
        if (g.act == TFR_ACT_RELU) v = fmaxf(v, 0.f);
      } else if (EPI == EPI_MASK_POS) {
        if (g.act == TFR_ACT_RELU && !(g.aux[(size_t)gm * g.ldc + gn] > 0.f)) v = 0.f;
      }
      C[(size_t)gm * g.ldc + gn] = v;
    }
  }
}

template <bool TA, bool TB, int EPI>
static int launch_gemm(GemmArgs g, int splits, cudaStream_t st) {
  dim3 grid((g.N + BN - 1) / BN, (g.M + BM - 1) / BM, splits);
  sgemm_kernel<TA, TB, EPI><<<grid, GEMM_THREADS, 0, st>>>(g);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

// ------------------------------------------------------- output layer fwd ---
// scores[m, o] = H[m, :] . W[:, o] + b[o]; RestoreList fill for masked rows
// (keras/layers.py:265).  One warp per row.  kPlanar: task-major scores[o * M + m], with the
// fill on every plane (tfr_mlp_fwd_tasks); otherwise [M, O], filled only when O == 1.
template <bool kPlanar>
__device__ __forceinline__ void out_layer_fwd(const float* __restrict__ H, int M, int K, int O,
                                              const float* __restrict__ W,
                                              const float* __restrict__ bias,
                                              const uint8_t* __restrict__ mask,
                                              float* __restrict__ scores) {
  // one warp per 4 consecutive rows: 4 independent row loads in flight per lane
  const int lane = threadIdx.x & 31;
  const int row0 = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 4;
  if (row0 >= M) return;
  for (int o = 0; o < O; ++o) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k = lane; k < K; k += 32) {
      const float w = W[(size_t)k * O + o];
#pragma unroll
      for (int r = 0; r < 4; ++r)
        if (row0 + r < M) acc[r] = fmaf(H[(size_t)(row0 + r) * K + k], w, acc[r]);
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) acc[r] = warp_sum(acc[r]);
    if (lane < 4 && row0 + lane < M) {
      const int row = row0 + lane;
      float v = (lane == 0 ? acc[0] : lane == 1 ? acc[1] : lane == 2 ? acc[2] : acc[3]) + bias[o];
      if (mask && (kPlanar || O == 1) && !mask[row]) v = kLogEpsilon;
      scores[kPlanar ? (size_t)o * M + row : (size_t)row * O + o] = v;
    }
  }
}

__global__ void __launch_bounds__(256)
out_layer_fwd_kernel(const float* __restrict__ H, int M, int K, int O,
                     const float* __restrict__ W, const float* __restrict__ bias,
                     const uint8_t* __restrict__ mask, float* __restrict__ scores) {
  out_layer_fwd<false>(H, M, K, O, W, bias, mask, scores);
}

__global__ void __launch_bounds__(256)
out_layer_fwd_tasks_kernel(const float* __restrict__ H, int M, int K, int O,
                           const float* __restrict__ W, const float* __restrict__ bias,
                           const uint8_t* __restrict__ mask, float* __restrict__ scores) {
  out_layer_fwd<true>(H, M, K, O, W, bias, mask, scores);
}

// ------------------------------------------------------- output layer bwd ---
// Rows [z*rows_per, ...): dH[m, k] = (sum_o dS[m, o] W[k, o]) * act'(H[m, k]);
// partial[z][k*O + o] = sum_m H[m, k] dS[m, o]; partial[z][K*O + o] = sum_m dS[m, o].
// kPlanar: dS[m, o] is tw.w[o] * dS[o * M + m], zero on masked rows for every O.
constexpr int kMaxOut = 8;

template <bool kPlanar>
__device__ __forceinline__ void out_layer_bwd(const float* __restrict__ H, int M, int K, int O,
                                              const float* __restrict__ W,
                                              const float* __restrict__ dS,
                                              const uint8_t* __restrict__ mask, int act,
                                              int rows_per, float* __restrict__ dH,
                                              float* __restrict__ partial, size_t partial_stride,
                                              const TaskWeights& tw) {
  const int k = threadIdx.x;
  const int z = blockIdx.x;
  const int mbeg = z * rows_per, mend = min(M, mbeg + rows_per);
  float w[kMaxOut], dw[kMaxOut], db[kMaxOut];
#pragma unroll
  for (int o = 0; o < kMaxOut; ++o) {
    w[o] = (k < K && o < O) ? W[(size_t)k * O + o] : 0.f;
    dw[o] = 0.f;
    db[o] = 0.f;
  }
  for (int m = mbeg; m < mend; ++m) {
    const bool live = !(mask && (kPlanar || O == 1) && !mask[m]);
    float ds[kMaxOut];
    if (kPlanar) {
#pragma unroll
      for (int o = 0; o < kMaxOut; ++o)
        ds[o] = (o < O && live) ? dS[(size_t)o * M + m] * tw.w[o] : 0.f;
    } else {
#pragma unroll
      for (int o = 0; o < kMaxOut; ++o) ds[o] = (o < O && live) ? dS[(size_t)m * O + o] : 0.f;
    }
    if (k < K) {
      const float h = H[(size_t)m * K + k];
      float dh = 0.f;
#pragma unroll
      for (int o = 0; o < kMaxOut; ++o) {
        dh = fmaf(ds[o], w[o], dh);
        dw[o] = fmaf(h, ds[o], dw[o]);
      }
      if (dH) {
        if (act == TFR_ACT_RELU && !(h > 0.f)) dh = 0.f;
        dH[(size_t)m * K + k] = dh;
      }
    }
#pragma unroll
    for (int o = 0; o < kMaxOut; ++o) db[o] += ds[o];
  }
  float* p = partial + (size_t)z * partial_stride;
  if (k < K)
    for (int o = 0; o < O; ++o) p[(size_t)k * O + o] = dw[o];
  if (k == 0)
    for (int o = 0; o < O; ++o) p[(size_t)K * O + o] = db[o];
}

__global__ void __launch_bounds__(1024)
out_layer_bwd_kernel(const float* __restrict__ H, int M, int K, int O,
                     const float* __restrict__ W, const float* __restrict__ dS,
                     const uint8_t* __restrict__ mask, int act, int rows_per,
                     float* __restrict__ dH, float* __restrict__ partial,
                     size_t partial_stride) {
  out_layer_bwd<false>(H, M, K, O, W, dS, mask, act, rows_per, dH, partial, partial_stride,
                       TaskWeights{});
}

__global__ void __launch_bounds__(1024)
out_layer_bwd_tasks_kernel(const float* __restrict__ H, int M, int K, int O,
                           const float* __restrict__ W, const float* __restrict__ dS,
                           const uint8_t* __restrict__ mask, int act, int rows_per,
                           float* __restrict__ dH, float* __restrict__ partial,
                           size_t partial_stride, const TaskWeights tw) {
  out_layer_bwd<true>(H, M, K, O, W, dS, mask, act, rows_per, dH, partial, partial_stride, tw);
}

// partial[z][N cols] column sums of dZ rows handled by split z.
__global__ void __launch_bounds__(256)
colsum_kernel(const float* __restrict__ dZ, int M, int N, int rows_per,
              float* __restrict__ partial, size_t partial_stride, size_t col_offset) {
  const int z = blockIdx.x;
  const int mbeg = z * rows_per, mend = min(M, mbeg + rows_per);
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    float acc = 0.f;
    for (int m = mbeg; m < mend; ++m) acc += dZ[(size_t)m * N + n];
    partial[(size_t)z * partial_stride + col_offset + n] = acc;
  }
}

// out[i] = sum_z partial[z][i]  (deterministic order)
__global__ void __launch_bounds__(256)
reduce_partials_kernel(const float* __restrict__ partial, int splits, size_t stride,
                       size_t n, float* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float acc = 0.f;
#pragma unroll 8
  for (int z = 0; z < splits; ++z) acc += partial[(size_t)z * stride + i];
  out[i] = acc;
}

// Output-layer backward, finer grain: one block per `rows_per` rows, RL row lanes x
// K columns.  Per block b it writes slot[b] = { dW[K*O], db[O], pad to 4, csum[K] } where
// csum[k] = sum_m dH[m, k] (the bias gradient of the last hidden layer).
__global__ void __launch_bounds__(1024)
out_layer_bwd2_kernel(const float* __restrict__ H, int M, int K, int O,
                      const float* __restrict__ W, const float* __restrict__ dS,
                      const uint8_t* __restrict__ mask, int act, int rows_per, int RL,
                      float* __restrict__ dH, float* __restrict__ slots, size_t slot_stride) {
  extern __shared__ float sm[];   // [RL][round4(K * O + O) + K]
  const int KT = blockDim.x / RL;          // threads along k (>= K, multiple of 32)
  const int k = threadIdx.x % KT, rl = threadIdx.x / KT;
  const int mbeg = blockIdx.x * rows_per, mend = min(M, mbeg + rows_per);
  float w[kMaxOut], dw[kMaxOut], db[kMaxOut];
  float csum = 0.f;
#pragma unroll
  for (int o = 0; o < kMaxOut; ++o) {
    w[o] = (k < K && o < O) ? W[(size_t)k * O + o] : 0.f;
    dw[o] = 0.f;
    db[o] = 0.f;
  }
#pragma unroll 4
  for (int m = mbeg + rl; m < mend; m += RL) {
    const bool live = !(mask && O == 1 && !mask[m]);
    float ds[kMaxOut];
#pragma unroll
    for (int o = 0; o < kMaxOut; ++o) ds[o] = (o < O && live) ? dS[(size_t)m * O + o] : 0.f;
    if (k < K) {
      const float h = H[(size_t)m * K + k];
      float dh = 0.f;
#pragma unroll
      for (int o = 0; o < kMaxOut; ++o) {
        dh = fmaf(ds[o], w[o], dh);
        dw[o] = fmaf(h, ds[o], dw[o]);
      }
      if (dH) {
        if (act == TFR_ACT_RELU && !(h > 0.f)) dh = 0.f;
        dH[(size_t)m * K + k] = dh;
        csum += dh;
      }
    }
#pragma unroll
    for (int o = 0; o < kMaxOut; ++o) db[o] += ds[o];
  }
  const int co = (K * O + O + 3) & ~3;      // csum starts 16-byte aligned
  const int per = co + K;
  float* mine = sm + (size_t)rl * per;
  if (k < K) {
    for (int o = 0; o < O; ++o) mine[k * O + o] = dw[o];
    mine[co + k] = csum;
  }
  if (k == 0)
    for (int i = K * O + O; i < co; ++i) mine[i] = 0.f;
  if (k == 0)
    for (int o = 0; o < O; ++o) mine[K * O + o] = db[o];
  __syncthreads();
  float* out = slots + (size_t)blockIdx.x * slot_stride;
  for (int i = threadIdx.x; i < per; i += blockDim.x) {
    float acc = 0.f;
    for (int r = 0; r < RL; ++r) acc += sm[(size_t)r * per + i];
    out[i] = acc;
  }
}

// Same contract for the common single-output scorer (O == 1, K % 4 == 0, K <= 1024):
// a thread owns 4 consecutive k, so H is read and dH written as float4 and a block
// keeps 4x more bytes in flight (the kernel is a pure HBM stream: read H, write dH).
__global__ void __launch_bounds__(256)
out_layer_bwd2_o1_kernel(const float4* __restrict__ H4, int M, int K4,
                         const float4* __restrict__ W4, const float* __restrict__ dS,
                         const uint8_t* __restrict__ mask, int act, int rows_per, int RL,
                         float4* __restrict__ dH4, float* __restrict__ slots,
                         size_t slot_stride) {
  extern __shared__ float sm[];   // [RL][2K + 4]
  const int k4 = threadIdx.x % K4, rl = threadIdx.x / K4;
  const int K = K4 * 4;
  const int mbeg = blockIdx.x * rows_per, mend = min(M, mbeg + rows_per);
  const bool active = rl < RL;
  const float4 w = active ? W4[k4] : make_float4(0.f, 0.f, 0.f, 0.f);
  float4 dw = make_float4(0.f, 0.f, 0.f, 0.f), cs = dw;
  float db = 0.f;
  if (active) {
#pragma unroll 4
    for (int m = mbeg + rl; m < mend; m += RL) {
      const float ds = (mask && !mask[m]) ? 0.f : dS[m];
      const float4 h = H4[(size_t)m * K4 + k4];
      dw.x = fmaf(h.x, ds, dw.x); dw.y = fmaf(h.y, ds, dw.y);
      dw.z = fmaf(h.z, ds, dw.z); dw.w = fmaf(h.w, ds, dw.w);
      db += ds;
      if (dH4) {
        float4 dh = make_float4(ds * w.x, ds * w.y, ds * w.z, ds * w.w);
        if (act == TFR_ACT_RELU) {
          if (!(h.x > 0.f)) dh.x = 0.f;
          if (!(h.y > 0.f)) dh.y = 0.f;
          if (!(h.z > 0.f)) dh.z = 0.f;
          if (!(h.w > 0.f)) dh.w = 0.f;
        }
        dH4[(size_t)m * K4 + k4] = dh;
        cs.x += dh.x; cs.y += dh.y; cs.z += dh.z; cs.w += dh.w;
      }
    }
  }
  const int co = K + 4;                     // { dW[K], db, 3 x pad, csum[K] }
  const int per = co + K;
  if (active) {
    float* mine = sm + (size_t)rl * per;
    mine[4 * k4 + 0] = dw.x; mine[4 * k4 + 1] = dw.y;
    mine[4 * k4 + 2] = dw.z; mine[4 * k4 + 3] = dw.w;
    if (k4 == 0) { mine[K] = db; mine[K + 1] = 0.f; mine[K + 2] = 0.f; mine[K + 3] = 0.f; }
    mine[co + 4 * k4 + 0] = cs.x; mine[co + 4 * k4 + 1] = cs.y;
    mine[co + 4 * k4 + 2] = cs.z; mine[co + 4 * k4 + 3] = cs.w;
  }
  __syncthreads();
  float* out = slots + (size_t)blockIdx.x * slot_stride;
  for (int i = threadIdx.x; i < per; i += blockDim.x) {
    float acc = 0.f;
    for (int r = 0; r < RL; ++r) acc += sm[(size_t)r * per + i];
    out[i] = acc;
  }
}

// The same float4 streaming for 2 <= O <= 4 outputs (groupwise scoring: O = group_size): the
// slot layout is the generic one, { dW[K * O] (k-major, o fastest), db[O], pad to 4, csum[K] }.
// kPlanar (1 <= O <= 8, tfr_mlp_bwd_tasks): the signal is tw.w[o] * dS[o * M + m], zero on
// rows `mask` clears; the interleaved instantiations take no mask.
template <int O, bool kPlanar>
__device__ __forceinline__ void out_layer_bwd2_vec(const float4* __restrict__ H4, int M, int K4,
                                                   const float* __restrict__ W,
                                                   const float* __restrict__ dS, int act,
                                                   int rows_per, int RL,
                                                   float4* __restrict__ dH4,
                                                   float* __restrict__ slots, size_t slot_stride,
                                                   const uint8_t* __restrict__ mask,
                                                   const TaskWeights& tw) {
  extern __shared__ float sm[];   // [RL][round4(K * O + O) + K]
  const int k4 = threadIdx.x % K4, rl = threadIdx.x / K4;
  const int K = K4 * 4;
  const int mbeg = blockIdx.x * rows_per, mend = min(M, mbeg + rows_per);
  const bool active = rl < RL;
  float w[4][O], dw[4][O], cs[4], db[O];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    cs[i] = 0.f;
#pragma unroll
    for (int o = 0; o < O; ++o) {
      w[i][o] = active ? __ldg(W + (size_t)(4 * k4 + i) * O + o) : 0.f;
      dw[i][o] = 0.f;
    }
  }
#pragma unroll
  for (int o = 0; o < O; ++o) db[o] = 0.f;
  if (active) {
#pragma unroll 4
    for (int m = mbeg + rl; m < mend; m += RL) {
      float ds[O];
      if (kPlanar) {
        const bool live = !(mask && !mask[m]);
        const float* q = dS + m;
#pragma unroll
        for (int o = 0; o < O; ++o, q += M) ds[o] = live ? __ldg(q) * tw.w[o] : 0.f;
      } else {
#pragma unroll
        for (int o = 0; o < O; ++o) ds[o] = __ldg(dS + (size_t)m * O + o);
      }
      const float4 h4 = H4[(size_t)m * K4 + k4];
      const float h[4] = {h4.x, h4.y, h4.z, h4.w};
      float dh[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float d = 0.f;
#pragma unroll
        for (int o = 0; o < O; ++o) {
          d = fmaf(ds[o], w[i][o], d);
          dw[i][o] = fmaf(h[i], ds[o], dw[i][o]);
        }
        if (act == TFR_ACT_RELU && !(h[i] > 0.f)) d = 0.f;
        dh[i] = d;
      }
      if (dH4) {
        dH4[(size_t)m * K4 + k4] = make_float4(dh[0], dh[1], dh[2], dh[3]);
#pragma unroll
        for (int i = 0; i < 4; ++i) cs[i] += dh[i];
      }
      if (k4 == 0) {
#pragma unroll
        for (int o = 0; o < O; ++o) db[o] += ds[o];
      }
    }
  }
  const int co = (K * O + O + 3) & ~3;
  const int per = co + K;
  if (active) {
    float* mine = sm + (size_t)rl * per;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
      for (int o = 0; o < O; ++o) mine[(4 * k4 + i) * O + o] = dw[i][o];
      mine[co + 4 * k4 + i] = cs[i];
    }
    if (k4 == 0) {
      for (int i = K * O + O; i < co; ++i) mine[i] = 0.f;
#pragma unroll
      for (int o = 0; o < O; ++o) mine[K * O + o] = db[o];
    }
  }
  __syncthreads();
  float* out = slots + (size_t)blockIdx.x * slot_stride;
  for (int i = threadIdx.x; i < per; i += blockDim.x) {
    float acc = 0.f;
    for (int r = 0; r < RL; ++r) acc += sm[(size_t)r * per + i];
    out[i] = acc;
  }
}

template <int O>
__global__ void __launch_bounds__(256)
out_layer_bwd2_vec_kernel(const float4* __restrict__ H4, int M, int K4, const float* __restrict__ W,
                          const float* __restrict__ dS, int act, int rows_per, int RL,
                          float4* __restrict__ dH4, float* __restrict__ slots,
                          size_t slot_stride) {
  out_layer_bwd2_vec<O, false>(H4, M, K4, W, dS, act, rows_per, RL, dH4, slots, slot_stride,
                               nullptr, TaskWeights{});
}

// (256, 1): lets ptxas keep the O weights and accumulators in registers (it chose 64 and
// spilled at O = 3 without the hint).
template <int O>
__global__ void __launch_bounds__(256, 1)
out_layer_bwd2_vec_tasks_kernel(const float4* __restrict__ H4, int M, int K4,
                                const float* __restrict__ W, const float* __restrict__ dS,
                                int act, int rows_per, int RL, float4* __restrict__ dH4,
                                float* __restrict__ slots, size_t slot_stride,
                                const uint8_t* __restrict__ mask, const TaskWeights tw) {
  out_layer_bwd2_vec<O, true>(H4, M, K4, W, dS, act, rows_per, RL, dH4, slots, slot_stride, mask,
                              tw);
}

// out[i] = sum over slots of srcA (i < nA) or srcB (nA <= i < nA + nB): the weight
// part of a layer gradient comes from the dW split partials, the bias part straight
// from the per-CTA column sums.  16 outputs x 16 slot lanes per block, fixed order.
__global__ void __launch_bounds__(256)
reduce2_kernel(const float* __restrict__ srcA, int slotsA, size_t strideA, size_t nA,
               const float* __restrict__ srcB, int slotsB, size_t strideB, size_t nB,
               float* __restrict__ out) {
  __shared__ float part[16][17];
  const int o = threadIdx.x & 15, sl = threadIdx.x >> 4;
  const size_t i = (size_t)blockIdx.x * 16 + o;
  float acc = 0.f;
  if (i < nA) {
#pragma unroll 4
    for (int z = sl; z < slotsA; z += 16) acc += srcA[(size_t)z * strideA + i];
  } else if (i < nA + nB) {
    const size_t j = i - nA;
#pragma unroll 4
    for (int z = sl; z < slotsB; z += 16) acc += srcB[(size_t)z * strideB + j];
  }
  part[sl][o] = acc;
  __syncthreads();
  if (sl == 0 && i < nA + nB) {
    float t = 0.f;
#pragma unroll
    for (int l = 0; l < 16; ++l) t += part[l][o];
    out[i] = t;
  }
}

// Vector variant: nA, nB, strides multiples of 4 and 16-byte aligned bases.  A thread
// sums one float4 of outputs over its slot lane; 8 float4 outputs x 32 slot lanes.
__global__ void __launch_bounds__(256)
reduce2_vec_kernel(const float4* __restrict__ srcA, int slotsA, size_t strideA4, size_t nA4,
                   const float4* __restrict__ srcB, int slotsB, size_t strideB4, size_t nB4,
                   float4* __restrict__ out) {
  __shared__ float4 part[32][9];
  const unsigned blocksA = (unsigned)((nA4 + 7) / 8);
  if (blockIdx.x >= blocksA) {
    // B part (bias gradients): few outputs, many slots (one per CTA and epilogue warp of the
    // producing GEMM, or one per block of the output-layer backward) -> one float4 per
    // block, 256 slot lanes, fixed-order tree.  (16 lanes per output made this the tail of
    // the launch: ~40 dependent iterations.)
    const size_t j = blockIdx.x - blocksA;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
    for (int z = threadIdx.x; z < slotsB; z += 256) {
      const float4 v = srcB[(size_t)z * strideB4 + j];
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    float4* flat = &part[0][0];          // 288 float4 >= 256
    flat[threadIdx.x] = acc;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
      if ((int)threadIdx.x < w) {
        const float4 a = flat[threadIdx.x], b = flat[threadIdx.x + w];
        flat[threadIdx.x] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) out[nA4 + j] = flat[0];
    return;
  }
  const int o = threadIdx.x & 7, sl = threadIdx.x >> 3;
  const size_t i = (size_t)blockIdx.x * 8 + o;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i < nA4) {
#pragma unroll 4
    for (int z = sl; z < slotsA; z += 32) {
      const float4 v = srcA[(size_t)z * strideA4 + i];
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  part[sl][o] = acc;
  __syncthreads();
  if (sl == 0 && i < nA4) {
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int l = 0; l < 32; ++l) {
      const float4 v = part[l][o];
      t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
    }
    out[i] = t;
  }
}

// One output per block, 256 slot lanes: for few outputs over many slots (the output
// layer's [K * O + O] gradient over ~600 block slots).
__global__ void __launch_bounds__(256)
reduce_tall_kernel(const float* __restrict__ src, int slots, size_t stride, size_t n,
                   float* __restrict__ out) {
  __shared__ float red[32];
  const size_t i = blockIdx.x;
  float acc = 0.f;
#pragma unroll 4
  for (int z = threadIdx.x; z < slots; z += 256) acc += src[(size_t)z * stride + i];
  acc = block_sum(acc, red);
  if (threadIdx.x == 0 && i < n) out[i] = acc;
}

// ------------------------------------------------------------- host side ---
int mlp_reduce2(const float* srcA, int slotsA, size_t strideA, size_t nA, const float* srcB,
                int slotsB, size_t strideB, size_t nB, float* out, cudaStream_t st) {
  const size_t n = nA + nB;
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if (nA % 4 == 0 && nB % 4 == 0 && strideA % 4 == 0 && strideB % 4 == 0 && al16(srcA) &&
      al16(srcB) && al16(out)) {
    reduce2_vec_kernel<<<(unsigned)((nA / 4 + 7) / 8 + nB / 4), 256, 0, st>>>(
        reinterpret_cast<const float4*>(srcA), slotsA, strideA / 4, nA / 4,
        reinterpret_cast<const float4*>(srcB), slotsB, strideB / 4, nB / 4,
        reinterpret_cast<float4*>(out));
    TFR_LAUNCH_OK();
    return TFR_OK;
  }
  if (nB == 0 && slotsA >= 128 && nA <= 4096) {
    reduce_tall_kernel<<<(unsigned)nA, 256, 0, st>>>(srcA, slotsA, strideA, nA, out);
    TFR_LAUNCH_OK();
    return TFR_OK;
  }
  reduce2_kernel<<<(unsigned)((n + 15) / 16), 256, 0, st>>>(srcA, slotsA, strideA, nA, srcB,
                                                          slotsB, strideB, nB, out);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

int mlp_out_layer_bwd2(const float* H, int M, int K, int O, const float* W, const float* dS,
                       const uint8_t* mask, int act, int rows_per, float* dH, float* slots,
                       size_t slot_stride, cudaStream_t st) {
  if (O == 1 && K % 4 == 0 && K <= 1024 && (reinterpret_cast<uintptr_t>(H) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(W) & 15) == 0 && (!dH || (reinterpret_cast<uintptr_t>(dH) & 15) == 0)) {
    const int K4 = K / 4;
    const int RL = 256 / K4;                       // >= 1 (K <= 1024)
    const int blocks = (M + rows_per - 1) / rows_per;
    const size_t smem = (size_t)RL * (2 * K + 4) * sizeof(float);
    if (smem > 48 * 1024)
      TFR_CUDA_OK(cudaFuncSetAttribute(out_layer_bwd2_o1_kernel,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    out_layer_bwd2_o1_kernel<<<blocks, 256, smem, st>>>(
        reinterpret_cast<const float4*>(H), M, K4, reinterpret_cast<const float4*>(W), dS, mask,
        act, rows_per, RL, reinterpret_cast<float4*>(dH), slots, slot_stride);
    TFR_LAUNCH_OK();
    return TFR_OK;
  }
  if (O >= 2 && O <= 4 && !mask && K % 4 == 0 && K <= 1024 &&
      (reinterpret_cast<uintptr_t>(H) & 15) == 0 &&
      (!dH || (reinterpret_cast<uintptr_t>(dH) & 15) == 0)) {
    const int K4 = K / 4;
    const int RL = 256 / K4;
    const int blocks = (M + rows_per - 1) / rows_per;
    const size_t smem = (size_t)RL * (((K * O + O + 3) & ~3) + K) * sizeof(float);
#define TFR_OUT_VEC(O_)                                                                         \
  {                                                                                             \
    if (smem > 48 * 1024)                                                                       \
      TFR_CUDA_OK(cudaFuncSetAttribute(out_layer_bwd2_vec_kernel<O_>,                           \
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    out_layer_bwd2_vec_kernel<O_><<<blocks, 256, smem, st>>>(                                   \
        reinterpret_cast<const float4*>(H), M, K4, W, dS, act, rows_per, RL,                    \
        reinterpret_cast<float4*>(dH), slots, slot_stride);                                     \
  }
    if (O == 2) TFR_OUT_VEC(2)
    else if (O == 3) TFR_OUT_VEC(3)
    else TFR_OUT_VEC(4)
#undef TFR_OUT_VEC
    TFR_LAUNCH_OK();
    return TFR_OK;
  }
  const int K32 = ((K + 31) / 32) * 32;
  int RL = 1, threads = K32;
  if (K32 <= 256) { RL = 256 / K32; threads = RL * K32; }
  const int blocks = (M + rows_per - 1) / rows_per;
  const size_t smem = (size_t)RL * (((K * O + O + 3) & ~3) + K) * sizeof(float);
  if (smem > 48 * 1024)
    TFR_CUDA_OK(cudaFuncSetAttribute(out_layer_bwd2_kernel,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  out_layer_bwd2_kernel<<<blocks, threads, smem, st>>>(H, M, K, O, W, dS, mask, act, rows_per, RL,
                                                      dH, slots, slot_stride);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

int mlp_out_layer_bwd2_tasks(const float* H, int M, int K, int O, const float* W,
                             const float* dS, const TaskWeights& tw, const uint8_t* mask, int act,
                             int rows_per, float* dH, float* slots, size_t slot_stride,
                             cudaStream_t st) {
  const int blocks = (M + rows_per - 1) / rows_per;
  if (K % 4 == 0 && K <= 1024 && (reinterpret_cast<uintptr_t>(H) & 15) == 0 &&
      (!dH || (reinterpret_cast<uintptr_t>(dH) & 15) == 0)) {
    const int K4 = K / 4;
    const int RL = 256 / K4;
    const size_t smem = (size_t)RL * (((K * O + O + 3) & ~3) + K) * sizeof(float);
    auto launch = [&](auto kernel) -> int {
      if (smem > 48 * 1024)
        TFR_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
      kernel<<<blocks, 256, smem, st>>>(reinterpret_cast<const float4*>(H), M, K4, W, dS, act,
                                        rows_per, RL, reinterpret_cast<float4*>(dH), slots,
                                        slot_stride, mask, tw);
      TFR_LAUNCH_OK();
      return TFR_OK;
    };
    switch (O) {
      case 1: return launch(out_layer_bwd2_vec_tasks_kernel<1>);
      case 2: return launch(out_layer_bwd2_vec_tasks_kernel<2>);
      case 3: return launch(out_layer_bwd2_vec_tasks_kernel<3>);
      case 4: return launch(out_layer_bwd2_vec_tasks_kernel<4>);
      case 5: return launch(out_layer_bwd2_vec_tasks_kernel<5>);
      case 6: return launch(out_layer_bwd2_vec_tasks_kernel<6>);
      case 7: return launch(out_layer_bwd2_vec_tasks_kernel<7>);
      default: return launch(out_layer_bwd2_vec_tasks_kernel<8>);
    }
  }
  // An unaligned H is the tower input itself (no hidden layer, no input BN), so there is no
  // dH and no column sums to write: out_layer_bwd_kernel's per-split {dW, db} is the slot
  // prefix that is read.
  TFR_REQUIRE(dH == nullptr, "planar output-layer backward needs a 16-byte aligned H (K = %d)", K);
  out_layer_bwd_tasks_kernel<<<blocks, ((K + 31) / 32) * 32, 0, st>>>(
      H, M, K, O, W, dS, mask, act, rows_per, nullptr, slots, slot_stride, tw);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

int mlp_out_layer_fwd(const float* H, int M, int K, int O, const float* W, const float* bias,
                      const uint8_t* mask, float* scores, cudaStream_t st, bool planar) {
  const int rows_per_block = 32;
  auto kernel = planar ? out_layer_fwd_tasks_kernel : out_layer_fwd_kernel;
  kernel<<<(M + rows_per_block - 1) / rows_per_block, 256, 0, st>>>(H, M, K, O, W, bias, mask,
                                                                     scores);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

int mlp_colsum(const float* dZ, int M, int N, int rows_per, int splits, float* partial,
               size_t pstride, size_t col_offset, cudaStream_t st) {
  colsum_kernel<<<splits, 256, 0, st>>>(dZ, M, N, rows_per, partial, pstride, col_offset);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

int mlp_reduce_partials(const float* partial, int splits, size_t stride, size_t n, float* out,
                        cudaStream_t st) {
  reduce_partials_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(partial, splits, stride, n,
                                                                     out);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

int mlp_simt_fwd(const float* X, int M, const MlpPlan& p, const float* params,
                 const uint8_t* mask, float* ws, float* scores, cudaStream_t st, bool planar) {
  const int L = p.n_dense - 1;  // hidden layers
  const float* in = X;
  if (p.input_bn) {
    int rc = mlp_input_bn_fwd(X, M, p, params, ws, st);
    if (rc) return rc;
    in = ws + p.xin_off;
  }
  for (int d = 0; d < L; ++d) {
    GemmArgs g{};
    g.A = in; g.lda = p.dims[d];
    g.B = params + p.w_off[d]; g.ldb = p.dims[d + 1];
    g.C = ws + (p.use_bn ? p.xhat_off[d] : p.act_off[d]); g.ldc = p.dims[d + 1];
    g.M = M; g.N = p.dims[d + 1]; g.K = p.dims[d];
    g.bias = params + p.b_off[d];
    g.act = p.use_bn ? TFR_ACT_NONE : p.activation;   // BN sits before the activation
    g.k_per_split = g.K; g.split_stride = 0;
    int rc = launch_gemm<false, false, EPI_BIAS_ACT>(g, 1, st);
    if (rc) return rc;
    rc = mlp_hidden_post_fwd(d, M, p, params, ws, st);
    if (rc) return rc;
    in = ws + p.act_off[d];
  }
  const int K = p.dims[L], O = p.dims[L + 1];
  return mlp_out_layer_fwd(in, M, K, O, params + p.w_off[L], params + p.b_off[L], mask, scores,
                           st, planar);
}

int mlp_simt_bwd(const float* X, int M, const MlpPlan& p, const float* params,
                 const float* dscores, const uint8_t* mask, float* ws, float* grads,
                 cudaStream_t st, const TaskWeights* tw) {
  const int L = p.n_dense - 1;
  float* partial = ws + p.partial_off;
  const size_t pstride = p.partial_stride;
  const int rows_per = p.rows_per_split, splits = p.splits;
  float* dz_cur = ws + p.dz_off[0];
  float* dz_nxt = ws + p.dz_off[1];
  const float* X0 = p.input_bn ? ws + p.xin_off : X;   // what Dense 0 consumed
  // With BN / dropout the producers emit raw dL/dH; mlp_hidden_pre_bwd turns it into dL/dZ.
  const int mact = p.post() ? TFR_ACT_NONE : p.activation;

  // output layer
  {
    const int K = p.dims[L], O = p.dims[L + 1];
    const float* H = L > 0 ? ws + p.act_off[L - 1] : X0;
    const int threads = ((K + 31) / 32) * 32;
    const int act = L > 0 ? mact : TFR_ACT_NONE;
    float* dH = (L > 0 || p.input_bn) ? dz_cur : nullptr;
    if (tw)
      out_layer_bwd_tasks_kernel<<<splits, threads, 0, st>>>(
          H, M, K, O, params + p.w_off[L], dscores, mask, act, rows_per, dH, partial, pstride, *tw);
    else
      out_layer_bwd_kernel<<<splits, threads, 0, st>>>(
          H, M, K, O, params + p.w_off[L], dscores, mask, act, rows_per, dH, partial, pstride);
    TFR_LAUNCH_OK();
    const size_t n = (size_t)K * O + O;
    reduce_partials_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(partial, splits, pstride, n,
                                                                       grads + p.w_off[L]);
    TFR_LAUNCH_OK();
  }
  // hidden layers, last to first: dz_cur = dZ_d  [M, dims[d+1]]
  for (int d = L - 1; d >= 0; --d) {
    const int Kin = p.dims[d], Nout = p.dims[d + 1];
    const float* A = d > 0 ? ws + p.act_off[d - 1] : X0;
    if (p.post()) {
      int rc = mlp_hidden_pre_bwd(d, M, p, params, ws, dz_cur, grads, st);
      if (rc) return rc;
    }
    colsum_kernel<<<splits, 256, 0, st>>>(dz_cur, M, Nout, rows_per, partial, pstride,
                                          (size_t)Kin * Nout);
    TFR_LAUNCH_OK();
    {  // dW = A^T dZ, split over rows
      GemmArgs g{};
      g.A = A; g.lda = Kin;           // opA(A)[kin, m] = A[m, kin]
      g.B = dz_cur; g.ldb = Nout;     // [m, nout]
      g.C = partial; g.ldc = Nout;
      g.M = Kin; g.N = Nout; g.K = M;
      g.k_per_split = rows_per; g.split_stride = pstride;
      int rc = launch_gemm<true, false, EPI_NONE>(g, splits, st);
      if (rc) return rc;
    }
    const size_t n = (size_t)Kin * Nout + Nout;
    reduce_partials_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(partial, splits, pstride, n,
                                                                       grads + p.w_off[d]);
    TFR_LAUNCH_OK();
    if (d > 0 || p.input_bn) {  // dZ_{d-1} = (dZ_d W_d^T) * act'(H_{d-1});  d == 0: dL/dXin
      GemmArgs g{};
      g.A = dz_cur; g.lda = Nout;
      g.B = params + p.w_off[d]; g.ldb = Nout;   // opB(B)[nout, kin] = W[kin, nout]
      g.C = dz_nxt; g.ldc = Kin;
      g.M = M; g.N = Kin; g.K = Nout;
      g.aux = d > 0 ? ws + p.act_off[d - 1] : nullptr;
      g.act = d > 0 ? mact : TFR_ACT_NONE;
      g.k_per_split = g.K; g.split_stride = 0;
      int rc = launch_gemm<false, true, EPI_MASK_POS>(g, 1, st);
      if (rc) return rc;
      float* t = dz_cur; dz_cur = dz_nxt; dz_nxt = t;
    }
  }
  if (p.input_bn) return mlp_input_bn_bwd(X, M, p, params, ws, dz_cur, grads, st);
  return TFR_OK;
}

}  // namespace tfr
