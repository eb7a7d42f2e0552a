// K5/K6 companions: BatchNormalization and Dropout of create_tower
// (keras/layers.py:65-76), shared by the fp32 and the tensor-core scorer paths.
//
// Layer order per hidden layer (reference): Dense -> [BN] -> activation -> [Dropout].
//   forward   Z = A W + b  (GEMM)                       -> Z in the xhat buffer
//             mean, var over the M rows (two passes: sum, then centred squares)
//             xhat = (Z - mean) rstd   (kept for backward, in place)
//             H = drop(act(gamma xhat + beta))          -> act buffer
//   backward  dY = dH * keep_scale * [mask from H]      (H > 0 for relu, H != 0 for
//                                                         identity + dropout)
//             dbeta = sum dY, dgamma = sum dY xhat
//             dZ = gamma rstd (dY - mean(dY) - xhat mean(dY xhat))     in place
// tf.keras BatchNormalization on a rank-2 tensor is the non-fused implementation:
// population variance for both the normalisation and the moving average, and
//   moving = moving * momentum + batch * (1 - momentum).
// All passes are HBM-bound column reductions / elementwise sweeps over [M, w].
#include "common.cuh"
#include "mlp.h"

namespace tfr {

namespace {

// ---- column reductions over blocks of rows --------------------------------
// Thread (lane_r, c): columns are contiguous across threads (coalesced rows).
enum RedMode {
  RED_SUM = 0,        // s1 = sum a
  RED_CSQ = 1,        // s1 = sum (a - shift[c])^2
  RED_DY = 2,         // dY = a * scale * mask(h);  s1 = sum dY, s2 = sum dY * b   (b = xhat)
  RED_DXIN = 3        // s1 = sum a, s2 = sum a * (b - shift[c]) * rs[c]          (b = X)
};

__device__ __forceinline__ float keep_mask(float h, int act, bool drop) {
  if (act == TFR_ACT_RELU) return h > 0.f ? 1.f : 0.f;
  if (drop) return h != 0.f ? 1.f : 0.f;
  return 1.f;
}

template <int MODE>
__global__ void __launch_bounds__(256)
col_reduce_kernel(const float* __restrict__ a, const float* __restrict__ b,
                  const float* __restrict__ h, const float* __restrict__ shift,
                  const float* __restrict__ rs, int M, int N, int cw, int rows_per,
                  float scale, int act, int drop, float* __restrict__ part, size_t pstride) {
  __shared__ float sh[2][256];
  const int tid = threadIdx.x;
  const int rl = 256 / cw;               // row lanes
  const int lane_r = tid / cw, c0 = tid % cw;
  const int mbeg = blockIdx.x * rows_per, mend = min(M, mbeg + rows_per);
  float* out = part + (size_t)blockIdx.x * pstride;
  for (int cb = 0; cb < N; cb += cw) {
    const int c = cb + c0;
    float s1 = 0.f, s2 = 0.f;
    if (c < N) {
      const float sft = (MODE == RED_CSQ || MODE == RED_DXIN) ? shift[c] : 0.f;
      const float r = MODE == RED_DXIN ? rs[c] : 0.f;
      for (int m = mbeg + lane_r; m < mend; m += rl) {
        const size_t i = (size_t)m * N + c;
        const float v = a[i];
        if (MODE == RED_SUM) {
          s1 += v;
        } else if (MODE == RED_CSQ) {
          const float t = v - sft;
          s1 = fmaf(t, t, s1);
        } else if (MODE == RED_DY) {
          const float dy = v * scale * keep_mask(h[i], act, drop != 0);
          s1 += dy;
          s2 = fmaf(dy, b[i], s2);
        } else {
          s1 += v;
          s2 = fmaf(v, (b[i] - sft) * r, s2);
        }
      }
    }
    sh[0][tid] = s1;
    sh[1][tid] = s2;
    __syncthreads();
    if (lane_r == 0 && c < N) {
      for (int j = 1; j < rl; ++j) {
        s1 += sh[0][j * cw + c0];
        s2 += sh[1][j * cw + c0];
      }
      out[c] = s1;
      if (MODE >= RED_DY) out[N + c] = s2;
    }
    __syncthreads();
  }
}

// Sums `nblk` partial rows per output; 16 lanes per output (same scheme as reduce2).
__device__ __forceinline__ float sum_partials(const float* __restrict__ part, int nblk,
                                              size_t pstride, int col, int lane16) {
  float s = 0.f;
  for (int z = lane16; z < nblk; z += 16) s += part[(size_t)z * pstride + col];
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o, 16);
  return s;
}

// mode 0: stat[c] = mean.
// mode 1: stat[N + c] = rstd; moving averages updated (training).
__global__ void __launch_bounds__(256)
bn_fwd_finalize_kernel(const float* __restrict__ part, int nblk, size_t pstride, int N, int M,
                       int mode, float eps, float mom, float* __restrict__ stat,
                       float* __restrict__ moving) {
  const int lane16 = threadIdx.x & 15;
  const int c = blockIdx.x * 16 + (threadIdx.x >> 4);
  const bool live = c < N;
  const float s = sum_partials(part, nblk, pstride, live ? c : 0, lane16);
  if (!live || lane16 != 0) return;
  if (mode == 0) {
    stat[c] = s / (float)M;
  } else {
    const float var = s / (float)M;
    stat[N + c] = rsqrtf(var + eps);
    moving[c] = moving[c] * mom + stat[c] * (1.f - mom);
    moving[N + c] = moving[N + c] * mom + var * (1.f - mom);
  }
}

// Inference: batch statistics replaced by the moving ones.
__global__ void __launch_bounds__(256)
bn_stat_from_moving_kernel(const float* __restrict__ moving, int N, float eps,
                           float* __restrict__ stat) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= N) return;
  stat[c] = moving[c];
  stat[N + c] = rsqrtf(moving[N + c] + eps);
}

// Counter-based uniform in [0, 1): splitmix64 of (seed, layer, element).
__device__ __forceinline__ float uniform01(unsigned long long seed, unsigned long long idx) {
  unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (idx + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (float)(z >> 40) * (1.0f / 16777216.0f);
}

// H = drop(act(gamma * xhat + beta)); BN == false: H = drop(H) in place (z unused).
template <bool BN>
__global__ void __launch_bounds__(256)
post_fwd_kernel(float* __restrict__ z, float* __restrict__ H, const float* __restrict__ stat,
                const float* __restrict__ gamma, const float* __restrict__ beta, size_t total,
                int N, int act, float drop, unsigned long long seed) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % N);
  float v;
  if (BN) {
    const float xh = (z[i] - stat[c]) * stat[N + c];
    z[i] = xh;
    v = fmaf(gamma[c], xh, beta[c]);
    if (act == TFR_ACT_RELU) v = fmaxf(v, 0.f);
  } else {
    v = H[i];
  }
  if (drop > 0.f) v = uniform01(seed, i) < drop ? 0.f : v * (1.f / (1.f - drop));
  H[i] = v;
}

// Input BN: Xin = gamma * (X - mean) * rstd + beta.
__global__ void __launch_bounds__(256)
input_bn_apply_kernel(const float* __restrict__ X, float* __restrict__ Xin,
                      const float* __restrict__ stat, const float* __restrict__ gamma,
                      const float* __restrict__ beta, size_t total, int N) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % N);
  Xin[i] = fmaf(gamma[c], (X[i] - stat[c]) * stat[N + c], beta[c]);
}

// dbeta = s1, dgamma = s2; coef[c] = s1 / M, coef[N + c] = s2 / M (zero in inference:
// the statistics are constants there).
__global__ void __launch_bounds__(256)
bn_bwd_finalize_kernel(const float* __restrict__ part, int nblk, size_t pstride, int N, int M,
                       int training, float* __restrict__ dgamma, float* __restrict__ dbeta,
                       float* __restrict__ coef) {
  const int lane16 = threadIdx.x & 15;
  const int c = blockIdx.x * 16 + (threadIdx.x >> 4);
  const bool live = c < N;
  const float s1 = sum_partials(part, nblk, pstride, live ? c : 0, lane16);
  const float s2 = sum_partials(part, nblk, pstride, N + (live ? c : 0), lane16);
  if (!live || lane16 != 0) return;
  dbeta[c] = s1;
  dgamma[c] = s2;
  if (coef) {
    coef[c] = training ? s1 / (float)M : 0.f;
    coef[N + c] = training ? s2 / (float)M : 0.f;
  }
}

// dz: dH -> dZ in place.
template <bool BN>
__global__ void __launch_bounds__(256)
pre_bwd_kernel(float* __restrict__ dz, const float* __restrict__ H,
               const float* __restrict__ xhat, const float* __restrict__ stat,
               const float* __restrict__ gamma, const float* __restrict__ coef, size_t total,
               int N, int act, float drop) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float scale = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  float dy = dz[i] * scale * keep_mask(H[i], act, drop > 0.f);
  if (BN) {
    const int c = (int)(i % N);
    dy = gamma[c] * stat[N + c] * (dy - coef[c] - xhat[i] * coef[N + c]);
  }
  dz[i] = dy;
}

int col_width(int N) {
  int cw = 32;
  while (cw < N && cw < 256) cw <<= 1;
  return cw;
}

inline unsigned blocks_for(size_t total) { return (unsigned)((total + 255) / 256); }

// Batch statistics of src [M, N] into stat (mean, rstd), updating `moving`.
int batch_stats(const float* src, int M, int N, const MlpPlan& p, float* ws, float* stat,
                float* moving, cudaStream_t st) {
  if (!p.training) {
    bn_stat_from_moving_kernel<<<(N + 255) / 256, 256, 0, st>>>(moving, N, p.bn_eps, stat);
    TFR_LAUNCH_OK();
    return TFR_OK;
  }
  float* part = ws + p.red_off;
  const int cw = col_width(N);
  col_reduce_kernel<RED_SUM><<<p.red_blocks, 256, 0, st>>>(
      src, nullptr, nullptr, nullptr, nullptr, M, N, cw, p.red_rows, 1.f, 0, 0, part,
      p.red_stride);
  TFR_LAUNCH_OK();
  bn_fwd_finalize_kernel<<<(N + 15) / 16, 256, 0, st>>>(part, p.red_blocks, p.red_stride, N, M, 0,
                                                       p.bn_eps, p.bn_mom, stat, moving);
  TFR_LAUNCH_OK();
  col_reduce_kernel<RED_CSQ><<<p.red_blocks, 256, 0, st>>>(
      src, nullptr, nullptr, stat, nullptr, M, N, cw, p.red_rows, 1.f, 0, 0, part, p.red_stride);
  TFR_LAUNCH_OK();
  bn_fwd_finalize_kernel<<<(N + 15) / 16, 256, 0, st>>>(part, p.red_blocks, p.red_stride, N, M, 1,
                                                       p.bn_eps, p.bn_mom, stat, moving);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

}  // namespace

int mlp_hidden_post_fwd(int d, int M, const MlpPlan& p, const float* params, float* ws,
                        cudaStream_t st) {
  const int N = p.dims[d + 1];
  const size_t total = (size_t)M * N;
  float* H = ws + p.act_off[d];
  const float drop = p.training ? p.dropout : 0.f;
  // one dropout stream per layer: fold the layer index into the seed
  const unsigned long long seed = p.seed * 0x100000001B3ull + (unsigned long long)(d + 1);
  if (p.use_bn) {
    float* z = ws + p.xhat_off[d];
    float* stat = ws + p.bnstat_off[d];
    int rc = batch_stats(z, M, N, p, ws, stat, p.bn_state + p.st_off[d], st);
    if (rc) return rc;
    post_fwd_kernel<true><<<blocks_for(total), 256, 0, st>>>(
        z, H, stat, params + p.g_off[d], params + p.be_off[d], total, N, p.activation, drop, seed);
    TFR_LAUNCH_OK();
  } else if (drop > 0.f) {
    post_fwd_kernel<false><<<blocks_for(total), 256, 0, st>>>(
        nullptr, H, nullptr, nullptr, nullptr, total, N, p.activation, drop, seed);
    TFR_LAUNCH_OK();
  }
  return TFR_OK;
}

int mlp_hidden_pre_bwd(int d, int M, const MlpPlan& p, const float* params, float* ws,
                       float* dz, float* grads, cudaStream_t st) {
  const int N = p.dims[d + 1];
  const size_t total = (size_t)M * N;
  const float* H = ws + p.act_off[d];
  const float drop = p.training ? p.dropout : 0.f;
  if (p.use_bn) {
    const float* xhat = ws + p.xhat_off[d];
    const float* stat = ws + p.bnstat_off[d];
    float* part = ws + p.red_off;
    float* coef = part + (size_t)p.red_blocks * p.red_stride;
    const float scale = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
    col_reduce_kernel<RED_DY><<<p.red_blocks, 256, 0, st>>>(
        dz, xhat, H, nullptr, nullptr, M, N, col_width(N), p.red_rows, scale, p.activation,
        drop > 0.f, part, p.red_stride);
    TFR_LAUNCH_OK();
    bn_bwd_finalize_kernel<<<(N + 15) / 16, 256, 0, st>>>(
        part, p.red_blocks, p.red_stride, N, M, p.training, grads + p.g_off[d],
        grads + p.be_off[d], coef);
    TFR_LAUNCH_OK();
    pre_bwd_kernel<true><<<blocks_for(total), 256, 0, st>>>(
        dz, H, xhat, stat, params + p.g_off[d], coef, total, N, p.activation, drop);
    TFR_LAUNCH_OK();
  } else {
    pre_bwd_kernel<false><<<blocks_for(total), 256, 0, st>>>(
        dz, H, nullptr, nullptr, nullptr, nullptr, total, N, p.activation, drop);
    TFR_LAUNCH_OK();
  }
  return TFR_OK;
}

int mlp_bn_batch_stats(const float* src, int M, int N, const MlpPlan& p, float* ws, float* stat,
                       float* moving, cudaStream_t st) {
  return batch_stats(src, M, N, p, ws, stat, moving, st);
}

int mlp_input_bn_fwd(const float* X, int M, const MlpPlan& p, const float* params, float* ws,
                     cudaStream_t st) {
  const int N = p.dims[0];
  float* stat = ws + p.bnstat_in_off;
  int rc = batch_stats(X, M, N, p, ws, stat, p.bn_state + p.stin_off, st);
  if (rc) return rc;
  const size_t total = (size_t)M * N;
  input_bn_apply_kernel<<<blocks_for(total), 256, 0, st>>>(
      X, ws + p.xin_off, stat, params + p.gin_off, params + p.bein_off, total, N);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

int mlp_input_bn_bwd(const float* X, int M, const MlpPlan& p, const float* params, float* ws,
                     const float* dxin, float* grads, cudaStream_t st) {
  const int N = p.dims[0];
  const float* stat = ws + p.bnstat_in_off;
  float* part = ws + p.red_off;
  col_reduce_kernel<RED_DXIN><<<p.red_blocks, 256, 0, st>>>(
      dxin, X, nullptr, stat, stat + N, M, N, col_width(N), p.red_rows, 1.f, 0, 0, part,
      p.red_stride);
  TFR_LAUNCH_OK();
  bn_bwd_finalize_kernel<<<(N + 15) / 16, 256, 0, st>>>(
      part, p.red_blocks, p.red_stride, N, M, p.training, grads + p.gin_off,
      grads + p.bein_off, nullptr);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

}  // namespace tfr
