// C-ABI glue: error string, scorer-tower dispatch, fused optimizer.
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstring>

#include "common.cuh"
#include "mlp.h"

namespace tfr {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static unsigned long long g_launches = 0;
void count_launch() { __atomic_add_fetch(&g_launches, 1ull, __ATOMIC_RELAXED); }

int num_sms() {
  static int n = 0;
  if (n <= 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      return 132;   // no device to ask (e.g. planning on a CPU-only build machine)
  }
  return n;
}

size_t smem_optin_limit() {
  // one cached value per device ordinal; racing first calls store the same value
  constexpr int kMaxDevices = 64;
  static std::atomic<size_t> cache[kMaxDevices];
  int dev = 0, v = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    (void)cudaGetLastError();
    return 48 * 1024;   // no device to ask: the limit every device grants without opt-in
  }
  if (dev >= 0 && dev < kMaxDevices) {
    const size_t hit = cache[dev].load(std::memory_order_relaxed);
    if (hit != 0) return hit;
  }
  if (cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
      v <= 0) {
    (void)cudaGetLastError();
    return 48 * 1024;
  }
  if (dev >= 0 && dev < kMaxDevices) cache[dev].store((size_t)v, std::memory_order_relaxed);
  return (size_t)v;
}

static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

int make_mlp_plan(const tfr_mlp_cfg* cfg, int M, MlpPlan* p) {
  TFR_REQUIRE(cfg != nullptr, "cfg must not be NULL");
  TFR_REQUIRE(cfg->n_dense >= 1 && cfg->n_dense <= TFR_MLP_MAX_LAYERS,
              "n_dense %d must be in [1, %d]", cfg->n_dense, TFR_MLP_MAX_LAYERS);
  TFR_REQUIRE(M >= 0, "M must be >= 0");
  TFR_REQUIRE(cfg->activation == TFR_ACT_NONE || cfg->activation == TFR_ACT_RELU,
              "activation %d unsupported", cfg->activation);
  for (int i = 0; i <= cfg->n_dense; ++i)
    TFR_REQUIRE(cfg->dims[i] >= 1, "dims[%d] = %d must be >= 1", i, cfg->dims[i]);
  const int L = cfg->n_dense - 1;
  TFR_REQUIRE(cfg->dims[L] <= 1024, "width %d feeding the output layer exceeds 1024", cfg->dims[L]);
  TFR_REQUIRE(cfg->dims[L + 1] <= 8, "output_units %d exceeds 8", cfg->dims[L + 1]);
  std::memset(p, 0, sizeof(*p));
  p->n_dense = cfg->n_dense;
  p->activation = cfg->activation;
  size_t off = 0, max_wb = 0;
  int max_hidden = 1;
  for (int d = 0; d <= cfg->n_dense; ++d) p->dims[d] = cfg->dims[d];
  for (int d = 0; d < cfg->n_dense; ++d) {
    p->w_off[d] = off;
    off += (size_t)p->dims[d] * p->dims[d + 1];
    p->b_off[d] = off;
    off += p->dims[d + 1];
    // (rows rounded up to 128: the bf16 dW GEMM stores whole 128-row blocks per split)
    const size_t wb = (size_t)((p->dims[d] + 127) / 128 * 128) * p->dims[d + 1] + p->dims[d + 1];
    if (wb > max_wb) max_wb = wb;
    if (d < L && p->dims[d + 1] > max_hidden) max_hidden = p->dims[d + 1];
  }
  // BatchNormalization / Dropout options
  TFR_REQUIRE(cfg->dropout >= 0.f && cfg->dropout < 1.f, "dropout %g must be in [0, 1)",
              (double)cfg->dropout);
  p->use_bn = cfg->use_batch_norm != 0 && L > 0;
  p->input_bn = cfg->input_batch_norm != 0;
  p->training = cfg->training != 0;
  p->bn_eps = cfg->bn_epsilon;
  p->bn_mom = cfg->bn_momentum;
  p->dropout = L > 0 ? cfg->dropout : 0.f;
  p->seed = cfg->dropout_seed;
  p->bn_state = cfg->bn_state;
  if (p->use_bn || p->input_bn) {
    TFR_REQUIRE(cfg->bn_epsilon > 0.f, "bn_epsilon must be > 0");
    TFR_REQUIRE(cfg->bn_momentum >= 0.f && cfg->bn_momentum <= 1.f,
                "bn_momentum %g must be in [0, 1]", (double)cfg->bn_momentum);
  }
  size_t soff = 0;
  int max_bn_w = 1;
  if (p->input_bn) {
    p->gin_off = off; off += p->dims[0];
    p->bein_off = off; off += p->dims[0];
    p->stin_off = soff; soff += 2 * (size_t)p->dims[0];
    max_bn_w = p->dims[0];
  }
  if (p->use_bn)
    for (int d = 0; d < L; ++d) {
      p->g_off[d] = off; off += p->dims[d + 1];
      p->be_off[d] = off; off += p->dims[d + 1];
      p->st_off[d] = soff; soff += 2 * (size_t)p->dims[d + 1];
      if (p->dims[d + 1] > max_bn_w) max_bn_w = p->dims[d + 1];
    }
  p->n_state = soff;
  p->n_params = off;
  // workspace
  size_t w = 0;
  for (int d = 0; d < L; ++d) {
    p->act_off[d] = w;
    w += align_up((size_t)M * p->dims[d + 1], 64);
    p->bits_off[d] = w;
    w += align_up((size_t)M * ((p->dims[d + 1] + 31) / 32), 64);
  }
  if (p->use_bn)
    for (int d = 0; d < L; ++d) {
      p->xhat_off[d] = w;
      w += align_up((size_t)M * p->dims[d + 1], 64);
      p->bnstat_off[d] = w;
      w += align_up(2 * (size_t)p->dims[d + 1], 64);
    }
  if (p->input_bn) {
    p->xin_off = w;
    w += align_up((size_t)M * p->dims[0], 64);
    p->bnstat_in_off = w;
    w += align_up(2 * (size_t)p->dims[0], 64);
    if (p->dims[0] > max_hidden) max_hidden = p->dims[0];   // dZ ping-pong also holds dL/dXin
  }
  if (p->use_bn || p->input_bn) {
    p->red_rows = 256;
    p->red_blocks = M > 0 ? (M + p->red_rows - 1) / p->red_rows : 1;
    p->red_stride = align_up(2 * (size_t)max_bn_w, 64);
    p->red_off = w;
    w += (size_t)p->red_blocks * p->red_stride + align_up(2 * (size_t)max_bn_w, 64);
  }
  for (int i = 0; i < 2; ++i) {
    p->dz_off[i] = w;
    w += align_up((size_t)M * max_hidden, 64);
  }
  const int sms = num_sms();
  // Row splits of the dW GEMMs / bias partials: about one per SM, so that the persistent
  // GEMM has a split for every SM even when the dW output is one or two 128 x 128 tiles.
  {
    const int per = (M + sms - 1) / sms;
    p->rows_per_split = per < 256 ? 256 : ((per + 127) / 128) * 128;
    p->splits = M > 0 ? (M + p->rows_per_split - 1) / p->rows_per_split : 1;
  }
  p->partial_stride = align_up(max_wb, 64);
  p->partial_off = w;
  w += (size_t)p->splits * p->partial_stride;
  p->whi_off = w;
  w += align_up(p->n_params, 64);
  p->wlo_off = w;
  w += align_up(p->n_params, 64);
  p->wthi_off = w;
  w += align_up(p->n_params, 64);
  p->wtlo_off = w;
  w += align_up(p->n_params, 64);
  // column-sum slots: 8 warps x persistent GEMM CTAs (one per SM; room for 512 SMs), or one
  // per row split (about one per SM)
  p->tile_slots = 4 * 1024;
  p->tile_stride = align_up((size_t)max_hidden, 64);
  p->tile_off = w;
  w += (size_t)p->tile_slots * p->tile_stride;
  // output-layer backward: about 4 blocks per SM, each owning one slot
  p->out_rows = M > 0 ? ((M + 4 * sms - 1) / (4 * sms) + 3) / 4 * 4 : 4;
  if (p->out_rows < 16) p->out_rows = 16;
  p->out_slots = (M + p->out_rows - 1) / p->out_rows;
  p->oslot_stride = align_up((size_t)p->dims[L] * (p->dims[L + 1] + 1) + p->dims[L + 1] + 4, 64);
  p->oslot_off = w;
  w += (size_t)p->out_slots * p->oslot_stride;
  p->ws_floats = w;
  return TFR_OK;
}

__global__ void __launch_bounds__(256)
optimizer_kernel(float* __restrict__ params, const float* __restrict__ grads,
                 float* __restrict__ accum, size_t n, int kind, float lr, float eps,
                 float grad_scale) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float g = grads[i] * grad_scale;
  if (kind == 0) {
    params[i] -= lr * g;
  } else {
    // tf.keras.optimizers.Adagrad: accum += g^2; var -= lr * g / (sqrt(accum) + eps)
    const float a = accum[i] + g * g;
    accum[i] = a;
    params[i] -= lr * g / (sqrtf(a) + eps);
  }
}


// AdamWeightDecay; step_size = lr sqrt(1 - beta2^t) / (1 - beta1^t) (host, double).
// Clip: g is scaled by the global-norm factor read from *norm (the header's contract); the
// factor is exactly 1 when the norm is within clip_norm, so those steps keep the unclipped bits.
template <bool Clip>
__global__ void __launch_bounds__(256)
adamw_kernel(float* __restrict__ params, const float* __restrict__ grads, float* __restrict__ m,
             float* __restrict__ v, const uint8_t* __restrict__ decay_mask, size_t n, float lr,
             float beta1, float beta2, float eps, float wd, float step_size, float grad_scale,
             float clip_norm, const float* __restrict__ norm) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float g = grads[i] * grad_scale;
  if (Clip) {
    const float nrm = *norm;
    // tf.clip_by_global_norm: an inf or NaN norm makes every clipped gradient NaN
    const float s = !isfinite(nrm) ? __int_as_float(0x7fc00000)
                                   : (nrm <= clip_norm ? 1.f : clip_norm / nrm);
    g *= s;
  }
  const float mi = beta1 * m[i] + (1.f - beta1) * g;
  const float vi = beta2 * v[i] + (1.f - beta2) * g * g;
  m[i] = mi;
  v[i] = vi;
  float p = params[i];
  if (!decay_mask || decay_mask[i]) p -= lr * wd * p;
  params[i] = p - step_size * mi / (sqrtf(vi) + eps);
}

// Loss-scaled AdamW (the header's dynamic loss scale rule): the step is skipped -- params, m
// and v left as they are -- when *norm (the global norm of the scaled gradient) is inf or NaN;
// otherwise g = grads * (1 / S) with S = *scale, clipped on the unscaled norm when clip_norm > 0,
// then the update of adamw_kernel.  A kernel of its own, so adamw_kernel's code is unchanged.
__global__ void __launch_bounds__(256)
adamw_scaled_kernel(float* __restrict__ params, const float* __restrict__ grads,
                    float* __restrict__ m, float* __restrict__ v,
                    const uint8_t* __restrict__ decay_mask, size_t n, float lr, float beta1,
                    float beta2, float eps, float wd, float step_size, float clip_norm,
                    const float* __restrict__ norm, const float* __restrict__ scale) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const float nrm = *norm;
  if (i >= n || !isfinite(nrm)) return;
  const float S = *scale;
  float g = grads[i] * (1.f / S);
  if (clip_norm > 0.f) {
    const float nu = (float)((double)nrm / (double)S);
    g *= nu <= clip_norm ? 1.f : clip_norm / nu;
  }
  const float mi = beta1 * m[i] + (1.f - beta1) * g;
  const float vi = beta2 * v[i] + (1.f - beta2) * g * g;
  m[i] = mi;
  v[i] = vi;
  float p = params[i];
  if (!decay_mask || decay_mask[i]) p -= lr * wd * p;
  params[i] = p - step_size * mi / (sqrtf(vi) + eps);
}

// out = x * *scale (out may alias x).
__global__ void __launch_bounds__(256)
loss_scale_mul_kernel(const float* x, size_t n, const float* __restrict__ scale, float* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = x[i] * *scale;
}

// One thread, after the step that read the old scale: the unscaled norm, then the dynamic
// rule's new scale and good-step count (growth_steps 0: a fixed scale, left as it is).
__global__ void __launch_bounds__(32)
loss_scale_update_kernel(float* scale, int64_t* good_steps, const float* __restrict__ norm,
                         float* unscaled_norm, int64_t growth_steps) {
  if (threadIdx.x != 0) return;
  const float S = *scale, nrm = *norm;
  if (unscaled_norm) *unscaled_norm = (float)((double)nrm / (double)S);
  if (growth_steps <= 0) return;
  if (!isfinite(nrm)) {
    *scale = fmaxf(S * 0.5f, 1.f);
    *good_steps = 0;
    return;
  }
  const int64_t c = *good_steps + 1;
  if (c >= growth_steps) {
    const float grown = S * 2.f;
    if (isfinite(grown)) *scale = grown;
    *good_steps = 0;
  } else {
    *good_steps = c;
  }
}

// Global L2 norm, in two fixed-order passes.  Pass 1: thread t of block b sums squares (in
// double) over fixed positions p = b * 256 + t + k * norm_blocks(n) * 256 -- float4 number p
// when x is 16-byte aligned (the n % 4 tail elements then go to the first threads of block 0),
// float number p otherwise -- and the block reduces them in a fixed tree.  Pass 2: one block
// sums the per-block partials the same way and writes sqrt as float.
constexpr int kNormThreads = 256;
constexpr int kNormPerThread = 16;   // elements per thread before the grid saturates
constexpr int kNormMaxBlocks = 2048;

static unsigned norm_blocks(size_t n) {
  const size_t per_block = (size_t)kNormThreads * kNormPerThread;
  const size_t b = (n + per_block - 1) / per_block;
  return (unsigned)(b < 1 ? 1 : (b > kNormMaxBlocks ? kNormMaxBlocks : b));
}

__device__ __forceinline__ double block_sum_fixed(double x, double* sh) {
  // fixed shuffle tree inside each warp, then warp 0 over the warp sums in warp order
  for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) sh[warp] = x;
  __syncthreads();
  x = 0.0;
  if (warp == 0) {
    const int nw = blockDim.x >> 5;
    x = lane < nw ? sh[lane] : 0.0;
    for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
  }
  return x;   // valid in thread 0
}

__global__ void __launch_bounds__(kNormThreads)
sumsq_partials_kernel(const float* __restrict__ x, size_t n, double* __restrict__ partials) {
  __shared__ double sh[kNormThreads / 32];
  const size_t stride = (size_t)gridDim.x * kNormThreads;
  const size_t first = (size_t)blockIdx.x * kNormThreads + threadIdx.x;
  double a0 = 0.0, a1 = 0.0;   // two chains, so the FMA latency does not throttle the loads
  if ((reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    const float4* __restrict__ x4 = reinterpret_cast<const float4*>(x);
    const size_t n4 = n >> 2;
#pragma unroll 2
    for (size_t i = first; i < n4; i += stride) {
      const float4 v = __ldg(x4 + i);
      a0 = fma((double)v.x, (double)v.x, a0);
      a1 = fma((double)v.y, (double)v.y, a1);
      a0 = fma((double)v.z, (double)v.z, a0);
      a1 = fma((double)v.w, (double)v.w, a1);
    }
    if (first < (n & 3)) {
      const double v = (double)__ldg(x + (n4 << 2) + first);
      a0 = fma(v, v, a0);
    }
  } else {
#pragma unroll 4
    for (size_t i = first; i < n; i += stride) {
      const double v = (double)__ldg(x + i);
      a0 = fma(v, v, a0);
    }
  }
  const double acc = block_sum_fixed(a0 + a1, sh);
  if (threadIdx.x == 0) partials[blockIdx.x] = acc;
}

__global__ void __launch_bounds__(1024)
norm_final_kernel(const double* __restrict__ partials, int nparts, float* __restrict__ norm) {
  __shared__ double sh[32];
  double acc = 0.0;
  for (int i = threadIdx.x; i < nparts; i += blockDim.x) acc += partials[i];
  acc = block_sum_fixed(acc, sh);
  if (threadIdx.x == 0) *norm = (float)sqrt(acc);
}
}  // namespace tfr

using namespace tfr;

extern "C" const char* tfr_last_error(void) { return g_err; }
extern "C" int tfr_version(void) { return 2; }
extern "C" unsigned long long tfr_launch_count(void) {
  return __atomic_load_n(&g_launches, __ATOMIC_RELAXED);
}

extern "C" size_t tfr_mlp_param_count(const tfr_mlp_cfg* cfg) {
  MlpPlan p;
  if (make_mlp_plan(cfg, 0, &p)) return 0;
  return p.n_params;
}

extern "C" size_t tfr_mlp_bn_state_count(const tfr_mlp_cfg* cfg) {
  MlpPlan p;
  if (make_mlp_plan(cfg, 0, &p)) return 0;
  return p.n_state;
}

extern "C" size_t tfr_mlp_workspace_bytes(const tfr_mlp_cfg* cfg, int M) {
  MlpPlan p;
  if (make_mlp_plan(cfg, M, &p)) return 0;
  return p.ws_floats * sizeof(float) + 256;
}

static float* ws_base(void* workspace) {
  uintptr_t a = reinterpret_cast<uintptr_t>(workspace);
  a = (a + 255) & ~(uintptr_t)255;
  return reinterpret_cast<float*>(a);
}

extern "C" int tfr_mlp_fwd(const void* Xv, int M, const tfr_mlp_cfg* cfg,
                           const float* params, const uint8_t* mask, void* workspace,
                           float* scores_out, int precision, void* stream) {
  MlpPlan p;
  int rc = make_mlp_plan(cfg, M, &p);
  if (rc) return rc;
  const float* X = static_cast<const float*>(Xv);   // bf16 when precision == TFR_PREC_BF16
  TFR_REQUIRE(X && params && workspace && scores_out, "NULL argument");
  TFR_REQUIRE(!(p.use_bn || p.input_bn) || p.bn_state, "cfg->bn_state must be set with BN");
  if (M == 0) return TFR_OK;
  switch (precision) {
    case TFR_PREC_FP32:
      return mlp_simt_fwd(X, M, p, params, mask, ws_base(workspace), scores_out,
                          (cudaStream_t)stream);
    case TFR_PREC_TF32X3:
    case TFR_PREC_TF32:
      return mlp_tc_fwd(X, M, p, params, mask, ws_base(workspace), scores_out,
                        precision == TFR_PREC_TF32X3 ? 3 : 1, (cudaStream_t)stream);
    case TFR_PREC_BF16:
      return mlp_bf16_fwd(Xv, M, p, params, mask, ws_base(workspace), scores_out,
                          (cudaStream_t)stream);
    default:
      set_error("precision %d is not available in this build", precision);
      return TFR_UNSUPPORTED;
  }
}

extern "C" int tfr_mlp_bwd(const void* Xv, int M, const tfr_mlp_cfg* cfg,
                           const float* params, const float* dscores, const uint8_t* mask,
                           void* workspace, float* grads, int precision, void* stream) {
  MlpPlan p;
  int rc = make_mlp_plan(cfg, M, &p);
  if (rc) return rc;
  const float* X = static_cast<const float*>(Xv);
  TFR_REQUIRE(X && params && workspace && dscores && grads, "NULL argument");
  TFR_REQUIRE(!(p.use_bn || p.input_bn) || p.bn_state, "cfg->bn_state must be set with BN");
  if (M == 0) {   // an empty shard contributes a zero gradient (never stale memory)
    TFR_CUDA_OK(cudaMemsetAsync(grads, 0, p.n_params * sizeof(float), (cudaStream_t)stream));
    return TFR_OK;
  }
  switch (precision) {
    case TFR_PREC_FP32:
      return mlp_simt_bwd(X, M, p, params, dscores, mask, ws_base(workspace), grads,
                          (cudaStream_t)stream);
    case TFR_PREC_TF32X3:
    case TFR_PREC_TF32:
      return mlp_tc_bwd(X, M, p, params, dscores, mask, ws_base(workspace), grads,
                        precision == TFR_PREC_TF32X3 ? 3 : 1, (cudaStream_t)stream);
    case TFR_PREC_BF16:
      return mlp_bf16_bwd(Xv, M, p, params, dscores, mask, ws_base(workspace), grads,
                          (cudaStream_t)stream);
    default:
      set_error("precision %d is not available in this build", precision);
      return TFR_UNSUPPORTED;
  }
}

// Limits of the task-major entry points, checked before any CUDA call (make_mlp_plan asks the
// device for its SM count).
static int check_tasks_args(const tfr_mlp_cfg* cfg, int precision) {
  TFR_REQUIRE(cfg != nullptr, "cfg must not be NULL");
  TFR_REQUIRE(cfg->n_dense >= 1 && cfg->n_dense <= TFR_MLP_MAX_LAYERS,
              "n_dense %d must be in [1, %d]", cfg->n_dense, TFR_MLP_MAX_LAYERS);
  const int O = cfg->dims[cfg->n_dense];
  TFR_REQUIRE(O >= 1 && O <= 8, "task count (output_units) %d must be in [1, 8]", O);
  TFR_REQUIRE(precision == TFR_PREC_FP32 || precision == TFR_PREC_TF32X3 ||
                  precision == TFR_PREC_TF32,
              "task-major scores need precision fp32, tf32x3 or tf32 (got %d)", precision);
  return TFR_OK;
}

extern "C" int tfr_mlp_fwd_tasks(const void* Xv, int M, const tfr_mlp_cfg* cfg,
                                 const float* params, const uint8_t* mask, void* workspace,
                                 float* score_planes, int precision, void* stream) {
  int rc = check_tasks_args(cfg, precision);
  if (rc) return rc;
  const float* X = static_cast<const float*>(Xv);
  TFR_REQUIRE(X && params && workspace && score_planes, "NULL argument");
  MlpPlan p;
  rc = make_mlp_plan(cfg, M, &p);
  if (rc) return rc;
  TFR_REQUIRE(!(p.use_bn || p.input_bn) || p.bn_state, "cfg->bn_state must be set with BN");
  if (M == 0) return TFR_OK;
  if (precision == TFR_PREC_FP32)
    return mlp_simt_fwd(X, M, p, params, mask, ws_base(workspace), score_planes,
                        (cudaStream_t)stream, true);
  return mlp_tc_fwd(X, M, p, params, mask, ws_base(workspace), score_planes,
                    precision == TFR_PREC_TF32X3 ? 3 : 1, (cudaStream_t)stream, true);
}

extern "C" int tfr_mlp_bwd_tasks(const void* Xv, int M, const tfr_mlp_cfg* cfg,
                                 const float* params, const float* dscore_planes,
                                 const float* task_weights_host, const uint8_t* mask,
                                 void* workspace, float* grads, int precision, void* stream) {
  int rc = check_tasks_args(cfg, precision);
  if (rc) return rc;
  const float* X = static_cast<const float*>(Xv);
  TFR_REQUIRE(X && params && workspace && dscore_planes && grads, "NULL argument");
  const int O = cfg->dims[cfg->n_dense];
  TaskWeights tw{};
  bool unit = true;
  for (int o = 0; o < O; ++o) {
    tw.w[o] = task_weights_host ? task_weights_host[o] : 1.f;
    TFR_REQUIRE(std::isfinite(tw.w[o]), "task weight %d is not finite", o);
    unit = unit && tw.w[o] == 1.f;
  }
  MlpPlan p;
  rc = make_mlp_plan(cfg, M, &p);
  if (rc) return rc;
  TFR_REQUIRE(!(p.use_bn || p.input_bn) || p.bn_state, "cfg->bn_state must be set with BN");
  if (M == 0) {
    TFR_CUDA_OK(cudaMemsetAsync(grads, 0, p.n_params * sizeof(float), (cudaStream_t)stream));
    return TFR_OK;
  }
  // One task of weight 1: the planar signal is the interleaved one, and tfr_mlp_bwd already
  // zeroes masked rows of a single output.
  const TaskWeights* twp = O == 1 && unit ? nullptr : &tw;
  if (precision == TFR_PREC_FP32)
    return mlp_simt_bwd(X, M, p, params, dscore_planes, mask, ws_base(workspace), grads,
                        (cudaStream_t)stream, twp);
  return mlp_tc_bwd(X, M, p, params, dscore_planes, mask, ws_base(workspace), grads,
                    precision == TFR_PREC_TF32X3 ? 3 : 1, (cudaStream_t)stream, twp);
}

extern "C" int tfr_mlp_input_grad(const tfr_mlp_cfg* cfg, int M, const float* params,
                                  void* workspace, int col0, int ncols, float* dX, int ldx,
                                  int precision, void* stream) {
  MlpPlan p;
  int rc = make_mlp_plan(cfg, M, &p);
  if (rc) return rc;
  TFR_REQUIRE(params && workspace && dX, "NULL argument");
  TFR_REQUIRE(precision == TFR_PREC_TF32X3 || precision == TFR_PREC_TF32,
              "tower input gradients need precision tf32x3 or tf32 (got %d)", precision);
  TFR_REQUIRE(!p.input_bn, "tower input gradients are not offered with input BatchNormalization");
  TFR_REQUIRE(p.n_dense >= 2, "tower input gradients need at least one hidden layer");
  TFR_REQUIRE(col0 >= 0 && ncols >= 1 && col0 + ncols <= p.dims[0],
              "columns [%d, %d) outside the tower input [0, %d)", col0, col0 + ncols, p.dims[0]);
  TFR_REQUIRE(ldx >= ncols, "ldx %d must be >= ncols %d", ldx, ncols);
  if (M == 0) return TFR_OK;
  return mlp_tc_input_grad(M, p, params, ws_base(workspace), col0, ncols, dX, ldx,
                           precision == TFR_PREC_TF32X3 ? 3 : 1, (cudaStream_t)stream);
}

extern "C" int tfr_optimizer_step(float* params, const float* grads, float* accum, size_t n,
                                  int kind, float lr, float eps, float grad_scale,
                                  void* stream) {
  TFR_REQUIRE(params && grads, "NULL argument");
  TFR_REQUIRE(kind == 0 || kind == 1, "optimizer kind %d unsupported", kind);
  TFR_REQUIRE(kind == 0 || accum != nullptr, "Adagrad needs an accumulator");
  if (n == 0) return TFR_OK;
  optimizer_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      params, grads, accum, n, kind, lr, eps, grad_scale);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

extern "C" int tfr_adamw_step(float* params, const float* grads, float* m, float* v,
                              const uint8_t* decay_mask, size_t n, float lr, float beta1,
                              float beta2, float eps, float weight_decay, int64_t step,
                              float grad_scale, void* stream) {
  TFR_REQUIRE(params && grads && m && v, "NULL argument");
  TFR_REQUIRE(step >= 1, "AdamW step %lld must be >= 1", (long long)step);
  TFR_REQUIRE(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f,
              "beta1 %g and beta2 %g must be in [0, 1)", (double)beta1, (double)beta2);
  if (n == 0) return TFR_OK;
  const double t = (double)step;
  const float step_size =
      (float)((double)lr * std::sqrt(1.0 - std::pow((double)beta2, t)) /
              (1.0 - std::pow((double)beta1, t)));
  adamw_kernel<false><<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      params, grads, m, v, decay_mask, n, lr, beta1, beta2, eps, weight_decay, step_size,
      grad_scale, 0.f, nullptr);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

extern "C" size_t tfr_global_norm_workspace_bytes(size_t n) {
  return (size_t)norm_blocks(n) * sizeof(double);
}

extern "C" int tfr_global_norm(const float* x, size_t n, float* norm_out, void* workspace,
                               size_t workspace_bytes, void* stream) {
  TFR_REQUIRE(norm_out && workspace && (x || n == 0), "NULL argument");
  const unsigned blocks = norm_blocks(n);
  TFR_REQUIRE(workspace_bytes >= (size_t)blocks * sizeof(double),
              "global norm of %zu floats needs a %zu-byte workspace, got %zu", n,
              (size_t)blocks * sizeof(double), workspace_bytes);
  const cudaStream_t st = (cudaStream_t)stream;
  double* partials = (double*)workspace;
  if (n == 0) {
    TFR_CUDA_OK(cudaMemsetAsync(norm_out, 0, sizeof(float), st));
    return TFR_OK;
  }
  sumsq_partials_kernel<<<blocks, kNormThreads, 0, st>>>(x, n, partials);
  TFR_LAUNCH_OK();
  norm_final_kernel<<<1, 1024, 0, st>>>(partials, (int)blocks, norm_out);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

extern "C" int tfr_adamw_step_clipped(float* params, const float* grads, float* m, float* v,
                                      const uint8_t* decay_mask, size_t n, float lr,
                                      float beta1, float beta2, float eps, float weight_decay,
                                      int64_t step, float grad_scale, float clip_norm,
                                      const float* norm, void* stream) {
  TFR_REQUIRE(params && grads && m && v && norm, "NULL argument");
  TFR_REQUIRE(step >= 1, "AdamW step %lld must be >= 1", (long long)step);
  TFR_REQUIRE(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f,
              "beta1 %g and beta2 %g must be in [0, 1)", (double)beta1, (double)beta2);
  TFR_REQUIRE(clip_norm > 0.f && std::isfinite(clip_norm),
              "clip_norm %g must be finite and > 0", (double)clip_norm);
  if (n == 0) return TFR_OK;
  const double t = (double)step;
  const float step_size =
      (float)((double)lr * std::sqrt(1.0 - std::pow((double)beta2, t)) /
              (1.0 - std::pow((double)beta1, t)));
  adamw_kernel<true><<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      params, grads, m, v, decay_mask, n, lr, beta1, beta2, eps, weight_decay, step_size,
      grad_scale, clip_norm, norm);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

extern "C" int tfr_loss_scale_mul(const float* x, size_t n, const float* scale, float* out,
                                  void* stream) {
  TFR_REQUIRE(scale && out && (x || n == 0), "NULL argument");
  if (n == 0) return TFR_OK;
  loss_scale_mul_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      x, n, scale, out);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

extern "C" int tfr_adamw_step_scaled(float* params, const float* grads, float* m, float* v,
                                     const uint8_t* decay_mask, size_t n, float lr, float beta1,
                                     float beta2, float eps, float weight_decay, int64_t step,
                                     float clip_norm, const float* norm, const float* scale,
                                     void* stream) {
  TFR_REQUIRE(params && grads && m && v && norm && scale, "NULL argument");
  TFR_REQUIRE(step >= 1, "AdamW step %lld must be >= 1", (long long)step);
  TFR_REQUIRE(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f,
              "beta1 %g and beta2 %g must be in [0, 1)", (double)beta1, (double)beta2);
  TFR_REQUIRE(clip_norm == 0.f || (clip_norm > 0.f && std::isfinite(clip_norm)),
              "clip_norm %g must be 0 (off) or finite and > 0", (double)clip_norm);
  if (n == 0) return TFR_OK;
  const double t = (double)step;
  const float step_size =
      (float)((double)lr * std::sqrt(1.0 - std::pow((double)beta2, t)) /
              (1.0 - std::pow((double)beta1, t)));
  adamw_scaled_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      params, grads, m, v, decay_mask, n, lr, beta1, beta2, eps, weight_decay, step_size,
      clip_norm, norm, scale);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

extern "C" int tfr_loss_scale_update(float* scale, int64_t* good_steps, const float* norm,
                                     float* unscaled_norm, int64_t growth_steps, void* stream) {
  TFR_REQUIRE(scale && norm && (good_steps || growth_steps == 0), "NULL argument");
  TFR_REQUIRE(growth_steps >= 0, "growth_steps %lld must be >= 0", (long long)growth_steps);
  loss_scale_update_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(scale, good_steps, norm,
                                                               unscaled_norm, growth_steps);
  TFR_LAUNCH_OK();
  return TFR_OK;
}
