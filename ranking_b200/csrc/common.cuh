// Shared helpers for the tfr_b200 kernels (sm_90a).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdarg>
#include <cstdio>

#include "tfr_b200.h"

namespace tfr {

// ---- error plumbing (host) -------------------------------------------------
void set_error(const char* fmt, ...);
void count_launch();   // bumps the host-side launch counter (tfr_launch_count)
int num_sms();         // SM count of the current device; 132 (H100 SXM) when none can be queried
// Opt-in dynamic shared memory per block of the current device (232,448 bytes on H100), queried
// once per device ordinal; 48 KB when no device can be queried.
size_t smem_optin_limit();

#define TFR_REQUIRE(cond, ...)              \
  do {                                      \
    if (!(cond)) {                          \
      ::tfr::set_error(__VA_ARGS__);        \
      return TFR_INVALID_ARGUMENT;          \
    }                                       \
  } while (0)

// A failed API call also leaves its error as the runtime's last error; it is cleared here so
// that the next launch's TFR_LAUNCH_OK does not report it again.
#define TFR_CUDA_OK(expr)                                                  \
  do {                                                                     \
    cudaError_t _e = (expr);                                               \
    if (_e != cudaSuccess) {                                               \
      (void)cudaGetLastError();                                            \
      ::tfr::set_error("%s failed: %s (%s:%d)", #expr,                     \
                       cudaGetErrorString(_e), __FILE__, __LINE__);        \
      return TFR_CUDA_ERROR;                                               \
    }                                                                      \
  } while (0)

#define TFR_LAUNCH_OK()                                                    \
  do {                                                                     \
    cudaError_t _e = cudaGetLastError();                                   \
    if (_e != cudaSuccess) {                                               \
      ::tfr::set_error("kernel launch failed: %s (%s:%d)",                 \
                       cudaGetErrorString(_e), __FILE__, __LINE__);        \
      return TFR_CUDA_ERROR;                                               \
    }                                                                      \
    ::tfr::count_launch();                                                 \
  } while (0)

// ---- device helpers ---------------------------------------------------------
constexpr float kLogEpsilon = -23.025850929940457f;  // ln(1e-10), losses_impl.py:30

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_int(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Deterministic block reductions through a small smem scratch (>= 32 floats).
// All threads of the block must call; the result is broadcast to every thread.
template <typename Op>
__device__ __forceinline__ float block_reduce(float v, float* scratch, Op op,
                                              float identity) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nwarps = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();  // scratch may still be read from a previous reduction
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  float r = identity;
  if (warp == 0) {
    r = lane < nwarps ? scratch[lane] : identity;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r = op(r, __shfl_xor_sync(0xffffffffu, r, o));
    if (lane == 0) scratch[0] = r;
  }
  __syncthreads();
  r = scratch[0];
  return r;
}
struct OpSum { __device__ float operator()(float a, float b) const { return a + b; } };
struct OpMax { __device__ float operator()(float a, float b) const { return fmaxf(a, b); } };
struct OpMin { __device__ float operator()(float a, float b) const { return fminf(a, b); } };

__device__ __forceinline__ float block_sum(float v, float* s) { return block_reduce(v, s, OpSum(), 0.f); }
__device__ __forceinline__ float block_max(float v, float* s) { return block_reduce(v, s, OpMax(), -INFINITY); }
__device__ __forceinline__ float block_min(float v, float* s) { return block_reduce(v, s, OpMin(), INFINITY); }

// gain / discount enums (keras/utils.py:50-107)
__device__ __forceinline__ float gain_of(int gain_fn, float label) {
  return gain_fn == TFR_GAIN_POW2_MINUS_1 ? exp2f(label) - 1.f : label;
}
__device__ __forceinline__ float disc_of(int disc_fn, float rank) {
  switch (disc_fn) {
    case TFR_DISC_LOG2_INVERSE: {
      float d = log1pf(rank);
      return d == 0.f ? 0.f : 0.6931471805599453f / d;
    }
    case TFR_DISC_LOG1P_INVERSE:
      return 1.f / log1pf(rank);
    default:
      return rank == 0.f ? 0.f : 1.f / rank;
  }
}

}  // namespace tfr
