// K7: the one collective of the data-parallel step (all-reduce(SUM) of the flat scorer
// gradient, tf.distribute in the reference: keras/strategy_utils.py:45-116,
// extension/task.py:256-262) fused with the optimizer update, over NVLink peer memory.
//
// Every rank owns a gradient buffer in device memory that its peers map through CUDA IPC
// (one process per GPU, one node: every GPU reaches every peer at full NVLink bandwidth
// through NVSwitch).  The step's last kernel on every rank
//   1. tells its peers "my gradient of step e is complete" (one 4-byte system-scope
//      release store per peer into the peer's flag pad) and waits until its own pad shows
//      step e for every rank;
//   2. reads all `world` gradient buffers — its own from HBM, the others as peer loads over
//      NVLink — sums them in rank order 0..world-1 (so every replica computes bit-identical
//      sums and the replicas never drift), scales by 1/world and applies SGD / Adagrad to
//      its parameter replica.
// The gradient is 76 K floats (0.3 MB) at the benchmark configuration: (world - 1) * 0.3 MB
// of peer reads per rank, a few microseconds — the step is latency-bound, which is why the
// collective is one kernel with one flag round instead of a library call followed by an
// optimizer launch.  Gradient buffers alternate between two slots from step to step, so the
// flag round of step e + 1 also proves that every peer has finished READING slot e % 2
// before anyone overwrites it in step e + 2: one barrier per step.
#include <cstring>

#include "common.cuh"

namespace tfr {

namespace {

constexpr int kMaxRanks = 16;

struct PeerTable {
  const float* grad[kMaxRanks];   // this step's gradient slot of every rank
  uint32_t* flags[kMaxRanks];     // flag pad of every rank: [kMaxRanks] words
};

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__global__ void __launch_bounds__(256)
allreduce_optimizer_kernel(PeerTable t, int rank, int world, uint32_t epoch,
                           float* __restrict__ params, float* __restrict__ accum,
                           float* __restrict__ summed, size_t n4, size_t n, int kind, float lr,
                           float eps, float grad_scale) {
  // -- flag round ----------------------------------------------------------------------
  if (blockIdx.x == 0 && threadIdx.x < world) {
    __threadfence_system();   // (the gradient was written by earlier kernels of this stream)
    st_release_sys(t.flags[threadIdx.x] + rank, epoch);
  }
  if (threadIdx.x < world) {
    const uint32_t* mine = t.flags[rank] + threadIdx.x;
    unsigned long long t0, now;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    // epochs only grow; "not yet" is a smaller value (wrap-safe signed distance).  A peer that
    // never arrives (a crashed rank) must trap, not hang the GPU: 5 s of wall clock.
    while ((int32_t)(ld_acquire_sys(mine) - epoch) < 0) {
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
      if (now - t0 > 5000000000ull) {
        printf("tfr all-reduce: rank %d timed out waiting for rank %d (epoch %u)\n", rank,
               (int)threadIdx.x, epoch);
        __trap();
      }
    }
  }
  __syncthreads();
  // -- reduce + optimizer ----------------------------------------------------------------
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (size_t)gridDim.x * blockDim.x) {
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
    for (int r = 0; r < world; ++r) {
      const float4 v = reinterpret_cast<const float4*>(t.grad[r])[i];   // peer load over NVLink
      g.x += v.x; g.y += v.y; g.z += v.z; g.w += v.w;
    }
    if (summed) reinterpret_cast<float4*>(summed)[i] = g;
    g.x *= grad_scale; g.y *= grad_scale; g.z *= grad_scale; g.w *= grad_scale;
    float4 p = reinterpret_cast<float4*>(params)[i];
    if (kind == 0) {
      p.x -= lr * g.x; p.y -= lr * g.y; p.z -= lr * g.z; p.w -= lr * g.w;
    } else {
      float4 a = reinterpret_cast<float4*>(accum)[i];
      a.x += g.x * g.x; a.y += g.y * g.y; a.z += g.z * g.z; a.w += g.w * g.w;
      reinterpret_cast<float4*>(accum)[i] = a;
      p.x -= lr * g.x / (sqrtf(a.x) + eps);
      p.y -= lr * g.y / (sqrtf(a.y) + eps);
      p.z -= lr * g.z / (sqrtf(a.z) + eps);
      p.w -= lr * g.w / (sqrtf(a.w) + eps);
    }
    reinterpret_cast<float4*>(params)[i] = p;
  }
  // scalar tail (n not a multiple of 4)
  if (blockIdx.x == 0) {
    for (size_t i = 4 * n4 + threadIdx.x; i < n; i += blockDim.x) {
      float g = 0.f;
      for (int r = 0; r < world; ++r) g += t.grad[r][i];
      if (summed) summed[i] = g;
      g *= grad_scale;
      if (kind == 0) {
        params[i] -= lr * g;
      } else {
        const float a = accum[i] + g * g;
        accum[i] = a;
        params[i] -= lr * g / (sqrtf(a) + eps);
      }
    }
  }
}

}  // namespace

}  // namespace tfr

using namespace tfr;

/* Device memory that peers can map: cudaMalloc (not the caching allocator: the IPC handle
 * names the whole allocation), zero-filled.  handle_out: the 64-byte cudaIpcMemHandle_t. */
extern "C" int tfr_dp_alloc(size_t bytes, void** ptr_out, unsigned char* handle_out) {
  TFR_REQUIRE(bytes > 0 && ptr_out && handle_out, "tfr_dp_alloc: bad argument");
  void* p = nullptr;
  TFR_CUDA_OK(cudaMalloc(&p, bytes));
  TFR_CUDA_OK(cudaMemset(p, 0, bytes));
  cudaIpcMemHandle_t h;
  TFR_CUDA_OK(cudaIpcGetMemHandle(&h, p));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  std::memcpy(handle_out, &h, sizeof(h));
  *ptr_out = p;
  return TFR_OK;
}

extern "C" int tfr_dp_open(const unsigned char* handle, void** ptr_out) {
  TFR_REQUIRE(handle && ptr_out, "tfr_dp_open: bad argument");
  cudaIpcMemHandle_t h;
  std::memcpy(&h, handle, sizeof(h));
  void* p = nullptr;
  TFR_CUDA_OK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  *ptr_out = p;
  return TFR_OK;
}

extern "C" int tfr_dp_close(void* peer_ptr) {
  if (peer_ptr) TFR_CUDA_OK(cudaIpcCloseMemHandle(peer_ptr));
  return TFR_OK;
}

extern "C" int tfr_dp_free(void* ptr) {
  if (ptr) TFR_CUDA_OK(cudaFree(ptr));
  return TFR_OK;
}

/* grad_ptrs / flag_ptrs: HOST arrays of `world` device pointers (entry `rank` is local, the
 * others are peer mappings): this step's gradient slot and the flag pad of every rank.
 * Every buffer must be 16-byte aligned.  summed_out
 * (optional): the rank-ordered sum before scaling, for inspection / metrics. */
extern "C" int tfr_allreduce_optimizer_step(const void* const* grad_ptrs,
                                            void* const* flag_ptrs, int rank, int world,
                                            uint32_t epoch, float* params, float* accum,
                                            float* summed_out, size_t n, int kind, float lr,
                                            float eps, float grad_scale, void* stream) {
  TFR_REQUIRE(grad_ptrs && flag_ptrs && params, "NULL argument");
  TFR_REQUIRE(world >= 1 && world <= kMaxRanks && rank >= 0 && rank < world,
              "bad rank %d / world %d (at most %d ranks)", rank, world, kMaxRanks);
  TFR_REQUIRE(kind == 0 || kind == 1, "optimizer kind %d unsupported", kind);
  TFR_REQUIRE(kind == 0 || accum != nullptr, "Adagrad needs an accumulator");
  if (n == 0) return TFR_OK;
  PeerTable t{};
  for (int r = 0; r < world; ++r) {
    TFR_REQUIRE(grad_ptrs[r] && flag_ptrs[r], "NULL peer pointer for rank %d", r);
    TFR_REQUIRE((reinterpret_cast<uintptr_t>(grad_ptrs[r]) & 15) == 0, "peer buffer alignment");
    t.grad[r] = static_cast<const float*>(grad_ptrs[r]);
    t.flags[r] = static_cast<uint32_t*>(flag_ptrs[r]);
  }
  const size_t n4 = n / 4;
  size_t blocks = (n4 + 255) / 256;
  if (blocks < 1) blocks = 1;
  // <= 2 CTAs per SM: every CTA is resident while it spins
  if (blocks > (size_t)(2 * num_sms())) blocks = (size_t)(2 * num_sms());
  allreduce_optimizer_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      t, rank, world, epoch, params, accum, summed_out, n4, n, kind, lr, eps, grad_scale);
  TFR_LAUNCH_OK();
  return TFR_OK;
}
