// K11 DocumentInteractionAttention: what the FP32 SIMT attention core (din.cu) and the TF32
// wgmma one (din_tc.cu) share, so that both draw the same dropout keep mask.
#pragma once
#include <cstdint>

#include <cuda_runtime.h>

namespace tfr {

constexpr float kMaskAdder = -1e9f;   // Keras Softmax's adder for masked logits

// Counter-based uniform in [0, 1): splitmix64 of (site seed, element), as the tower's dropout.
__device__ __forceinline__ float din_uniform(unsigned long long s, unsigned long long e) {
  unsigned long long z = s + 0x9E3779B97F4A7C15ull * (e + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (float)(z >> 40) * (1.0f / 16777216.0f);
}

// TF32 tensor-core attention core (din_tc.cu), same operands, outputs and dropout draws as the
// SIMT kernels: qkv [B N, 3 H h]; O [B N, H h]; lse [B N, H, 2] = {row max, 1 / sum};
// dsum [B N, H]; dqkv [B N, 3 H h].
int din_tc_attn_fwd(const float* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                    float drop, unsigned long long dseed, float* O, float* lse, cudaStream_t st);
int din_tc_attn_bwd(const float* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                    float drop, unsigned long long dseed, const float* O, const float* lse,
                    const float* dO, float* dsum, float* dqkv, cudaStream_t st);

}  // namespace tfr
