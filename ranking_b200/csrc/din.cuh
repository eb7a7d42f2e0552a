// K11 DocumentInteractionAttention: what the FP32 SIMT attention core (din.cu) and the TF32
// wgmma one (din_tc.cu) share, so that both draw the same dropout keep mask.
#pragma once
#include <cstdint>

#include <cuda_bf16.h>
#include <cuda_fp16.h>
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

// FP32 SIMT attention core (din.cu): qkv [B N, 3 H h] (q, k, v blocks of H heads of h
// columns each); lmask uint8 [B N] (0 = key masked with kMaskAdder; NULL = all valid);
// O [B N, H h]; lse [B N, H, 2] = {row max, 1 / sum}; dsum [B N, H]; dqkv [B N, 3 H h].
// Dropout of P with rate `drop` draws din_uniform(dseed, ((b H + head) N + i) N + j).
// h % 4 == 0, h <= 128.
int din_attn_fwd(const float* qkv, const uint8_t* lmask, int B, int N, int H, int h, float drop,
                 unsigned long long dseed, float* O, float* lse, cudaStream_t st);
int din_attn_bwd(const float* qkv, const uint8_t* lmask, int B, int N, int H, int h, float drop,
                 unsigned long long dseed, const float* O, const float* lse, const float* dO,
                 float* dsum, float* dqkv, cudaStream_t st);

// TF32 tensor-core attention core (din_tc.cu), same operands, outputs and dropout draws as the
// SIMT kernels.
int din_tc_attn_fwd(const float* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                    float drop, unsigned long long dseed, float* O, float* lse, cudaStream_t st);
int din_tc_attn_bwd(const float* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                    float drop, unsigned long long dseed, const float* O, const float* lse,
                    const float* dO, float* dsum, float* dqkv, cudaStream_t st);

// 16-bit tensor-core attention core (din_bf16.cu), one overload per element type (bf16, fp16):
// qkv, O, dO and dqkv 16-bit, lse and dsum fp32, same layouts and dropout draws.  P~ is rounded
// to 16 bits after normalisation, before P~ v; dS is rounded before dS K and dS^T Q, and dQ / dK
// are scaled by 1 / sqrt(h) after those products.  dsum = dO . O over the stored 16-bit values.
// h % 8 == 0, h <= 128.
int din16_attn_fwd(const __nv_bfloat16* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                   float drop, unsigned long long dseed, __nv_bfloat16* O, float* lse,
                   cudaStream_t st);
int din16_attn_fwd(const __half* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                   float drop, unsigned long long dseed, __half* O, float* lse, cudaStream_t st);
int din16_attn_bwd(const __nv_bfloat16* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                   float drop, unsigned long long dseed, const __nv_bfloat16* O,
                   const float* lse, const __nv_bfloat16* dO, float* dsum,
                   __nv_bfloat16* dqkv, cudaStream_t st);
int din16_attn_bwd(const __half* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                   float drop, unsigned long long dseed, const __half* O, const float* lse,
                   const __half* dO, float* dsum, __half* dqkv, cudaStream_t st);

// C [GM, GN] (ldc) = A B (+ bias, act) on the scorer GEMM engine, 3xTF32 (passes 3) or TF32
// (passes 1).  a_mn / b_mn: operand stored MN-major (A^T [GK, GM], B [GK, GN]) instead of
// K-major (A [GM, GK], B [GN, GK]).
int din_gemm(const float* A, int lda, int a_mn, const float* B, int ldb, int b_mn, float* C,
             int ldc, int GM, int GN, int GK, const float* bias, int act, int passes,
             cudaStream_t st);
// grads_w[0 .. Kin Nout + Nout) = {A^T dZ, column sums of dZ}: A [M, Kin] (lda), dZ [M, Nout]
// (ldz), split over M into `splits` row ranges of whole 32-row blocks (partials of pitch
// pstride), reduced in fixed order; colsum holds mlp_colsum's per-split column sums of dZ
// (pitch cs_stride).  Always in the direct orientation.
int din_weight_grad(const float* A, int lda, int Kin, const float* dZ, int ldz, int Nout, int M,
                    int splits, float* partial, size_t pstride, const float* colsum,
                    size_t cs_stride, float* grads_w, int passes, cudaStream_t st);

}  // namespace tfr
