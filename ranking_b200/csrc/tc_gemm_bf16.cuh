// Hopper wgmma 16-bit GEMM engine (bf16: the scorer tower's and TFR-BERT's TFR_PREC_BF16; fp16:
// TFR-BERT's TFR_PREC_FP16) — declarations.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace tfr {
namespace tcb {

enum Epi { EPI_STORE = 0, EPI_BIAS_ACT = 1, EPI_MASK_BITS = 3 };

// D[GM, GN] = A[GM, GK] * B[GK, GN], bf16 (f16 = 0) or fp16 (f16 = 1) operands, fp32
// accumulation; a 16-bit C has the operands' type.
//
//   mn == 0 (forward / dZ GEMMs): A stored [GM, GK], B stored [GN, GK] (K contiguous);
//           C is 16-bit [GM, GN] row-major; epilogues:
//             EPI_BIAS_ACT  C = act(D + bias), optionally the ReLU sign bits of the stored
//                           values to mask_bits_out, word [(col / 32) * GM + row]
//             EPI_MASK_BITS C = bit ? D : 0 with bits from mask_bits_in; optionally the
//                           column sums of C (fp32, before rounding) per CTA and
//                           warp to `colsum` (bias gradients)
//             EPI_STORE     C = D
//   mn == 1 (dW GEMMs): A stored [GK, GM], B stored [GK, GN] (M / N contiguous), i.e.
//           D = A^T B over a long GK; the GK range is split over `splits` work items and
//           split z writes its fp32 partial to C + z * split_stride (floats), rows padded
//           to a multiple of 128: split_stride >= roundup(GM, 128) * ldc.
// Requirements (checked): lda, ldb, ldc multiples of 8 elements (mn == 0 C: 16-bit) or 4
// floats (mn == 1 C), 16-byte aligned bases.
struct GemmDesc {
  const void* A; int lda;
  const void* B; int ldb;
  void* C; int ldc;
  int GM, GN, GK;
  int mn;
  int epi;
  const float* bias;
  int act;
  uint32_t* mask_bits_out;
  const uint32_t* mask_bits_in;
  float* colsum; int colsum_stride; int* colsum_slots_out;
  int splits; size_t split_stride;
  int f16;
};

int gemm(const GemmDesc& g, cudaStream_t stream);

}  // namespace tcb
}  // namespace tfr
