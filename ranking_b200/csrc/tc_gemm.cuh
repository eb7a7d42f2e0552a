// Hopper wgmma TF32 / 3xTF32 GEMM engine for the scorer tower — declarations.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace tfr {
namespace tc {

enum Epi { EPI_STORE = 0, EPI_BIAS_ACT = 1, EPI_MASK_POS = 2, EPI_MASK_BITS = 3 };

// D[GM, GN] = A[GM, GK] * B[GK, GN]  (fp32 in / fp32 out, TF32 tensor cores)
//
// Operand storage (all row-major fp32 in global memory):
//   a_mn == 0 : A stored [GM, GK]  (K contiguous  -> K-major)
//   a_mn == 1 : A stored [GK, GM]  (GM contiguous -> MN-major)
//   b_mn == 0 : B stored [GN, GK]  (K contiguous  -> K-major)
//   b_mn == 1 : B stored [GK, GN]  (GN contiguous -> MN-major)
// passes == 1 : one TF32 product (operands truncated to TF32)
// passes == 3 : error-compensated 3xTF32: x = hi + lo, D = Ahi*Bhi + Alo*Bhi + Ahi*Blo.
//               A is always split on the fly, in registers.  B is split on the
//               fly too when split_b != 0, otherwise `B` must hold the hi parts
//               and `B_lo` the lo parts (weights, pre-split once per step).
struct GemmDesc {
  const float* A; int lda;       // leading dimension in floats (row stride)
  const float* B; int ldb;
  const float* B_lo;             // may be null (see above)
  float* C; int ldc;
  int GM, GN, GK;
  int a_mn, b_mn, passes, split_b;
  int epi;                       // Epi
  const float* bias;             // EPI_BIAS_ACT: [GN]
  const float* aux;              // EPI_MASK_POS: [GM, GN] ld = ldc; C = aux > 0 ? C : 0
  int act;                       // tfr_activation
  int store_transposed;          // write element (r, c) to C[c * ldc + r]
  int splits;                    // split the GK loop over blockIdx.z; split z writes to
  size_t split_stride;           //   C + z * split_stride (floats); k range rounded to 32
  float* colsum;                 // optional: column sums of everything each CTA stored, slot
  int colsum_stride;             //   (cta * 8 + warp), row pitch in floats;
  int* colsum_slots_out;         //   receives the number of slots written (8 * CTAs)
  // ReLU sign bits, word [(col / 32) * GM + row] (bit j = column 32 * (col / 32) + j):
  uint32_t* mask_bits_out;       //   EPI_BIAS_ACT: written next to C (stored value > 0)
  const uint32_t* mask_bits_in;  //   EPI_MASK_BITS: C = bit ? C : 0  (replaces `aux`)
};

// Returns a tfr_status.  Requirements (checked): lda/ldb multiples of 4 floats,
// 16-byte aligned base pointers, any GN (128-column output tiles).
int gemm(const GemmDesc& g, cudaStream_t stream);

// Work units of a GM x GN output: 128-row tiles of one m64n128 (two units) or, when the
// tile's live columns fit in 64, one m64n64 (one unit) per warpgroup and k step, each
// walking the whole k range.  Picks the cheaper orientation of a dW GEMM.
inline int tile_units(int gm, int gn) { return ((gm + 127) / 128) * ((gn + 63) / 64); }

// True if a layer shape can run on this engine (alignment constraints).
bool shape_supported(int rows_ld_a, int rows_ld_b);

}  // namespace tc
}  // namespace tfr
