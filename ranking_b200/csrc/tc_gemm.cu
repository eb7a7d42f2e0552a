// TF32 / 3xTF32 GEMM engine for the scorer tower on the Hopper warpgroup MMA (wgmma_gemm.cuh).
#include <cuda_runtime.h>

#include "common.cuh"
#include "tc_gemm.cuh"
#include "wgmma_gemm.cuh"

namespace tfr {
namespace tc {

template <bool A_MN, bool B_MN>
static int dispatch(const GemmDesc& g, const wg::Args& a, cudaStream_t st, int* ctas) {
  if (g.passes == 1) return wg::launch<float, A_MN, B_MN, 1, false, false>(a, st, ctas);
  if (g.split_b) return wg::launch<float, A_MN, B_MN, 3, false, false>(a, st, ctas);
  return wg::launch<float, A_MN, B_MN, 3, true, false>(a, st, ctas);
}

int gemm(const GemmDesc& g, cudaStream_t st) {
  TFR_REQUIRE(g.A && g.B && g.C, "tc gemm: NULL operand");
  TFR_REQUIRE(g.GM >= 1 && g.GN >= 1 && g.GK >= 1, "tc gemm: empty problem");
  TFR_REQUIRE(g.passes == 1 || g.passes == 3, "tc gemm: passes must be 1 or 3");
  TFR_REQUIRE(g.lda % 4 == 0 && g.ldb % 4 == 0, "tc gemm: leading dimensions must be multiples of 4");
  TFR_REQUIRE((reinterpret_cast<uintptr_t>(g.A) & 15) == 0 && (reinterpret_cast<uintptr_t>(g.B) & 15) == 0,
              "tc gemm: operands must be 16-byte aligned");
  const bool pre_split_b = g.passes == 3 && !g.split_b;
  TFR_REQUIRE(!pre_split_b || g.B_lo != nullptr, "tc gemm: B_lo required for pre-split B");
  TFR_REQUIRE(!pre_split_b || (reinterpret_cast<uintptr_t>(g.B_lo) & 15) == 0, "tc gemm: B_lo alignment");
  const int splits = g.splits < 1 ? 1 : g.splits;
  TFR_REQUIRE(!g.colsum || (!g.store_transposed && splits == 1),
              "tc gemm: colsum output needs a row-major, unsplit store");
  TFR_REQUIRE(!g.colsum || g.GN <= 1024, "tc gemm: colsum output supports GN <= 1024");
  TFR_REQUIRE(g.epi != EPI_BIAS_ACT || g.bias, "tc gemm: bias required");
  TFR_REQUIRE(g.epi != EPI_MASK_POS || g.aux, "tc gemm: aux required");
  TFR_REQUIRE(g.epi != EPI_MASK_BITS || g.mask_bits_in, "tc gemm: mask_bits_in required");
  TFR_REQUIRE(!(g.mask_bits_out || g.epi == EPI_MASK_BITS) || (!g.store_transposed && splits == 1),
              "tc gemm: ReLU sign bits need a row-major, unsplit store");
  // the folded remainder columns of this layout take plain stores only
  TFR_REQUIRE(!(g.a_mn && g.b_mn) || (g.epi == EPI_STORE && !g.colsum),
              "tc gemm: MN-major A and B (the dW layout) take the plain store epilogue");

  wg::Args a{};
  a.A = g.A; a.lda = g.lda; a.B = g.B; a.ldb = g.ldb; a.B_lo = g.B_lo;
  a.C = g.C; a.ldc = g.ldc;
  a.GM = g.GM; a.GN = g.GN; a.GK = g.GK;
  a.epi = g.epi; a.act = g.act; a.bias = g.bias; a.aux = g.aux;
  a.bits_out = g.epi == EPI_BIAS_ACT ? g.mask_bits_out : nullptr;
  a.bits_in = g.mask_bits_in;
  a.store_transposed = g.store_transposed;
  a.splits = splits; a.split_stride = g.split_stride;
  a.colsum = g.colsum; a.colsum_stride = g.colsum_stride;
  a.colsum_cols = g.colsum ? (g.GN + 3) / 4 * 4 : 0;
  int ctas = 0, rc;
  if (!g.a_mn) rc = g.b_mn ? dispatch<false, true>(g, a, st, &ctas) : dispatch<false, false>(g, a, st, &ctas);
  else rc = g.b_mn ? dispatch<true, true>(g, a, st, &ctas) : dispatch<true, false>(g, a, st, &ctas);
  if (rc == TFR_OK && g.colsum_slots_out) *g.colsum_slots_out = wg::kWarps * ctas;
  return rc;
}

int tile_units(int gm, int gn) {
  return ((gm + wg::BM - 1) / wg::BM) * ((gn - wg::folded_cols(gn) + 63) / 64);
}

}  // namespace tc
}  // namespace tfr

// Test / parity entry: raw GEMM through the tensor-core engine.
extern "C" int tfr_tc_gemm(const float* A, int lda, const float* B, int ldb, const float* B_lo,
                           float* C, int ldc, int GM, int GN, int GK, int a_mn, int b_mn,
                           int passes, int split_b, int epi, const float* bias, const float* aux,
                           int act, int store_transposed, int splits, size_t split_stride,
                           uint32_t* mask_bits_out, const uint32_t* mask_bits_in,
                           void* stream) {
  tfr::tc::GemmDesc g{};
  g.mask_bits_out = mask_bits_out; g.mask_bits_in = mask_bits_in;
  g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.B_lo = B_lo; g.C = C; g.ldc = ldc;
  g.GM = GM; g.GN = GN; g.GK = GK; g.a_mn = a_mn; g.b_mn = b_mn; g.passes = passes;
  g.split_b = split_b; g.epi = epi; g.bias = bias; g.aux = aux; g.act = act;
  g.store_transposed = store_transposed; g.splits = splits; g.split_stride = split_stride;
  return tfr::tc::gemm(g, (cudaStream_t)stream);
}
