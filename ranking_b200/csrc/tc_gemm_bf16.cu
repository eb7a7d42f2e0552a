// bf16 GEMM engine for the scorer tower (TFR_PREC_BF16) on the Hopper warpgroup MMA
// (wgmma_gemm.cuh): bf16 operands, fp32 accumulation.
#include <cuda_bf16.h>

#include "common.cuh"
#include "tc_gemm_bf16.cuh"
#include "wgmma_gemm.cuh"

namespace tfr {
namespace tcb {

int gemm(const GemmDesc& g, cudaStream_t st) {
  TFR_REQUIRE(g.A && g.B && g.C, "bf16 gemm: NULL operand");
  TFR_REQUIRE(g.GM >= 1 && g.GN >= 1 && g.GK >= 1, "bf16 gemm: empty problem");
  TFR_REQUIRE(g.lda % 8 == 0 && g.ldb % 8 == 0,
              "bf16 gemm: leading dimensions must be multiples of 8 elements");
  TFR_REQUIRE((reinterpret_cast<uintptr_t>(g.A) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(g.B) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(g.C) & 15) == 0,
              "bf16 gemm: operands must be 16-byte aligned");
  const bool mn = g.mn != 0;
  TFR_REQUIRE(mn ? g.ldc % 4 == 0 : g.ldc % 8 == 0, "bf16 gemm: ldc alignment");
  TFR_REQUIRE(g.epi == EPI_STORE || g.epi == EPI_BIAS_ACT || g.epi == EPI_MASK_BITS,
              "bf16 gemm: bad epilogue %d", g.epi);
  TFR_REQUIRE(!mn || g.epi == EPI_STORE, "bf16 gemm: dW layout only stores");
  TFR_REQUIRE(g.epi != EPI_BIAS_ACT || g.bias, "bf16 gemm: bias required");
  TFR_REQUIRE(g.epi != EPI_MASK_BITS || g.mask_bits_in, "bf16 gemm: mask_bits_in required");
  TFR_REQUIRE(!g.colsum || (!mn && g.GN <= 1024), "bf16 gemm: colsum needs mn = 0, GN <= 1024");
  TFR_REQUIRE(!g.mask_bits_out || (g.epi == EPI_BIAS_ACT && g.act == TFR_ACT_RELU),
              "bf16 gemm: sign bits are written by the bias + ReLU epilogue only");
  const int splits = mn ? (g.splits < 1 ? 1 : g.splits) : 1;
  const size_t rows_per_split = (size_t)(g.GM + 127) / 128 * 128;
  TFR_REQUIRE(!mn || splits <= 1 || g.split_stride == rows_per_split * g.ldc,
              "bf16 gemm: split_stride must equal roundup(GM, 128) * ldc");

  wg::Args a{};
  a.A = g.A; a.lda = g.lda; a.B = g.B; a.ldb = g.ldb;
  a.C = g.C; a.ldc = g.ldc;
  a.GM = g.GM; a.GN = g.GN; a.GK = g.GK;
  a.epi = g.epi; a.act = g.act; a.bias = g.bias;
  a.bits_out = g.mask_bits_out; a.bits_in = g.mask_bits_in;
  a.splits = splits; a.split_stride = mn ? g.split_stride : 0;
  a.colsum = g.colsum; a.colsum_stride = g.colsum_stride;
  a.colsum_cols = g.colsum ? (g.GN + 3) / 4 * 4 : 0;
  int ctas = 0;
  // mn = 0: A [GM, GK], B [GN, GK] (K-major), bf16 out; mn = 1: A [GK, GM], B [GK, GN], fp32 out
  const int rc = mn ? wg::launch<__nv_bfloat16, true, true, 1, false, false>(a, st, &ctas)
                    : wg::launch<__nv_bfloat16, false, false, 1, false, true>(a, st, &ctas);
  if (rc == TFR_OK && g.colsum_slots_out) *g.colsum_slots_out = wg::kWarps * ctas;
  return rc;
}

}  // namespace tcb
}  // namespace tfr

// Test / parity entry: raw GEMM through the bf16 tensor-core engine (see tc_gemm_bf16.cuh).
extern "C" int tfr_tc_gemm_bf16(const void* A, int lda, const void* B, int ldb, void* C, int ldc,
                                int GM, int GN, int GK, int mn, int epi, const float* bias,
                                int act, uint32_t* mask_bits_out, const uint32_t* mask_bits_in,
                                float* colsum, int colsum_stride, int* colsum_slots_out,
                                int splits, size_t split_stride, void* stream) {
  tfr::tcb::GemmDesc g{};
  g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.C = C; g.ldc = ldc;
  g.GM = GM; g.GN = GN; g.GK = GK; g.mn = mn; g.epi = epi; g.bias = bias; g.act = act;
  g.mask_bits_out = mask_bits_out; g.mask_bits_in = mask_bits_in;
  g.colsum = colsum; g.colsum_stride = colsum_stride; g.colsum_slots_out = colsum_slots_out;
  g.splits = splits; g.split_stride = split_stride;
  return tfr::tcb::gemm(g, (cudaStream_t)stream);
}
