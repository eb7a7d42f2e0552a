// Hopper (sm_90a) warpgroup-MMA GEMM core shared by the TF32 / 3xTF32 engine (tc_gemm.cu) and
// the 16-bit engine (tc_gemm_bf16.cu: bf16 or fp16 operands, the same code on either type).
//
//   * a CTA owns a 128 x 128 output tile: two consumer warpgroups of 64 rows, each issuing one
//     wgmma.mma_async m64n128 per k step (m64n64 when the tile's live columns fit in 64).  In
//     the TF32 dW kernels (A and B MN-major) the last column tile also owns a remainder of up
//     to 8 columns past it (folded_cols), and their wide wgmma is m64n136;
//   * A comes from registers: each warpgroup loads its fragments from a plain (unswizzled,
//     padded) fp32 / bf16 tile in shared memory, at transposed addresses when A is MN-major.
//     The 3xTF32 hi / lo split of A happens there, in registers;
//   * operands that need no arithmetic (A in both layouts, K-major B and its pre-split lo part,
//     every bf16 B) are copied global -> shared by cp.async 16-byte copies into a ring of 3-4
//     stages; the 128-byte swizzle of B is applied in the destination address.  bf16 MN-major
//     B is read by the wgmma through the descriptor's transpose bit.  TF32 wgmma reads K-major
//     B only, so MN-major TF32 B is transposed (and, for 3xTF32, split) in shared memory:
//       - in the dW GEMMs (A and B MN-major) a producer warpgroup (threads 256..383) owns the
//         whole ring: it copies A and the raw MN-major B slab of each k block by cp.async,
//         transposes the slab in place into the swizzled K-major tile(s), and hands the stage
//         over on an mbarrier; the MMA warpgroups hand it back on another.  Nothing but
//         fragment loads and wgmma issue is left on the MMA warps;
//       - with K-major A (the single-pass TF32 forward) the third warpgroup is the epilogue's,
//         and the MMA warps stage B through registers themselves;
//   * one wgmma group stays in flight across k blocks (two A fragment register sets);
//   * the copies for the next tile start before the epilogue of the current one;
//   * the epilogue: bias / activation, ReLU masks (from an fp32 array or from 1-bit sign
//     words), ReLU sign words out, column sums, row-major, transposed or split-K partial
//     stores, fp32 or bf16 output.  Where it runs follows from A's layout:
//       - K-major A (forward and dZ GEMMs: GM long, a few k blocks per tile): a third
//         warpgroup runs it.  The MMA warpgroups write a tile's raw accumulators to a staging
//         tile in shared memory and start the next tile's k loop; the epilogue warpgroup reads
//         the staging tile row-major (a lane takes 4 adjacent columns, a warp whole rows, or
//         two rows at a time on tiles of at most 64 columns) and
//         overlaps that k loop.  The staging tile takes the room of one ring stage.
//       - MN-major A (the dW GEMMs: one epilogue per 50-100 k blocks): the two MMA warpgroups
//         run it on their accumulator registers and keep the fourth stage.
// The grid is persistent (at most one CTA per SM), so the column-sum slots are bounded by
// 8 x the SM count.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include <type_traits>

#include "common.cuh"

namespace tfr {
namespace wg {

constexpr int BM = 128;          // rows of an output tile (two warpgroups of 64)
constexpr int BN = 128;          // columns of an output tile (one m64n128 instruction)
constexpr int kThreads = 256;    // the two MMA warpgroups
constexpr int kWarps = kThreads / 32;
constexpr int kEpiThreads = 128; // the epilogue warpgroup of a staged kernel (threads 256..383)
constexpr int kTileBytes = 128 * 128;   // one swizzled B tile: 128 rows x 128 bytes of k
// A tile: 128 rows x 128 bytes of k.  K-major rows are padded to 144 B, MN-major k rows
// (512 B of m) to 544 B (fp32, 32 rows) / 272 B (bf16, 64 rows): either way the fragment
// loads of a warp hit 32 different banks.
constexpr int kAPitchK = 144;
constexpr int kAPitchMN = 4 * (128 + 8);   // bytes per k row (fp32); bf16 uses half of it
constexpr int kATileBytes = 128 * kAPitchK;
constexpr int kMaxStages = 4;
constexpr int kSmemLimit = 227 * 1024;  // dynamic shared memory of one CTA on sm_90
// Staging tile: 128 x 128 fp32 accumulators, rows padded to 136 floats.  The pitch is 8 banks
// mod 32, so the float2 stores of the accumulator layout (8 rows x 4 column pairs per warp)
// are conflict-free per half-warp; the float4 row reads and the column reads are contiguous.
constexpr int kStagingPitch = BN + 8;
constexpr int kStagingBytes = BM * kStagingPitch * 4;
// Named barriers of a staged kernel (0 is __syncthreads, which it never uses).
//   kBarMma:  bar.sync over the 256 MMA threads: the k loop's barrier.
//   kBarFull: 256 MMA threads arrive after writing the staging tile, the 128 epilogue threads
//             wait: 384.  Once per tile.
//   kBarFree: 128 epilogue threads arrive after their last read of the staging tile, the 256
//             MMA threads wait before writing the next one: 384.  Once per tile but a CTA's
//             last, which nobody would wait for.
//   kBarEpi:  bar.sync over the 128 epilogue threads, between the row pass and the column sums.
// A producer kernel uses kBarMma the same way, and kBarProd (bar.sync over its 128 producer
// threads) around the in-place transpose; its stage ring runs on mbarriers (see producer_ring).
constexpr int kBarMma = 1, kBarFull = 2, kBarFree = 3, kBarEpi = 4, kBarProd = 5;
// Registers after setmaxnreg: 2 x 128 x 208 + 128 x 88 = 64,512 of the SM's 65,536.  The
// epilogue's row loop needs 88 without spills: it holds the tile's mask words and running
// column sums beside the unrolled rows.  The producer warpgroup runs on the same 88.
constexpr int kMmaRegs = 208, kEpiRegs = 88;

enum Epi { EPI_STORE = 0, EPI_BIAS_ACT = 1, EPI_MASK_POS = 2, EPI_MASK_BITS = 3 };

struct Args {
  const void* A; int lda;
  const void* B; int ldb;
  const void* B_lo;              // pre-split B (3xTF32): lo parts, same layout as B
  void* C; int ldc;
  int GM, GN, GK;
  int epi, act;
  const float* bias;             // EPI_BIAS_ACT: [GN]
  const float* aux;              // EPI_MASK_POS: keep where aux[row * ldc + col] > 0
  uint32_t* bits_out;            // EPI_BIAS_ACT: ReLU sign words [(col / 32) * GM + row]
  const uint32_t* bits_in;       // EPI_MASK_BITS: keep where the bit is set
  int store_transposed;          // element (r, c) goes to C[c * ldc + r]
  int splits; size_t split_stride;   // split z of the k range writes C + z * split_stride
  int kb_per_split;
  int m_tiles, n_tiles;
  float* colsum; int colsum_stride;  // slot (cta * 8 + warp): column sums of what it stored
  int colsum_cols;                   // shared-memory accumulator width (0: off)
};

// Column tiling of the kernels that can fold (TF32, A and B MN-major: the dW GEMMs).  A
// remainder of 1..kFoldMax columns past the last full 128-column tile rides in that tile, which
// then owns 128 + r columns.  The folding kernel gives every B tile kFoldMax more rows (zero
// where no column lives) and issues m64n136 where the plain one issues m64n128.  As a tile of
// its own the remainder would run the whole k loop of a 128-column tile.
constexpr int kFoldMax = 8;
template <typename T, bool A_MN, bool B_MN>
__host__ __device__ constexpr bool folds() {
  return sizeof(T) == 4 && A_MN && B_MN;
}
// Remainder columns folded into the last column tile (0: none).
__host__ __device__ constexpr int folded_cols(int gn) {
  return gn > BN && gn % BN <= kFoldMax ? gn % BN : 0;
}
__host__ __device__ constexpr int col_tiles(int gn, bool fold) {
  return (gn - (fold ? folded_cols(gn) : 0) + BN - 1) / BN;
}

// The kernels whose stage ring a producer warpgroup runs: the same dW layout.
template <typename T, bool A_MN, bool B_MN>
__host__ __device__ constexpr bool has_producer() {
  return sizeof(T) == 4 && A_MN && B_MN;
}
template <typename T, bool A_MN, bool B_MN>
__host__ __device__ constexpr int block_threads() {
  return A_MN && !has_producer<T, A_MN, B_MN>() ? kThreads : kThreads + kEpiThreads;
}

// Bytes of one swizzled B tile (hi or lo): 128 rows, 136 when the kernel folds.  A producer
// kernel first copies the raw MN-major slab of the same k block into it, 32 k rows of 128
// columns then 32 k rows of the kFoldMax folded ones: the same byte count.
__host__ __device__ constexpr int b_tile_bytes(bool fold) {
  return fold ? kTileBytes + kFoldMax * 128 : kTileBytes;
}
// Bytes of one pipeline stage: the B tile (plus its lo tile for 3xTF32), then the A tile.
__host__ __device__ constexpr int stage_bytes(int passes, bool fold = false) {
  return (passes == 3 ? 2 : 1) * b_tile_bytes(fold) + kATileBytes;
}
// A producer ring's full and empty mbarriers, kMaxStages of each.
constexpr int kRingBarBytes = 2 * kMaxStages * 8;
// What follows the stages: the staging tile of a staged kernel (its column sums live in
// global memory), else the [8][colsum_cols] column-sum accumulator and, with a producer, the
// ring's mbarriers.
__host__ __device__ constexpr int tail_bytes(int colsum_cols, bool staged, bool prod = false) {
  return staged ? kStagingBytes : kWarps * colsum_cols * 4 + (prod ? kRingBarBytes : 0);
}
// Stages that fit beside the tail and the 1 KB alignment slack; at most kMaxStages.  The one
// place that sizes the shared memory of a launch.
__host__ __device__ constexpr int num_stages(int passes, int colsum_cols, bool staged, bool fold = false,
                                             bool prod = false) {
  return (kSmemLimit - 1024 - tail_bytes(colsum_cols, staged, prod)) / stage_bytes(passes, fold) < kMaxStages
             ? (kSmemLimit - 1024 - tail_bytes(colsum_cols, staged, prod)) / stage_bytes(passes, fold)
             : kMaxStages;
}
static_assert(num_stages(3, 1024, false, true) >= 3, "3xTF32 needs three stages beside a 1024-column colsum");
static_assert(num_stages(3, 0, false, true, true) == kMaxStages, "the 3xTF32 dW GEMMs keep four stages");
static_assert(num_stages(1, 0, false, true, true) == kMaxStages, "the TF32 dW GEMMs keep four stages");
static_assert(num_stages(3, 1024, true) >= 3, "3xTF32 needs three stages beside the staging tile");
inline size_t smem_bytes(int passes, int colsum_cols, bool staged, bool fold, bool prod = false) {
  return (size_t)num_stages(passes, colsum_cols, staged, fold, prod) * stage_bytes(passes, fold) +
         (size_t)tail_bytes(colsum_cols, staged, prod) + 1024;
}
static_assert(kMaxStages * stage_bytes(3, true) + kRingBarBytes + 1024 <= kSmemLimit,
              "a 3xTF32 dW ring of four folding stages fits in shared memory");

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// Round-to-nearest TF32 (low 13 mantissa bits cleared).  With RN the residual lo = x - hi is
// at most 2^-12 |x| and zero-mean, so the dropped lo*lo term of the 3xTF32 product is ~2^-24
// and unbiased (a truncating split leaves a one-sided 2^-20 bias over long reductions).
__device__ __forceinline__ float tf32_rn(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// sm_90 shared-memory matrix descriptor: K-major, 128-byte swizzle, 8-row atoms of 1024 B.
__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;                 // leading byte offset (unused here)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;         // stride byte offset
  d |= static_cast<uint64_t>(1) << 62;                 // SWIZZLE_128B
  return d;
}
// MN-major, 128-byte swizzle (bf16 B read with the transpose bit): 64 columns (128 B) per
// swizzle atom, 8 k rows per 1024 B; the next 64 columns start `atom_stride` bytes further.
__device__ __forceinline__ uint64_t desc_sw128_mn(uint32_t saddr, uint32_t atom_stride) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(atom_stride >> 4) << 16;  // leading byte offset: next 64 columns
  d |= static_cast<uint64_t>(1024 >> 4) << 32;         // stride byte offset: next 8 k rows
  d |= static_cast<uint64_t>(1) << 62;                 // SWIZZLE_128B
  return d;
}

__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// 16-byte global -> shared copy; the `bytes` (0..16) first bytes are read, the rest zero-filled.
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() {
  asm volatile("cp.async.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void bar_arrive(int id, int threads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void mbar_init(uint64_t* b, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* b) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(b))
               : "memory");
}
// Returns once the phase of parity `parity` has completed.  On a fresh barrier the phase
// before the first (parity 1) counts as completed.
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n"
      "WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@!p bra WAIT;\n\t}" ::"r"(smem_u32(b)), "r"(parity)
      : "memory");
}
// Arrives once and adds `bytes` to the transactions the current phase waits for.
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)),
               "r"(bytes)
               : "memory");
}

// TMA: the box of a 2-D tensor map at coordinates (c0 innermost, c1) -> shared memory, counted
// on mbarrier `bar` (the whole box, zero-filled outside the tensor); and shared memory -> the
// box, clipped to the tensor, in one bulk group of the issuing thread.
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* map, int c0, int c1,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const void* map, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(c0), "r"(c1), "r"(src)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// Returns once the issuing thread's bulk groups but the N youngest have read their source.
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// ... and have completed their writes.
template <int N>
__device__ __forceinline__ void bulk_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// Every warp of a warpgroup executes these.
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}

#define TFR_WG_D32                                                                           \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, "  \
  "%19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define TFR_WG_D64                                                                           \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, "  \
  "%19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, "   \
  "%36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, "   \
  "%53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define TFR_WG_OUT32(d)                                                                      \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),       \
      "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]),             \
      "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),          \
      "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),          \
      "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])

// D[64 x N] += A[64 x k] B[k x N]; A: four registers of this thread's fragment, B: descriptor.
// acc[0] holds columns 0..63, acc[1] columns 64..127 (the m64n128 accumulator layout).
// TF32 (k = 8): fp32 bits, the low 13 are ignored.
__device__ __forceinline__ void mma_tf32_n64(float (&d)[2][32], const uint32_t (&a)[4], uint64_t db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " TFR_WG_D32
               ", {%32, %33, %34, %35}, %36, 1, 1, 1;"
               : TFR_WG_OUT32(d[0])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}
__device__ __forceinline__ void mma_tf32_n128(float (&d)[2][32], const uint32_t (&a)[4], uint64_t db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " TFR_WG_D64
               ", {%64, %65, %66, %67}, %68, 1, 1, 1;"
               : TFR_WG_OUT32(d[0]), TFR_WG_OUT32(d[1])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}
// m64n136: d as m64n128, then t holds columns 128..135 (t[0..1] row g, t[2..3] row g + 8,
// columns 128 + 2 (lane % 4) and the one after it).
__device__ __forceinline__ void mma_tf32_n136(float (&d)[2][32], float (&t)[4], const uint32_t (&a)[4],
                                              uint64_t db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n136k8.f32.tf32.tf32 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, "
               "%18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, "
               "%34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, "
               "%50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, "
               "%66, %67}, {%68, %69, %70, %71}, %72, 1, 1, 1;"
               : TFR_WG_OUT32(d[0]), TFR_WG_OUT32(d[1]),
                 "+f"(t[0]), "+f"(t[1]), "+f"(t[2]), "+f"(t[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}
// bf16 / fp16 (k = 16): two elements per register.  TRANS_B: B is MN-major in shared memory.
template <typename T, int TRANS_B>
__device__ __forceinline__ void mma16_n64(float (&d)[2][32], const uint32_t (&a)[4], uint64_t db) {
  if constexpr (std::is_same_v<T, __half>)
    asm volatile("wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " TFR_WG_D32
                 ", {%32, %33, %34, %35}, %36, 1, 1, 1, %37;"
                 : TFR_WG_OUT32(d[0])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "n"(TRANS_B));
  else
    asm volatile("wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " TFR_WG_D32
                 ", {%32, %33, %34, %35}, %36, 1, 1, 1, %37;"
                 : TFR_WG_OUT32(d[0])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "n"(TRANS_B));
}
template <typename T, int TRANS_B>
__device__ __forceinline__ void mma16_n128(float (&d)[2][32], const uint32_t (&a)[4], uint64_t db) {
  if constexpr (std::is_same_v<T, __half>)
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " TFR_WG_D64
                 ", {%64, %65, %66, %67}, %68, 1, 1, 1, %69;"
                 : TFR_WG_OUT32(d[0]), TFR_WG_OUT32(d[1])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "n"(TRANS_B));
  else
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " TFR_WG_D64
                 ", {%64, %65, %66, %67}, %68, 1, 1, 1, %69;"
                 : TFR_WG_OUT32(d[0]), TFR_WG_OUT32(d[1])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "n"(TRANS_B));
}
#undef TFR_WG_D32
#undef TFR_WG_D64
#undef TFR_WG_OUT32

// Element traits: a 16-byte chunk holds EPC elements; a 128-byte row holds BK of k.
template <typename T> struct Elem;
template <> struct Elem<float> { static constexpr int EPC = 4; static constexpr int BK = 32; };
template <> struct Elem<__nv_bfloat16> { static constexpr int EPC = 8; static constexpr int BK = 64; };
template <> struct Elem<__half> { static constexpr int EPC = 8; static constexpr int BK = 64; };

// Byte offset of 16-byte chunk `kc` of row `row` in a K-major 128B-swizzled tile.
__device__ __forceinline__ int swz_chunk(int row, int kc) { return row * 128 + (((kc ^ row) & 7) << 4); }

// Stores columns r .. r + 3 of k row k of an MN-major fp32 B slab at their K-major places in
// the swizzled tile(s) and, for 3xTF32 (SPLIT), split into hi / lo.  The caller gives a warp 8
// consecutive column chunks (one 128-byte line per k row) of 4 consecutive k rows, so all 32
// lanes of a scalar K-major store write the same 16-byte k chunk position of their rows and
// differ only in the row's swizzle phase (row mod 8) and in k mod 4.  Store step j of a lane
// writes column r + ((j + s) & 3) of its chunk, s = (lane mod 8) / 2: the 8 lanes of a k row
// then write rows of 8 different phases, and the 32 lanes hit 32 different banks.  (With
// s = 0 they would write rows of 2 phases: 4 ways of bank conflict.)
template <bool SPLIT>
__device__ __forceinline__ void store_mn_chunk(unsigned char* hi, unsigned char* lo, float4 v, int k, int r) {
  const int s = (threadIdx.x & 7) >> 1;
  // rotate the chunk left by s with selects (a dynamic index would go to local memory)
  float e0 = v.x, e1 = v.y, e2 = v.z, e3 = v.w;
  if (s & 1) {
    const float t = e0;
    e0 = e1; e1 = e2; e2 = e3; e3 = t;
  }
  if (s & 2) {
    float t = e0; e0 = e2; e2 = t;
    t = e1; e1 = e3; e3 = t;
  }
  const float e[4] = {e0, e1, e2, e3};   // e[j]: column r + ((j + s) & 3)
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int off = swz_chunk(r + ((j + s) & 3), k >> 2) + (k & 3) * 4;
    if (SPLIT) {
      const float h = tf32_rn(e[j]);
      *reinterpret_cast<float*>(hi + off) = h;
      *reinterpret_cast<float*>(lo + off) = e[j] - h;
    } else {
      *reinterpret_cast<float*>(hi + off) = e[j];
    }
  }
}
// Stores a 4 x 4 block of an MN-major fp32 B slab, v[i] = columns r .. r + 3 of k row 4 kc + i,
// at its K-major places: per column one 16-byte store of its 4 k (split into hi / lo for
// 3xTF32).  Store step j of a lane writes column r + ((j + s) & 3), s = (lane mod 8) / 2, as
// in store_mn_chunk: when the 8 lanes of a quarter warp hold 8 consecutive 4-column groups of
// the same kc, they write rows of 8 different swizzle phases, all 32 banks once.
template <bool SPLIT>
__device__ __forceinline__ void store_mn_block(unsigned char* hi, unsigned char* lo, const float4 (&v)[4],
                                               int kc, int r) {
  const int s = (threadIdx.x & 7) >> 1;
  float4 c0 = make_float4(v[0].x, v[1].x, v[2].x, v[3].x), c1 = make_float4(v[0].y, v[1].y, v[2].y, v[3].y);
  float4 c2 = make_float4(v[0].z, v[1].z, v[2].z, v[3].z), c3 = make_float4(v[0].w, v[1].w, v[2].w, v[3].w);
  if (s & 1) {   // rotate the columns left by s with selects
    const float4 t = c0;
    c0 = c1; c1 = c2; c2 = c3; c3 = t;
  }
  if (s & 2) {
    float4 t = c0; c0 = c2; c2 = t;
    t = c1; c1 = c3; c3 = t;
  }
  const float4 c[4] = {c0, c1, c2, c3};   // c[j]: column r + ((j + s) & 3)
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int off = swz_chunk(r + ((j + s) & 3), kc);
    if (SPLIT) {
      const float4 h = make_float4(tf32_rn(c[j].x), tf32_rn(c[j].y), tf32_rn(c[j].z), tf32_rn(c[j].w));
      *reinterpret_cast<float4*>(hi + off) = h;
      *reinterpret_cast<float4*>(lo + off) = make_float4(c[j].x - h.x, c[j].y - h.y, c[j].z - h.z, c[j].w - h.w);
    } else {
      *reinterpret_cast<float4*>(hi + off) = c[j];
    }
  }
}
// Stores element (k, folded column c) of an MN-major slab at K-major row BN + c.  The 32
// lanes of a warp store 4 k of one 16-byte chunk position into 8 rows of 8 different swizzle
// phases: 32 different banks.
template <bool SPLIT>
__device__ __forceinline__ void store_mn_tail(unsigned char* hi, unsigned char* lo, float v, int k, int c) {
  const int off = swz_chunk(BN + c, k >> 2) + (k & 3) * 4;
  if (SPLIT) {
    const float h = tf32_rn(v);
    *reinterpret_cast<float*>(hi + off) = h;
    *reinterpret_cast<float*>(lo + off) = v - h;
  } else {
    *reinterpret_cast<float*>(hi + off) = v;
  }
}

// The register-staged operand of the K-major-A kernel: an MN-major fp32 B tile ([k][n], n
// contiguous) of 128 columns x 32 k, loaded by the 256 MMA threads, transposed into the K-major
// swizzled tile(s) by store_mn_chunk and, for 3xTF32, split into hi / lo.
struct BTileMN {
  float4 v[4];
  __device__ __forceinline__ static void chunk(int i, int& k, int& r) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    k = (lane >> 3) + 4 * (warp / 4) + 8 * i;
    r = ((lane & 7) + 8 * (warp % 4)) * 4;
  }
  __device__ __forceinline__ void load(const float* base, int ld, int r0, int rows, int k0, int ks) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int k, r;
      chunk(i, k, r);
      const int n = (k0 + k < ks) ? min(4, rows - r) : 0;
      const float* p = base + static_cast<size_t>(k0 + k) * ld + r0 + r;
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (n >= 4) {
        v[i] = __ldg(reinterpret_cast<const float4*>(p));
      } else {
        if (n > 0) v[i].x = p[0];
        if (n > 1) v[i].y = p[1];
        if (n > 2) v[i].z = p[2];
      }
    }
  }
  template <bool SPLIT>
  __device__ __forceinline__ void store(unsigned char* hi, unsigned char* lo) const {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int k, r;
      chunk(i, k, r);
      store_mn_chunk<SPLIT>(hi, lo, v[i], k, r);
    }
  }
};

// The producer warpgroup of a dW kernel (TF32, A and B MN-major): it runs the stage ring of the
// two MMA warpgroups.  It walks the CTA's (tile, k block) sequence as they do, across tiles,
// block g in stage g mod stages, and per block
//   issues:   once the MMA warps have released the stage (empty[s]), the cp.async copies of the
//             block's A tile (MN-major, padded) and of its raw MN-major B slab into the stage's
//             B tile (the pre-split lo slab into the lo tile): 128 columns, then the folded
//             remainder's 8 (zero on a tile without it, whose m64n136 reads them too).  One
//             cp.async group per block;
//   finishes it, depth = stages - 2 blocks later and before it waits to issue the next one:
//             once the block's group has landed, each thread reads two 4 x 4 blocks (4 k rows
//             of 4 columns) and 2 folded elements of the slab, and after a barrier over the
//             producer threads writes them back transposed into the swizzled K-major tile, one
//             16-byte store per column of a block, split for 3xTF32 (hi = tf32_rn(x),
//             lo = x - hi, as the A split); then it fences the writes to the async proxy and
//             arrives at full[s].
// The MMA warps hold only the stage whose group they issue and the one of the group still in
// flight before it, so with 4 stages a block's copies have two blocks' time to land.  Block b of
// a thread covers k chunk slot / 4 and column group 8 (slot % 4) + lane % 8, slot = 4 warp +
// lane / 8 + 16 b: a quarter warp reads 128 contiguous bytes of a k row, and stores rows of 8
// different swizzle phases (store_mn_block).
template <bool P3, bool PRE_B, bool FOLD>
__device__ __forceinline__ void producer_ring(const Args& args, unsigned char* smem, int stages,
                                              uint64_t* full, uint64_t* empty) {
  constexpr int kBTile = b_tile_bytes(FOLD);
  constexpr int kStage = stage_bytes(P3 ? 3 : 1, FOLD);
  constexpr int kAOff = (P3 ? 2 : 1) * kBTile;
  constexpr int kSlabPitch = BN * 4;   // bytes per k row of the raw slab
  const int pt = threadIdx.x - kThreads, lane = pt & 31, pw = pt >> 5;
  const float* A = static_cast<const float*>(args.A);
  const float* B = static_cast<const float*>(args.B);
  const float* Blo = static_cast<const float*>(args.B_lo);
  const int nkb_total = (args.GK + Elem<float>::BK - 1) / Elem<float>::BK;
  const int tiles_mn = args.m_tiles * args.n_tiles;
  const int total = tiles_mn * args.splits;
  const int fold = FOLD ? folded_cols(args.GN) : 0;
  const uint32_t smem_base = smem_u32(smem);

  // raw slab of k rows k0 .. k0 + 31: columns n0 .. n0 + 127, then `tail` folded ones
  auto copy_slab = [&](const float* src, uint32_t dst, int n0, int k0, int tail) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = pt + i * kEpiThreads;
      const int k = c >> 5, nc = c & 31, n = n0 + nc * 4;
      const int cnt = k0 + k < args.GK ? min(max(args.GN - n, 0), 4) : 0;
      const float* p = cnt > 0 ? src + static_cast<size_t>(k0 + k) * args.ldb + n : src;
      cp_async16(dst + k * kSlabPitch + nc * 16, p, cnt * 4);
    }
    if (FOLD && pt < 64) {   // [32 k][8 columns], two chunks per k row
      const int k = pt >> 1, h = pt & 1;
      const int cnt = k0 + k < args.GK ? min(max(tail - 4 * h, 0), 4) : 0;
      const float* p = cnt > 0 ? src + static_cast<size_t>(k0 + k) * args.ldb + n0 + BN + 4 * h : src;
      cp_async16(dst + kTileBytes + k * 32 + h * 16, p, cnt * 4);
    }
  };
  // the slab in tile `t`, transposed in place (and split into t, lo)
  auto transpose = [&](unsigned char* t, unsigned char* lo, auto split) {
    constexpr bool SPLIT = decltype(split)::value;
    // opaque per call: keeps ptxas from holding every store offset in registers across blocks
    int qw = pw * 4 + (lane >> 3), q = pt;
    asm volatile("" : "+r"(qw), "+r"(q));
    float4 v[2][4];
    float tv[2];
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const int slot = qw + 16 * b, kc = slot >> 2, r = 4 * (8 * (slot & 3) + (lane & 7));
#pragma unroll
      for (int i = 0; i < 4; ++i)
        v[b][i] = *reinterpret_cast<const float4*>(t + (4 * kc + i) * kSlabPitch + r * 4);
    }
    if (FOLD) {
#pragma unroll
      for (int e = 0; e < 2; ++e)
        tv[e] = *reinterpret_cast<const float*>(t + kTileBytes + ((q >> 3) + 16 * e) * 32 + (q & 7) * 4);
    }
    bar_sync(kBarProd, kEpiThreads);   // the whole slab is read before any of it is overwritten
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const int slot = qw + 16 * b;
      store_mn_block<SPLIT>(t, lo, v[b], slot >> 2, 4 * (8 * (slot & 3) + (lane & 7)));
    }
    if (FOLD) {
#pragma unroll
      for (int e = 0; e < 2; ++e) store_mn_tail<SPLIT>(t, lo, tv[e], (q >> 3) + 16 * e, q & 7);
    }
  };
  // `younger`: cp.async groups committed after the block's own, which may still be pending
  auto finish = [&](int s, int younger) {
    if (younger > 0) cp_async_wait<1>();
    else cp_async_wait<0>();
    bar_sync(kBarProd, kEpiThreads);   // the copies of every producer thread have landed
    unsigned char* sb = smem + s * kStage;
    if (PRE_B) {
      transpose(sb, nullptr, std::false_type{});
      transpose(sb + kBTile, nullptr, std::false_type{});
    } else {
      transpose(sb, sb + kBTile, std::integral_constant<bool, P3>{});
    }
    fence_proxy_async();   // st.shared writes -> visible to the tensor cores
    __syncwarp();
    if (lane == 0) mbar_arrive(full + s);   // one arrival per producer warp
  };

  const int depth = stages - 2;
  int is = 0, fs = 0, pending = 0;   // stage of the next block to issue / to finish
  uint32_t eph = 1;                  // parity of the empty phase the issue waits for
  for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
    const int z = tile / tiles_mn;
    const int rt = tile - z * tiles_mn;
    const int m0 = (rt / args.n_tiles) * BM, n0 = (rt % args.n_tiles) * BN;
    const int kb0 = z * args.kb_per_split;
    const int nkb = max(min(nkb_total, kb0 + args.kb_per_split) - kb0, 0);
    const int tail = FOLD && n0 + BN + fold == args.GN ? fold : 0;
    for (int kb = 0; kb < nkb; ++kb) {
      // the oldest block first: its transpose does not wait for a stage to come free
      if (pending == depth) {
        finish(fs, depth - 1);
        fs = fs + 1 == stages ? 0 : fs + 1;
        --pending;
      }
      mbar_wait(empty + is, eph);
      const uint32_t st = smem_base + is * kStage;
      const int k0 = (kb0 + kb) * Elem<float>::BK;
#pragma unroll
      for (int i = 0; i < 8; ++i) {   // A: [32 k rows][32 chunks of m]
        const int c = pt + i * kEpiThreads;
        const int k = c >> 5, mc = c & 31, m = m0 + mc * 4;
        const int cnt = (k0 + k < args.GK && m < args.GM) ? min(4, args.GM - m) : 0;
        const float* p = cnt > 0 ? A + static_cast<size_t>(k0 + k) * args.lda + m : A;
        cp_async16(st + kAOff + k * kAPitchMN + mc * 16, p, cnt * 4);
      }
      copy_slab(B, st, n0, k0, tail);
      if (PRE_B) copy_slab(Blo, st + kBTile, n0, k0, tail);
      cp_async_commit();
      if (++is == stages) {
        is = 0;
        eph ^= 1u;
      }
      ++pending;
    }
  }
  for (; pending > 0; --pending) {
    finish(fs, pending - 1);
    fs = fs + 1 == stages ? 0 : fs + 1;
  }
}

// producer_ring's slab copy and in-place transpose, for a kernel that runs its own ring
// (mlp_tc_fused_bwd.cu).  copy_slab: producer thread pt (0..127) copies k rows k0 .. k0 + 31 of B
// [GK][GN] (row pitch ldb) raw into the B tile at `dst`, columns n0 .. n0 + 127 as 32 rows of
// BN * 4 bytes, then (FOLD) the `tail` folded columns past them as 32 rows of 32 bytes at
// kTileBytes; zero past GK and GN.  One cp.async group's worth; the caller commits it.
template <bool FOLD>
__device__ __forceinline__ void copy_slab(const float* src, int ldb, int GK, int GN, uint32_t dst,
                                          int n0, int k0, int tail, int pt) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = pt + i * kEpiThreads;
    const int k = c >> 5, nc = c & 31, n = n0 + nc * 4;
    const int cnt = k0 + k < GK ? min(max(GN - n, 0), 4) : 0;
    const float* p = cnt > 0 ? src + static_cast<size_t>(k0 + k) * ldb + n : src;
    cp_async16(dst + k * (BN * 4) + nc * 16, p, cnt * 4);
  }
  if (FOLD && pt < 64) {   // [32 k][8 columns], two chunks per k row
    const int k = pt >> 1, h = pt & 1;
    const int cnt = k0 + k < GK ? min(max(tail - 4 * h, 0), 4) : 0;
    const float* p = cnt > 0 ? src + static_cast<size_t>(k0 + k) * ldb + n0 + BN + 4 * h : src;
    cp_async16(dst + kTileBytes + k * 32 + h * 16, p, cnt * 4);
  }
}
// Producer thread pt: the landed slab in tile `t` transposed in place into the swizzled K-major
// tile (and, SPLIT, split into t = hi and lo).  Every producer thread takes part: it holds a
// barrier over the 128 between its reads and its writes.
template <bool SPLIT, bool FOLD>
__device__ __forceinline__ void transpose_slab(unsigned char* t, unsigned char* lo, int pt) {
  const int lane = pt & 31, pw = pt >> 5;
  // opaque per call: keeps ptxas from holding every store offset in registers across blocks
  int qw = pw * 4 + (lane >> 3), q = pt;
  asm volatile("" : "+r"(qw), "+r"(q));
  float4 v[2][4];
  float tv[2];
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    const int slot = qw + 16 * b, kc = slot >> 2, r = 4 * (8 * (slot & 3) + (lane & 7));
#pragma unroll
    for (int i = 0; i < 4; ++i)
      v[b][i] = *reinterpret_cast<const float4*>(t + (4 * kc + i) * (BN * 4) + r * 4);
  }
  if (FOLD) {
#pragma unroll
    for (int e = 0; e < 2; ++e)
      tv[e] = *reinterpret_cast<const float*>(t + kTileBytes + ((q >> 3) + 16 * e) * 32 + (q & 7) * 4);
  }
  bar_sync(kBarProd, kEpiThreads);   // the whole slab is read before any of it is overwritten
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    const int slot = qw + 16 * b;
    store_mn_block<SPLIT>(t, lo, v[b], slot >> 2, 4 * (8 * (slot & 3) + (lane & 7)));
  }
  if (FOLD) {
#pragma unroll
    for (int e = 0; e < 2; ++e) store_mn_tail<SPLIT>(t, lo, tv[e], (q >> 3) + 16 * e, q & 7);
  }
}

// 16-bit stores of C (H: bf16 or fp16), rounded to nearest even.  fp16 keeps subnormals and
// rounds magnitudes past its range to inf, which the stores pass on.
template <typename H>
__device__ __forceinline__ uint32_t pack16(float lo, float hi) {
  uint32_t r;
  if constexpr (std::is_same_v<H, __half>) asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  else asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
template <typename H>
__device__ __forceinline__ H to16(float x) {
  if constexpr (std::is_same_v<H, __half>) return __float2half_rn(x);
  else return __float2bfloat16_rn(x);
}
template <typename H>
__device__ __forceinline__ float round16(float x) {   // the value a 16-bit store keeps
  if constexpr (std::is_same_v<H, __half>) return __half2float(__float2half_rn(x));
  else return __bfloat162float(__float2bfloat16_rn(x));
}
// The 16-bit type of C when OUT16: the operand type (bf16 when the operands are fp32, a case
// no launch instantiates with OUT16).
template <typename T>
using Out16 = std::conditional_t<sizeof(T) == 2, T, __nv_bfloat16>;

// The epilogue warpgroup of a staged kernel: walks the CTA's tiles as the MMA warpgroups do and
// finishes each from the staging tile `stg`.  Warp `ew` takes rows 32 ew .. 32 ew + 31, a lane
// 4 adjacent columns of each, so a row is stored as one 512-byte line and the eight lanes of a
// 32-column chunk assemble its sign word with three shuffles.  On a tile of at most 64 live columns
// the warp takes two rows at a time instead, lanes 0-15 row i and lanes 16-31 row i + 1 (a
// 256-byte line each), so no lane idles.  Column tests are made once per tile, row tests once
// per row.  Nothing in the row loop waits on global memory: the tile's mask words are loaded
// into registers while the previous tile's column sums run, and reach their rows by shuffle.
// The fast loop stores sign words 8 rows at a time, one word per lane: 32-byte sectors whole.
// Column sums: the row pass writes the stored fp32 values back to the staging tile; thread t
// then owns tile column t, adds the 16 rows of each of the 8 row groups in the order the
// accumulator layout gave them (rows g and g + 8, then g pairs 1, 2, 4 apart) and adds that to
// its running sum in the group's slot in global memory.  Slot and column always meet the same
// thread, so plain loads and stores keep the running sums; the loads are issued before the row
// pass, so the tile's tail only stores.
template <typename H, bool OUT16>
__device__ __forceinline__ void epilogue_warpgroup(const Args& args, float* stg) {
  const int lane = threadIdx.x & 31;
  const int et = threadIdx.x - kThreads, ew = et >> 5;
  const int tiles_mn = args.m_tiles * args.n_tiles;
  const int total = tiles_mn * args.splits;
  if (args.colsum_cols) {
    for (int w = 0; w < kWarps; ++w) {
      float* dst = args.colsum + static_cast<size_t>(blockIdx.x * kWarps + w) * args.colsum_stride;
      for (int c = et; c < args.GN; c += kEpiThreads) dst[c] = 0.f;
    }
  }
  // Mask words of a tile's 32 rows of this warp: lane 8 p + q holds, in mw[k], the word of
  // plane p (tile columns 32 p .. 32 p + 31) for row 8 k + q; a warp's load is 4 whole sectors.
  // Zero past GM and GN.
  uint32_t mw[4] = {0u, 0u, 0u, 0u};
  auto load_masks = [&](int tile) {
    const int r = tile % tiles_mn;
    const int m0 = (r / args.n_tiles) * BM, n0 = (r % args.n_tiles) * BN;
    const int c = n0 + 32 * (lane >> 3), row = m0 + ew * 32 + (lane & 7);
    const uint32_t* p = args.bits_in + static_cast<size_t>(c >> 5) * args.GM + row;
#pragma unroll
    for (int k = 0; k < 4; ++k) mw[k] = c < args.GN && row + 8 * k < args.GM ? __ldg(p + 8 * k) : 0u;
  };
  // the word of row `rw` (0..31 within the warp) in plane `pl` of the tile.  The shuffle reads
  // the source lane's choice of register, so rw >> 3 must agree across the warp: it does, as
  // the two rows of a paired step are i and i + 1 with i even.
  auto mask_word = [&](int rw, int pl) {
    const int k = rw >> 3;
    const uint32_t m = k == 0 ? mw[0] : k == 1 ? mw[1] : k == 2 ? mw[2] : mw[3];
    return __shfl_sync(0xffffffffu, m, 8 * pl + (rw & 7));
  };
  const bool masks = args.epi == EPI_MASK_BITS;
  if (masks && static_cast<int>(blockIdx.x) < total) load_masks(blockIdx.x);
  for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
    const int z = tile / tiles_mn;
    const int r = tile - z * tiles_mn;
    const int m0 = (r / args.n_tiles) * BM, n0 = (r % args.n_tiles) * BN;
    // lane mapping: a lane's columns 4 cl .. 4 cl + 3 of row i + half, rows advancing by step
    const bool pair = args.GN - n0 <= 64;
    const int cl = pair ? lane & 15 : lane, half = pair ? lane >> 4 : 0;
    const int col = n0 + 4 * cl;
    const int live = min(max(args.GN - col, 0), 4);   // live columns of this lane
    // the running column sums this tile adds to, loaded while the row pass runs
    float run[kWarps];
    const bool sums = args.colsum_cols && n0 + et < args.GN;
    if (sums) {
#pragma unroll
      for (int w = 0; w < kWarps; ++w)
        run[w] = args.colsum[static_cast<size_t>(blockIdx.x * kWarps + w) * args.colsum_stride + n0 + et];
    }
    float b4[4] = {0.f, 0.f, 0.f, 0.f};
    if (args.epi == EPI_BIAS_ACT) {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (j < live) b4[j] = __ldg(args.bias + col + j);
    }
    float* Cf = static_cast<float*>(args.C) + static_cast<size_t>(z) * args.split_stride;
    H* Cb = static_cast<H*>(args.C);
    // vector stores need a row pitch of a multiple of 4 elements and a 16-byte (bf16: 8-byte)
    // aligned base (C and every split-K slice C + z * split_stride)
    const uintptr_t cbase = OUT16 ? reinterpret_cast<uintptr_t>(Cb) : reinterpret_cast<uintptr_t>(Cf);
    const bool vec_ok = (args.ldc % 4) == 0 && (cbase & (OUT16 ? 7u : 15u)) == 0;
    const bool vec4 = live == 4 && vec_ok;
    // this lane's plane of sign words (tile columns 32 mpl .. 32 mpl + 31); every lane of a
    // live plane stores rows in the fast loop, also those whose own columns lie past GN
    const int mpl = cl >> 3, pcol = n0 + 32 * mpl;
    uint32_t* bplane = args.bits_out && pcol < args.GN
                           ? args.bits_out + static_cast<size_t>(pcol >> 5) * args.GM : nullptr;
    // a row's sign word from the nibbles of the 8 lanes of its plane.  Shuffles, not a redux:
    // the redux's member mask differs between the warp's 4 groups, which sends it down the
    // divergent path.
    auto sign_word = [&](uint32_t nib) {
      uint32_t w = nib << (4 * (lane & 7));
      w |= __shfl_xor_sync(0xffffffffu, w, 1);
      w |= __shfl_xor_sync(0xffffffffu, w, 2);
      w |= __shfl_xor_sync(0xffffffffu, w, 4);
      return w;
    };
    bar_sync(kBarFull, kThreads + kEpiThreads);
    // Full row blocks whose lanes hold 4 live columns or none, stored as vectors: the row loop
    // has no bounds tests, its epilogue kind and lane mapping are compile-time constants and its
    // pointers advance by a constant per row.  Everything else takes the general loop below it.
    auto fast_rows = [&](auto kind, auto paired) {
      constexpr int EPI = decltype(kind)::value;
      constexpr bool PAIR = decltype(paired)::value;
      constexpr int STEP = PAIR ? 2 : 1;
      using V = std::conditional_t<OUT16, uint2, float4>;
      const bool on = live == 4, relu = args.act == TFR_ACT_RELU;
      const int row0 = m0 + ew * 32;
      const float4* sp =
          reinterpret_cast<const float4*>(stg + (ew * 32 + half) * kStagingPitch + 4 * cl);
      const size_t coff = static_cast<size_t>(row0 + half) * args.ldc + col;
      V* cp = OUT16 ? reinterpret_cast<V*>(Cb + coff) : reinterpret_cast<V*>(Cf + coff);
      const int cstep = args.ldc / 4;
      // sign words: lane q of a group keeps the word of row 8 b + q and stores it once the
      // group's 8 rows are done (with two rows a step, half h keeps the rows of parity h)
      uint32_t* bo = bplane && (!PAIR || (lane & 1) == half) ? bplane + row0 + (lane & 7) : nullptr;
      uint32_t keep = 0u;
      const int sh = (4 * cl) & 31;
#pragma unroll 4
      for (int i = 0; i < 32; i += STEP) {
        float4 v = sp[i * (kStagingPitch / 4)];
        if (EPI == EPI_BIAS_ACT) {
          v.x += b4[0]; v.y += b4[1]; v.z += b4[2]; v.w += b4[3];
          if (relu) {
            v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
          }
        } else if (EPI == EPI_MASK_BITS) {
          const uint32_t w = mask_word(i + half, mpl) >> sh;
          if (!(w & 1u)) v.x = 0.f;
          if (!(w & 2u)) v.y = 0.f;
          if (!(w & 4u)) v.z = 0.f;
          if (!(w & 8u)) v.w = 0.f;
        }
        if (!on) v = make_float4(0.f, 0.f, 0.f, 0.f);
        const uint2 packed = make_uint2(pack16<H>(v.x, v.y), pack16<H>(v.z, v.w));
        if (args.bits_out) {
          auto pos = [](float y) {   // the sign bit is that of the stored value
            return (OUT16 ? round16<H>(y) : y) > 0.f ? 1u : 0u;
          };
          const uint32_t nib = pos(v.x) | pos(v.y) << 1 | pos(v.z) << 2 | pos(v.w) << 3;
          const uint32_t w = sign_word(nib);
          if (((i + half) & 7) == (lane & 7)) keep = w;
          if (((i + STEP) & 7) == 0 && bo) bo[i & ~7] = keep;
        }
        if (args.colsum_cols) const_cast<float4*>(sp)[i * (kStagingPitch / 4)] = v;
        if (on) {
          if (OUT16) *reinterpret_cast<uint2*>(cp + static_cast<size_t>(i) * cstep) = packed;
          else *reinterpret_cast<float4*>(cp + static_cast<size_t>(i) * cstep) = v;
        }
      }
    };
    auto fast_kind = [&](auto kind) {
      if (pair) fast_rows(kind, std::true_type{});
      else fast_rows(kind, std::false_type{});
    };
    const bool fast = m0 + BM <= args.GM && (args.GN % 4) == 0 && vec_ok && !args.store_transposed;
    bool general = false;
    if (fast && args.epi == EPI_STORE) fast_kind(std::integral_constant<int, EPI_STORE>{});
    else if (fast && args.epi == EPI_BIAS_ACT) fast_kind(std::integral_constant<int, EPI_BIAS_ACT>{});
    else if (fast && masks) fast_kind(std::integral_constant<int, EPI_MASK_BITS>{});
    else general = true;
    const int step = pair ? 2 : 1;
#pragma unroll 1
    for (int i = general ? 0 : 32; i < 32; i += step) {
      const int rl = ew * 32 + i + half, row = m0 + rl;
      const bool rlive = row < args.GM;
      float* sp = stg + rl * kStagingPitch + 4 * cl;
      const float4 v = *reinterpret_cast<const float4*>(sp);
      float x[4] = {v.x, v.y, v.z, v.w};
      uint32_t wbits = 0u, nib = 0u;
      if (masks) wbits = mask_word(i + half, mpl);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float y = x[j];
        if (args.epi == EPI_BIAS_ACT) {
          y += b4[j];
          if (args.act == TFR_ACT_RELU) y = fmaxf(y, 0.f);
        } else if (args.epi == EPI_MASK_POS) {
          if (args.act == TFR_ACT_RELU && rlive && j < live &&
              !(__ldg(args.aux + static_cast<size_t>(row) * args.ldc + col + j) > 0.f))
            y = 0.f;
        } else if (args.epi == EPI_MASK_BITS) {
          if (!((wbits >> ((4 * cl + j) & 31)) & 1u)) y = 0.f;
        }
        if (!rlive || j >= live) y = 0.f;
        x[j] = y;   // column sums take the fp32 value, sign bits the stored one
        const float stored = OUT16 ? round16<H>(y) : y;
        nib |= (stored > 0.f ? 1u : 0u) << j;
      }
      if (args.bits_out) {
        const uint32_t w = sign_word(nib);
        if (bplane && (lane & 7) == 0 && rlive) bplane[row] = w;
      }
      if (args.colsum_cols) *reinterpret_cast<float4*>(sp) = make_float4(x[0], x[1], x[2], x[3]);
      if (!rlive || live == 0) continue;
      if (OUT16) {
        H* p = Cb + static_cast<size_t>(row) * args.ldc + col;
        if (vec4) {
          *reinterpret_cast<uint2*>(p) = make_uint2(pack16<H>(x[0], x[1]), pack16<H>(x[2], x[3]));
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (j < live) p[j] = to16<H>(x[j]);
        }
      } else if (args.store_transposed) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (j < live) Cf[static_cast<size_t>(col + j) * args.ldc + row] = x[j];
      } else {
        float* p = Cf + static_cast<size_t>(row) * args.ldc + col;
        if (vec4) {
          *reinterpret_cast<float4*>(p) = make_float4(x[0], x[1], x[2], x[3]);
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (j < live) p[j] = x[j];
        }
      }
    }
    if (masks && tile + gridDim.x < total) load_masks(tile + gridDim.x);   // in flight over the sums
    if (args.colsum_cols) {
      bar_sync(kBarEpi, kEpiThreads);   // the write-backs of all four warps
      if (sums) {
#pragma unroll
        for (int w = 0; w < kWarps; ++w) {
          const float* p = stg + w * 16 * kStagingPitch + et;
          float s[8];
#pragma unroll
          for (int g = 0; g < 8; ++g) s[g] = p[g * kStagingPitch] + p[(g + 8) * kStagingPitch];
          const float sum = ((s[0] + s[1]) + (s[2] + s[3])) + ((s[4] + s[5]) + (s[6] + s[7]));
          args.colsum[static_cast<size_t>(blockIdx.x * kWarps + w) * args.colsum_stride + n0 + et] =
              run[w] + sum;
        }
      }
    }
    if (tile + gridDim.x < total) bar_arrive(kBarFree, kThreads + kEpiThreads);
  }
}

// PASSES: 1 (one product) or 3 (3xTF32: Ahi Bhi + Alo Bhi + Ahi Blo; float only).
// PRE_B: B comes pre-split (B = hi parts, B_lo = lo parts).  OUT16: C has the operands' 16-bit
// type (row-major).
// Staged (K-major A): a third warpgroup runs the epilogue from a staging tile.
// Shared memory: num_stages x {B hi, [B lo,] A}, then the staging tile (staged) or
// [8][colsum_cols] floats.  FOLD (launched when GN has a remainder to fold): the last column
// tile owns it, B tiles have 136 rows and wide tiles issue m64n136.
template <typename T, bool A_MN, bool B_MN, int PASSES, bool PRE_B, bool OUT16, bool FOLD>
__global__ void __launch_bounds__(block_threads<T, A_MN, B_MN>(), 1)
gemm_kernel(const Args args) {
  constexpr bool STAGED = !A_MN;
  constexpr bool PROD = has_producer<T, A_MN, B_MN>();   // a producer warpgroup runs the ring
  constexpr bool F32 = sizeof(T) == 4;
  using H = Out16<T>;
  constexpr int EPC = Elem<T>::EPC;
  constexpr int BK = Elem<T>::BK;
  constexpr int KSTEP = F32 ? 8 : 16;   // k of one wgmma
  constexpr int NKS = BK / KSTEP;
  constexpr bool P3 = PASSES == 3;
  constexpr bool REG_B = F32 && B_MN && !PROD;   // TF32 MN-major B through the MMA warps' registers
  constexpr int kBTile = b_tile_bytes(FOLD);   // offset of the B lo tile
  constexpr int kStage = stage_bytes(PASSES, FOLD);
  constexpr int kAOff = (P3 ? 2 : 1) * kBTile;
  constexpr int kAPitch = A_MN ? kAPitchMN * static_cast<int>(sizeof(T)) / 4 : kAPitchK;
  static_assert(!P3 || F32, "3xTF32 is float only");
  static_assert(!PRE_B || P3, "pre-split B is 3xTF32");
  static_assert(!FOLD || folds<T, A_MN, B_MN>(), "only TF32 with A and B MN-major folds");
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int stages = num_stages(PASSES, args.colsum_cols, STAGED, FOLD, PROD);
  float* cacc = reinterpret_cast<float*>(smem + stages * kStage);   // staged: the staging tile
  // producer ring: full[s] (one arrival per producer warp) and empty[s] (one per MMA warp)
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + stages * kStage + kWarps * args.colsum_cols * 4);
  uint64_t* empty = full + kMaxStages;
  if (STAGED || PROD) {
    if (PROD) {
      if (threadIdx.x == 0) {
        for (int i = 0; i < stages; ++i) {
          mbar_init(full + i, kEpiThreads / 32);
          mbar_init(empty + i, kWarps);
        }
      }
      __syncthreads();
    }
    if (threadIdx.x >= kThreads) {
      setmaxnreg_dec<kEpiRegs>();
      if constexpr (PROD) producer_ring<P3, PRE_B, FOLD>(args, smem, stages, full, empty);
      else epilogue_warpgroup<Out16<T>, OUT16>(args, cacc);
      return;
    }
    setmaxnreg_inc<kMmaRegs>();
  }
  auto mma_sync = [] {   // barrier over the MMA warpgroups
    if (STAGED || PROD) bar_sync(kBarMma, kThreads);
    else __syncthreads();
  };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2, wq = warp & 3;   // warpgroup, warp within it
  const T* A = static_cast<const T*>(args.A);
  const T* B = static_cast<const T*>(args.B);
  const T* Blo = static_cast<const T*>(args.B_lo);
  const int nkb_total = (args.GK + BK - 1) / BK;
  const int tiles_mn = args.m_tiles * args.n_tiles;
  const int total = tiles_mn * args.splits;
  const uint32_t smem_base = smem_u32(smem);
  const int fold = FOLD ? folded_cols(args.GN) : 0;
  // the tile at column n0 owns the folded remainder: columns n0 + 128 .. GN - 1
  auto has_tail = [&](int n0) { return FOLD && n0 + BN + fold == args.GN; };

  if (!STAGED)
    for (int c = threadIdx.x; c < kWarps * args.colsum_cols; c += kThreads) cacc[c] = 0.f;

  // Issues the cp.async copies of k block kb (relative to the split) of the tile at (m0, n0)
  // into stage s: 4 chunks of A and, unless register-staged, 4 chunks of B (and 4 of B lo).
  auto copy_block = [&](int m0, int n0, int kb0, int kb, int s) {
    const int k0 = (kb0 + kb) * BK;
    const uint32_t st = smem_base + s * kStage;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = threadIdx.x + i * kThreads;
      if (!A_MN) {   // [128 rows of m][8 chunks of k]
        const int r = c >> 3, kc = c & 7, k = k0 + kc * EPC;
        const int n = (m0 + r < args.GM && k < args.GK) ? min(EPC, args.GK - k) : 0;
        const T* src = n > 0 ? A + static_cast<size_t>(m0 + r) * args.lda + k : A;
        cp_async16(st + kAOff + r * kAPitch + kc * 16, src, n * static_cast<int>(sizeof(T)));
      } else {       // [BK k rows][128 / EPC chunks of m]
        const int k = c / (128 / EPC), mc = c % (128 / EPC), m = m0 + mc * EPC;
        const int n = (k0 + k < args.GK && m < args.GM) ? min(EPC, args.GM - m) : 0;
        const T* src = n > 0 ? A + static_cast<size_t>(k0 + k) * args.lda + m : A;
        cp_async16(st + kAOff + k * kAPitch + mc * 16, src, n * static_cast<int>(sizeof(T)));
      }
    }
    if (!B_MN) {     // [128 rows of n][8 chunks of k], swizzled
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = threadIdx.x + i * kThreads;
        const int r = c >> 3, kc = c & 7, k = k0 + kc * EPC;
        const int n = (n0 + r < args.GN && k < args.GK) ? min(EPC, args.GK - k) : 0;
        const size_t off = n > 0 ? static_cast<size_t>(n0 + r) * args.ldb + k : 0;
        cp_async16(st + swz_chunk(r, kc), B + off, n * static_cast<int>(sizeof(T)));
        if (PRE_B) cp_async16(st + kBTile + swz_chunk(r, kc), Blo + off, n * static_cast<int>(sizeof(T)));
      }
    } else if (!F32) {   // 16-bit [2 atoms of 64 n][64 k rows][8 chunks of n], swizzled
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = threadIdx.x + i * kThreads;
        const int k = c >> 4, nc = c & 15, n = n0 + nc * 8;
        const int cnt = (k0 + k < args.GK && n < args.GN) ? min(8, args.GN - n) : 0;
        const T* src = cnt > 0 ? B + static_cast<size_t>(k0 + k) * args.ldb + n : B;
        cp_async16(st + (nc >> 3) * (BK * 128) + swz_chunk(k, nc & 7), src, cnt * 2);
      }
    }
  };

  // cp.async groups: a tile's prologue commits stages - 2 groups (blocks 0 .. stages - 3),
  // every k block one more (block kb + stages - 2), empty ones included, so that block kb's
  // group is complete once at most stages - 3 younger groups are pending.
  // A producer kernel's MMA warps copy nothing: the producer warpgroup runs the ring.
  BTileMN tb, tbl;
  auto load_b = [&](int n0, int kb) {
    tb.load(reinterpret_cast<const float*>(B), args.ldb, n0, args.GN - n0, kb * BK, args.GK);
    if (PRE_B) tbl.load(reinterpret_cast<const float*>(Blo), args.ldb, n0, args.GN - n0, kb * BK, args.GK);
  };
  auto prologue = [&](int tile) {
    if (PROD) return;
    const int z = tile / tiles_mn;
    const int r = tile - z * tiles_mn;
    const int m0 = (r / args.n_tiles) * BM, n0 = (r % args.n_tiles) * BN;
    const int kb0 = z * args.kb_per_split;
    const int nkb = max(min(nkb_total, kb0 + args.kb_per_split) - kb0, 0);
    for (int p = 0; p < stages - 2; ++p) {
      if (p < nkb) copy_block(m0, n0, kb0, p, p);
      cp_async_commit();
    }
    if (REG_B && nkb > 0) load_b(n0, kb0);
  };

  if (blockIdx.x < total) prologue(blockIdx.x);
  // stage of block kb and, with a producer, the parity of its full phase: a producer ring
  // runs on across tiles
  int s = 0;
  uint32_t fph = 0;
  for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
    const int z = tile / tiles_mn;
    const int r = tile - z * tiles_mn;
    const int m0 = (r / args.n_tiles) * BM, n0 = (r % args.n_tiles) * BN;
    const int kb0 = z * args.kb_per_split;
    const int nkb = max(min(nkb_total, kb0 + args.kb_per_split) - kb0, 0);
    const bool two_n = n0 + 64 < args.GN;           // the second 64 columns hold live columns
    const bool tail = has_tail(n0);

    float acc[2][32], acc_t[4];   // acc_t: the folded remainder columns
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[h][j] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) acc_t[j] = 0.f;

    // The k loop is software-pipelined one wgmma group deep: group kb is issued while group
    // kb - 1 may still run, from its own A fragment set (kb & 1), and `wait_group 1` then
    // retires group kb - 1.  Invariant: at the barrier of block kb every warpgroup has retired
    // every group up to kb - 2, and group kb - 1 may still read its stage.  So the refill after
    // that barrier goes to the stage of block kb - 2 and loads block kb + stages - 2 (copies
    // run stages - 2 blocks ahead), and the stage of block kb, last read by group
    // kb - stages <= kb - 3, may be written before the barrier.
    // With a producer the ring runs on the stage barriers instead: block kb waits for full[s]
    // and, once `wait_group 1` has retired group kb - 1, releases that group's stage at
    // empty[s - 1]; each MMA warp arrives for itself (wait_group is warp-wide), so neither
    // warpgroup waits for the other.
    uint32_t frag_hi[2][NKS][4], frag_lo[2][NKS][4];
    if (!PROD) s = 0;
    auto kblock = [&](int kb, auto set) {
      constexpr int F = decltype(set)::value;   // fragment set: compile-time, stays in registers
      const uint32_t st = smem_base + s * kStage;
      if (PROD) {
        mbar_wait(full + s, fph);   // the producer fenced its stores before it arrived
      } else {
        if (REG_B) {
          unsigned char* sb = smem + s * kStage;
          if (PRE_B) {
            tb.template store<false>(sb, nullptr);
            tbl.template store<false>(sb + kBTile, nullptr);
          } else {
            tb.template store<P3>(sb, sb + kBTile);
          }
        }
        if (stages == 4) cp_async_wait<1>(); else cp_async_wait<0>();
        if (P3 && !B_MN && !PRE_B) {   // K-major B split on the fly: each thread its own chunks
          unsigned char* sb = smem + s * kStage;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int c = threadIdx.x + i * kThreads;
            const int off = swz_chunk(c >> 3, c & 7);
            const float4 x = *reinterpret_cast<const float4*>(sb + off);
            const float4 h = make_float4(tf32_rn(x.x), tf32_rn(x.y), tf32_rn(x.z), tf32_rn(x.w));
            *reinterpret_cast<float4*>(sb + off) = h;
            *reinterpret_cast<float4*>(sb + kBTile + off) =
                make_float4(x.x - h.x, x.y - h.y, x.z - h.z, x.w - h.w);
          }
        }
        fence_proxy_async();   // cp.async and st.shared writes -> visible to the tensor cores
        mma_sync();
        {
          const int nb = kb + stages - 2;
          if (nb < nkb) copy_block(m0, n0, kb0, nb, s >= 2 ? s - 2 : s + stages - 2);
          cp_async_commit();
        }
        if (REG_B && kb + 1 < nkb) load_b(n0, kb0 + kb + 1);   // in flight while the tensor cores run
      }
      {
        // a K tail that is no multiple of BK is zero-filled: skip its all-zero k steps
        const int krem = args.GK - (kb0 + kb) * BK;
        const int ksteps = krem >= BK ? NKS : (krem + KSTEP - 1) / KSTEP;
        // A fragments of every k step (m64 x k, per warp 16 rows): register i holds row
        // g + 8 (i % 2), k t + 4 (i / 2) (TF32) / k pair 2t + 8 (i / 2) (16-bit)
        const int g = lane >> 2, t = lane & 3;
        const int row = wg * 64 + wq * 16 + g;
        const unsigned char* sa = smem + s * kStage + kAOff;
        uint32_t (&ahi)[NKS][4] = frag_hi[F];
        uint32_t (&alo)[NKS][4] = frag_lo[F];
#pragma unroll
        for (int ks = 0; ks < NKS; ++ks) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int rr = row + 8 * (i & 1);
            if (F32) {
              const int k = ks * KSTEP + t + 4 * (i >> 1);
              const float x = *reinterpret_cast<const float*>(
                  sa + (A_MN ? k * kAPitch + rr * 4 : rr * kAPitch + k * 4));
              if (P3) {
                const float h = tf32_rn(x);
                ahi[ks][i] = __float_as_uint(h);
                alo[ks][i] = __float_as_uint(x - h);
              } else {
                ahi[ks][i] = __float_as_uint(x);
              }
            } else {
              const int k = ks * KSTEP + 2 * t + 8 * (i >> 1);
              if (A_MN) {
                const uint32_t e0 = *reinterpret_cast<const unsigned short*>(sa + k * kAPitch + rr * 2);
                const uint32_t e1 = *reinterpret_cast<const unsigned short*>(sa + (k + 1) * kAPitch + rr * 2);
                ahi[ks][i] = e0 | (e1 << 16);
              } else {
                ahi[ks][i] = *reinterpret_cast<const uint32_t*>(sa + rr * kAPitch + k * 2);
              }
            }
          }
        }
        // one wgmma group per block.  Its width and k-step count are chosen outside it so
        // that the group is straight-line code: a branch inside makes ptxas fence every k step.
        auto mmas = [&](auto wide, auto nk) {
          constexpr bool W = decltype(wide)::value;
          constexpr int NK = decltype(nk)::value;
          // the fragments are final before the fence: keeps their computation from sinking
          // past it, where ptxas would fence each wgmma that reads them
#pragma unroll
          for (int ks = 0; ks < NKS; ++ks)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              asm volatile("" : "+r"(ahi[ks][i]));
              if (P3) asm volatile("" : "+r"(alo[ks][i]));
            }
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < NK; ++ks) {
            if (F32) {
              const uint64_t dbh = desc_sw128(st + ks * 32);   // 32 bytes of k per wgmma
              const uint64_t dbl = desc_sw128(st + kBTile + ks * 32);
              if (W) {
                if constexpr (FOLD) {   // B rows 128..135 (the folded columns) into acc_t
                  mma_tf32_n136(acc, acc_t, ahi[ks], dbh);
                  if (P3) {
                    mma_tf32_n136(acc, acc_t, alo[ks], dbh);
                    mma_tf32_n136(acc, acc_t, ahi[ks], dbl);
                  }
                } else {
                  mma_tf32_n128(acc, ahi[ks], dbh);
                  if (P3) {
                    mma_tf32_n128(acc, alo[ks], dbh);
                    mma_tf32_n128(acc, ahi[ks], dbl);
                  }
                }
              } else {
                mma_tf32_n64(acc, ahi[ks], dbh);
                if (P3) {
                  mma_tf32_n64(acc, alo[ks], dbh);
                  mma_tf32_n64(acc, ahi[ks], dbl);
                }
              }
            } else if (B_MN) {   // 16 k rows (2 KB) per wgmma
              const uint64_t db = desc_sw128_mn(st + ks * 2048, BK * 128);
              if (W) mma16_n128<T, 1>(acc, ahi[ks], db);
              else mma16_n64<T, 1>(acc, ahi[ks], db);
            } else {
              const uint64_t db = desc_sw128(st + ks * 32);
              if (W) mma16_n128<T, 0>(acc, ahi[ks], db);
              else mma16_n64<T, 0>(acc, ahi[ks], db);
            }
          }
          wgmma_commit();
        };
        auto by_width = [&](auto nk) {
          if (two_n) mmas(std::true_type{}, nk);
          else mmas(std::false_type{}, nk);
        };
        static_assert(NKS == 4, "k steps per block");
        if (ksteps == 4) by_width(std::integral_constant<int, 4>{});
        else if (ksteps == 3) by_width(std::integral_constant<int, 3>{});
        else if (ksteps == 2) by_width(std::integral_constant<int, 2>{});
        else by_width(std::integral_constant<int, 1>{});
        wgmma_wait<1>();   // retires group kb - 1; group kb stays in flight
      }
      if (PROD && kb > 0 && lane == 0) mbar_arrive(empty + (s == 0 ? stages - 1 : s - 1));
      if (++s == stages) {
        s = 0;
        fph ^= 1u;
      }
    };
    for (int kb = 0; kb < nkb; kb += 2) {   // unrolled by two: the fragment set is a constant
      kblock(kb, std::integral_constant<int, 0>{});
      if (kb + 1 < nkb) kblock(kb + 1, std::integral_constant<int, 1>{});
    }
    wgmma_wait<0>();
    if (PROD) {   // the tile's last stage; the producer is already filling the next tile's
      if (nkb > 0 && lane == 0) mbar_arrive(empty + (s == 0 ? stages - 1 : s - 1));
    } else {
      // every warpgroup is done with the stages: start the next tile's copies, then the epilogue
      mma_sync();
      if (tile + gridDim.x < total) prologue(tile + gridDim.x);
    }

    // accumulator element j of half h: row = 16 wq + lane / 4 + 8 ((j / 2) % 2),
    // column = 64 h + 8 (j / 4) + 2 (lane % 4) + j % 2
    if (STAGED) {
      // hand the raw accumulators to the epilogue warpgroup, once it has read the last tile
      if (tile != static_cast<int>(blockIdx.x)) bar_sync(kBarFree, kThreads + kEpiThreads);
      float* sp = cacc + (wg * 64 + wq * 16 + (lane >> 2)) * kStagingPitch + 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (h == 1 && !two_n) break;   // columns past GN: the epilogue does not use them
#pragma unroll
        for (int j = 0; j < 32; j += 2)
          *reinterpret_cast<float2*>(sp + 8 * ((j >> 1) & 1) * kStagingPitch + h * 64 + 8 * (j >> 2)) =
              make_float2(acc[h][j], acc[h][j + 1]);
      }
      bar_arrive(kBarFull, kThreads + kEpiThreads);
      continue;
    }
    // ------------------------------------------- epilogue on the accumulator registers ----
    const int rbase = m0 + wg * 64 + wq * 16 + (lane >> 2);
    float* Cf = static_cast<float*>(args.C) + static_cast<size_t>(z) * args.split_stride;
    H* Cb = static_cast<H*>(args.C);
    // paired stores need an even row pitch and a base aligned to two elements (C and every
    // split-K slice C + z * split_stride)
    const uintptr_t cbase = OUT16 ? reinterpret_cast<uintptr_t>(Cb) : reinterpret_cast<uintptr_t>(Cf);
    const bool vec2 = (args.ldc % 2) == 0 && (cbase & (OUT16 ? 3u : 7u)) == 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (h == 1 && !two_n) break;
#pragma unroll
      for (int c32 = 0; c32 < 2; ++c32) {   // 32-column chunks of this half
        const int chunk_col = n0 + h * 64 + c32 * 32;
        if (chunk_col >= args.GN) break;
        uint32_t bits_in[2] = {0u, 0u}, bits_out[2] = {0u, 0u};
        if (args.epi == EPI_MASK_BITS) {
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const int row = rbase + 8 * rr;
            if (row < args.GM)
              bits_in[rr] = __ldg(args.bits_in + static_cast<size_t>(chunk_col >> 5) * args.GM + row);
          }
        }
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          const int j = c32 * 16 + jj;
          const int rr = (j >> 1) & 1;
          const int cin = 8 * (j >> 2) + 2 * (lane & 3) + (j & 1);   // column within the half
          const int col = n0 + h * 64 + cin;
          const int row = rbase + 8 * rr;
          float x = acc[h][j];
          if (args.epi == EPI_BIAS_ACT) {
            x += col < args.GN ? __ldg(args.bias + col) : 0.f;
            if (args.act == TFR_ACT_RELU) x = fmaxf(x, 0.f);
          } else if (args.epi == EPI_MASK_POS) {
            if (args.act == TFR_ACT_RELU && row < args.GM && col < args.GN &&
                !(__ldg(args.aux + static_cast<size_t>(row) * args.ldc + col) > 0.f))
              x = 0.f;
          } else if (args.epi == EPI_MASK_BITS) {
            if (!((bits_in[rr] >> (cin & 31)) & 1u)) x = 0.f;
          }
          if (row >= args.GM || col >= args.GN) x = 0.f;
          acc[h][j] = x;   // column sums take the fp32 value, sign bits the stored one
          const float stored = OUT16 ? round16<H>(x) : x;
          bits_out[rr] |= (stored > 0.f ? 1u : 0u) << (cin & 31);
        }
        if (args.bits_out) {
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            uint32_t w = bits_out[rr];
            w |= __shfl_xor_sync(0xffffffffu, w, 1);
            w |= __shfl_xor_sync(0xffffffffu, w, 2);
            const int row = rbase + 8 * rr;
            if ((lane & 3) == 0 && row < args.GM)
              args.bits_out[static_cast<size_t>(chunk_col >> 5) * args.GM + row] = w;
          }
        }
      }
      // stores: one pair of adjacent columns per (row, 8-column block)
#pragma unroll
      for (int j = 0; j < 32; j += 2) {
        const int col = n0 + h * 64 + 8 * (j >> 2) + 2 * (lane & 3);
        const int row = rbase + 8 * ((j >> 1) & 1);
        if (row >= args.GM || col >= args.GN) continue;
        const float x0 = acc[h][j], x1 = acc[h][j + 1];
        const bool both = col + 1 < args.GN;
        if (OUT16) {
          H* p = Cb + static_cast<size_t>(row) * args.ldc + col;
          if (both && vec2) {
            *reinterpret_cast<uint32_t*>(p) = pack16<H>(x0, x1);
          } else {
            p[0] = to16<H>(x0);
            if (both) p[1] = to16<H>(x1);
          }
        } else if (args.store_transposed) {
          Cf[static_cast<size_t>(col) * args.ldc + row] = x0;
          if (both) Cf[static_cast<size_t>(col + 1) * args.ldc + row] = x1;
        } else {
          float* p = Cf + static_cast<size_t>(row) * args.ldc + col;
          if (both && vec2) {
            *reinterpret_cast<float2*>(p) = make_float2(x0, x1);
          } else {
            p[0] = x0;
            if (both) p[1] = x1;
          }
        }
      }
      if (args.colsum_cols) {
        // column sums of this warp's 16 rows: reduce over the 8 lanes that share lane % 4
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          float s0 = acc[h][j] + acc[h][j + 2], s1 = acc[h][j + 1] + acc[h][j + 3];
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            s0 += __shfl_xor_sync(0xffffffffu, s0, o);
            s1 += __shfl_xor_sync(0xffffffffu, s1, o);
          }
          const int col = n0 + h * 64 + 8 * (j >> 2) + 2 * (lane & 3);
          if (lane < 4 && col < args.colsum_cols) {
            float* a = cacc + warp * args.colsum_cols + col;
            a[0] += s0;
            if (col + 1 < args.colsum_cols) a[1] += s1;
          }
        }
      }
    }
    // the folded remainder (fp32 C): plain stores only, the host admits no other epilogue
    // for this layout.  Bounds, pairing and split-K slice as for the columns above.
    if (tail) {
      const int col = n0 + BN + 2 * (lane & 3);
      const bool both = col + 1 < args.GN;
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int row = rbase + 8 * rr;
        if (row >= args.GM || col >= args.GN) continue;
        const float x0 = acc_t[2 * rr], x1 = acc_t[2 * rr + 1];
        if (args.store_transposed) {
          Cf[static_cast<size_t>(col) * args.ldc + row] = x0;
          if (both) Cf[static_cast<size_t>(col + 1) * args.ldc + row] = x1;
        } else {
          float* p = Cf + static_cast<size_t>(row) * args.ldc + col;
          if (both && vec2) {
            *reinterpret_cast<float2*>(p) = make_float2(x0, x1);
          } else {
            p[0] = x0;
            if (both) p[1] = x1;
          }
        }
      }
    }
  }
  if (!STAGED && args.colsum_cols) {
    __syncwarp();
    float* dst = args.colsum + static_cast<size_t>(blockIdx.x * kWarps + warp) * args.colsum_stride;
    for (int c = lane; c < args.GN; c += 32) dst[c] = cacc[warp * args.colsum_cols + c];
  }
}

template <typename T, bool A_MN, bool B_MN, int PASSES, bool PRE_B, bool OUT16, bool FOLD>
int launch_grid(Args a, cudaStream_t st, int* ctas) {
  a.m_tiles = (a.GM + BM - 1) / BM;
  a.n_tiles = col_tiles(a.GN, FOLD);
  if (a.splits < 1) a.splits = 1;
  const int nkb_total = (a.GK + Elem<T>::BK - 1) / Elem<T>::BK;
  a.kb_per_split = (nkb_total + a.splits - 1) / a.splits;
  const int total = a.m_tiles * a.n_tiles * a.splits;
  const int sms = num_sms();
  const int grid = total < sms ? total : sms;
  if (ctas) *ctas = grid;
  const size_t smem = smem_bytes(PASSES, a.colsum_cols, !A_MN, FOLD, has_producer<T, A_MN, B_MN>());
  auto kern = gemm_kernel<T, A_MN, B_MN, PASSES, PRE_B, OUT16, FOLD>;
  TFR_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<grid, block_threads<T, A_MN, B_MN>(), smem, st>>>(a);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

// Launches the persistent grid; *ctas receives its size (column-sum slots = 8 x ctas).  A GN
// with a remainder to fold takes the folding kernel.  Every other GN takes the plain one, whose
// m64n128 MMAs and 128-row B tiles cost less per k block when no column is folded.
template <typename T, bool A_MN, bool B_MN, int PASSES, bool PRE_B, bool OUT16>
int launch(Args a, cudaStream_t st, int* ctas) {
  if constexpr (folds<T, A_MN, B_MN>())
    if (folded_cols(a.GN) > 0) return launch_grid<T, A_MN, B_MN, PASSES, PRE_B, OUT16, true>(a, st, ctas);
  return launch_grid<T, A_MN, B_MN, PASSES, PRE_B, OUT16, false>(a, st, ctas);
}

}  // namespace wg
}  // namespace tfr
