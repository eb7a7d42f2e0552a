// Hopper (sm_90a) warpgroup-MMA GEMM core shared by the TF32 / 3xTF32 engine (tc_gemm.cu) and
// the bf16 engine (tc_gemm_bf16.cu).
//
//   * a CTA owns a 128 x 128 output tile: two consumer warpgroups of 64 rows, each issuing one
//     wgmma.mma_async m64n128 per k step (m64n64 when the tile's live columns fit in 64);
//   * A comes from registers: each warpgroup loads its fragments from a plain (unswizzled,
//     padded) fp32 / bf16 tile in shared memory, at transposed addresses when A is MN-major.
//     The 3xTF32 hi / lo split of A happens there, in registers;
//   * operands that need no arithmetic (A in both layouts, K-major B and its pre-split lo part,
//     every bf16 B) are copied global -> shared by cp.async 16-byte copies into a ring of 3-4
//     stages; the 128-byte swizzle of B is applied in the destination address.  bf16 MN-major
//     B is read by the wgmma through the descriptor's transpose bit.  Only the MN-major TF32 B
//     of the dW GEMMs (TF32 wgmma reads K-major B only) is staged through registers, where it
//     is transposed and, for 3xTF32, split;
//   * the copies for the next tile start before the epilogue of the current one;
//   * the epilogue runs on the accumulator registers: bias / activation, ReLU masks (from an
//     fp32 array or from 1-bit sign words), ReLU sign words out, per-warp column sums,
//     row-major, transposed or split-K partial stores, fp32 or bf16 output.
// The grid is persistent (at most one CTA per SM), so the column-sum slots are bounded by
// 8 x the SM count.
#pragma once

#include <cuda_bf16.h>
#include <stdint.h>

#include <type_traits>

#include "common.cuh"

namespace tfr {
namespace wg {

constexpr int BM = 128;          // rows of an output tile (two warpgroups of 64)
constexpr int BN = 128;          // columns of an output tile (one m64n128 instruction)
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kTileBytes = 128 * 128;   // one swizzled B tile: 128 rows x 128 bytes of k
// A tile: 128 rows x 128 bytes of k.  K-major rows are padded to 144 B, MN-major k rows
// (512 B of m) to 544 B (fp32, 32 rows) / 272 B (bf16, 64 rows): either way the fragment
// loads of a warp hit 32 different banks.
constexpr int kAPitchK = 144;
constexpr int kAPitchMN = 4 * (128 + 8);   // bytes per k row (fp32); bf16 uses half of it
constexpr int kATileBytes = 128 * kAPitchK;
constexpr int kMaxStages = 4;
constexpr int kSmemLimit = 227 * 1024;  // dynamic shared memory of one CTA on sm_90

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

// Bytes of one pipeline stage: the B tile (plus its lo tile for 3xTF32), then the A tile.
__host__ __device__ constexpr int stage_bytes(int passes) {
  return (passes == 3 ? 2 : 1) * kTileBytes + kATileBytes;
}
// Stages that fit beside the [8][colsum_cols] column-sum accumulator and the 1 KB alignment
// slack; at most kMaxStages.  The one place that sizes the shared memory of a launch.
__host__ __device__ constexpr int num_stages(int passes, int colsum_cols) {
  return (kSmemLimit - 1024 - kWarps * colsum_cols * 4) / stage_bytes(passes) < kMaxStages
             ? (kSmemLimit - 1024 - kWarps * colsum_cols * 4) / stage_bytes(passes)
             : kMaxStages;
}
static_assert(num_stages(3, 1024) >= 3, "3xTF32 needs three stages beside a 1024-column colsum");
inline size_t smem_bytes(int passes, int colsum_cols) {
  return (size_t)num_stages(passes, colsum_cols) * stage_bytes(passes) +
         (size_t)kWarps * colsum_cols * sizeof(float) + 1024;
}

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
// bf16 (k = 16): two bf16 per register.  TRANS_B: B is MN-major in shared memory.
template <int TRANS_B>
__device__ __forceinline__ void mma_bf16_n64(float (&d)[2][32], const uint32_t (&a)[4], uint64_t db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " TFR_WG_D32
               ", {%32, %33, %34, %35}, %36, 1, 1, 1, %37;"
               : TFR_WG_OUT32(d[0])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "n"(TRANS_B));
}
template <int TRANS_B>
__device__ __forceinline__ void mma_bf16_n128(float (&d)[2][32], const uint32_t (&a)[4], uint64_t db) {
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

// Byte offset of 16-byte chunk `kc` of row `row` in a K-major 128B-swizzled tile.
__device__ __forceinline__ int swz_chunk(int row, int kc) { return row * 128 + (((kc ^ row) & 7) << 4); }

// The register-staged operand: an MN-major fp32 B tile ([k][n], n contiguous) of 128 columns
// x 32 k, transposed into the K-major swizzled tile(s) and, for 3xTF32, split into hi / lo.
// A warp takes 8 consecutive column chunks (one 128-byte line per k row) of 4 consecutive k
// rows: within one k row every lane's columns share their swizzle phase, which keeps the
// scalar K-major stores on 4 ways of bank conflict instead of 16.
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
      const float e[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int off = swz_chunk(r + j, k >> 2) + (k & 3) * 4;
        if (SPLIT) {
          const float h = tf32_rn(e[j]);
          *reinterpret_cast<float*>(hi + off) = h;
          *reinterpret_cast<float*>(lo + off) = e[j] - h;
        } else {
          *reinterpret_cast<float*>(hi + off) = e[j];
        }
      }
    }
  }
};

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// PASSES: 1 (one product) or 3 (3xTF32: Ahi Bhi + Alo Bhi + Ahi Blo; float only).
// PRE_B: B comes pre-split (B = hi parts, B_lo = lo parts).  OUT_BF16: C is bf16 (row-major).
// Shared memory: num_stages x {B hi, [B lo,] A}, then [8][colsum_cols] floats.
template <typename T, bool A_MN, bool B_MN, int PASSES, bool PRE_B, bool OUT_BF16>
__global__ void __launch_bounds__(kThreads, 1) gemm_kernel(const Args args) {
  constexpr bool F32 = sizeof(T) == 4;
  constexpr int EPC = Elem<T>::EPC;
  constexpr int BK = Elem<T>::BK;
  constexpr int KSTEP = F32 ? 8 : 16;   // k of one wgmma
  constexpr int NKS = BK / KSTEP;
  constexpr bool P3 = PASSES == 3;
  constexpr bool REG_B = F32 && B_MN;   // TF32 MN-major B: transposed through registers
  constexpr int kStage = stage_bytes(PASSES);
  constexpr int kAOff = (P3 ? 2 : 1) * kTileBytes;
  constexpr int kAPitch = A_MN ? kAPitchMN * static_cast<int>(sizeof(T)) / 4 : kAPitchK;
  static_assert(!P3 || F32, "3xTF32 is float only");
  static_assert(!PRE_B || P3, "pre-split B is 3xTF32");
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int stages = num_stages(PASSES, args.colsum_cols);
  float* cacc = reinterpret_cast<float*>(smem + stages * kStage);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2, wq = warp & 3;   // warpgroup, warp within it
  const T* A = static_cast<const T*>(args.A);
  const T* B = static_cast<const T*>(args.B);
  const T* Blo = static_cast<const T*>(args.B_lo);
  const int nkb_total = (args.GK + BK - 1) / BK;
  const int tiles_mn = args.m_tiles * args.n_tiles;
  const int total = tiles_mn * args.splits;
  const uint32_t smem_base = smem_u32(smem);

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
        if (PRE_B) cp_async16(st + kTileBytes + swz_chunk(r, kc), Blo + off, n * static_cast<int>(sizeof(T)));
      }
    } else if (!F32) {   // bf16 [2 atoms of 64 n][64 k rows][8 chunks of n], swizzled
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

  // cp.async groups: a tile's prologue commits stages - 1 groups (blocks 0 .. stages - 2),
  // every k block one more (block kb + stages - 1), empty ones included, so that block kb's
  // group is complete once at most stages - 2 younger groups are pending.
  BTileMN tb, tbl;
  auto load_b = [&](int n0, int kb) {
    tb.load(reinterpret_cast<const float*>(B), args.ldb, n0, args.GN - n0, kb * BK, args.GK);
    if (PRE_B) tbl.load(reinterpret_cast<const float*>(Blo), args.ldb, n0, args.GN - n0, kb * BK, args.GK);
  };
  auto prologue = [&](int tile) {
    const int z = tile / tiles_mn;
    const int r = tile - z * tiles_mn;
    const int m0 = (r / args.n_tiles) * BM, n0 = (r % args.n_tiles) * BN;
    const int kb0 = z * args.kb_per_split;
    const int nkb = max(min(nkb_total, kb0 + args.kb_per_split) - kb0, 0);
    for (int p = 0; p < stages - 1; ++p) {
      if (p < nkb) copy_block(m0, n0, kb0, p, p);
      cp_async_commit();
    }
    if (REG_B && nkb > 0) load_b(n0, kb0);
  };

  if (blockIdx.x < total) prologue(blockIdx.x);
  for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
    const int z = tile / tiles_mn;
    const int r = tile - z * tiles_mn;
    const int m0 = (r / args.n_tiles) * BM, n0 = (r % args.n_tiles) * BN;
    const int kb0 = z * args.kb_per_split;
    const int nkb = max(min(nkb_total, kb0 + args.kb_per_split) - kb0, 0);
    const bool two_n = n0 + 64 < args.GN;           // the second 64 columns hold live columns

    float acc[2][32];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[h][j] = 0.f;

    int s = 0;
    for (int kb = 0; kb < nkb; ++kb) {
      const uint32_t st = smem_base + s * kStage;
      // stage s was last read by the MMAs of block kb - stages, retired before the barrier
      // of block kb - stages + 1
      if (REG_B) {
        unsigned char* sb = smem + s * kStage;
        if (PRE_B) {
          tb.template store<false>(sb, nullptr);
          tbl.template store<false>(sb + kTileBytes, nullptr);
        } else {
          tb.template store<P3>(sb, sb + kTileBytes);
        }
      }
      if (stages == 4) cp_async_wait<2>(); else cp_async_wait<1>();
      if (P3 && !B_MN && !PRE_B) {   // K-major B split on the fly: each thread its own chunks
        unsigned char* sb = smem + s * kStage;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int c = threadIdx.x + i * kThreads;
          const int off = swz_chunk(c >> 3, c & 7);
          const float4 x = *reinterpret_cast<const float4*>(sb + off);
          const float4 h = make_float4(tf32_rn(x.x), tf32_rn(x.y), tf32_rn(x.z), tf32_rn(x.w));
          *reinterpret_cast<float4*>(sb + off) = h;
          *reinterpret_cast<float4*>(sb + kTileBytes + off) =
              make_float4(x.x - h.x, x.y - h.y, x.z - h.z, x.w - h.w);
        }
      }
      fence_proxy_async();   // cp.async and st.shared writes -> visible to the tensor cores
      __syncthreads();
      // refill the stage of block kb - 1, whose MMAs every warpgroup retired before the barrier
      {
        const int nb = kb + stages - 1;
        if (nb < nkb) copy_block(m0, n0, kb0, nb, nb % stages);
        cp_async_commit();
      }
      if (REG_B && kb + 1 < nkb) load_b(n0, kb0 + kb + 1);   // in flight while the tensor cores run
      {
        // a K tail that is no multiple of BK is zero-filled: skip its all-zero k steps
        const int krem = args.GK - (kb0 + kb) * BK;
        const int ksteps = krem >= BK ? NKS : (krem + KSTEP - 1) / KSTEP;
        // A fragments of every k step (m64 x k, per warp 16 rows): register i holds row
        // g + 8 (i % 2), k t + 4 (i / 2) (TF32) / k pair 2t + 8 (i / 2) (bf16)
        const int g = lane >> 2, t = lane & 3;
        const int row = wg * 64 + wq * 16 + g;
        const unsigned char* sa = smem + s * kStage + kAOff;
        uint32_t ahi[NKS][4], alo[NKS][4];
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
              const uint64_t dbl = desc_sw128(st + kTileBytes + ks * 32);
              if (W) {
                mma_tf32_n128(acc, ahi[ks], dbh);
                if (P3) {
                  mma_tf32_n128(acc, alo[ks], dbh);
                  mma_tf32_n128(acc, ahi[ks], dbl);
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
              if (W) mma_bf16_n128<1>(acc, ahi[ks], db);
              else mma_bf16_n64<1>(acc, ahi[ks], db);
            } else {
              const uint64_t db = desc_sw128(st + ks * 32);
              if (W) mma_bf16_n128<0>(acc, ahi[ks], db);
              else mma_bf16_n64<0>(acc, ahi[ks], db);
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
        wgmma_wait<0>();
      }
      s = s + 1 == stages ? 0 : s + 1;
    }
    // every warpgroup is done with the stages: start the next tile's copies, then the epilogue
    __syncthreads();
    if (tile + gridDim.x < total) prologue(tile + gridDim.x);

    // ---------------------------------------------------------------- epilogue ----
    // accumulator element j of half h: row = 16 wq + lane / 4 + 8 ((j / 2) % 2),
    // column = 64 h + 8 (j / 4) + 2 (lane % 4) + j % 2
    const int rbase = m0 + wg * 64 + wq * 16 + (lane >> 2);
    float* Cf = static_cast<float*>(args.C) + static_cast<size_t>(z) * args.split_stride;
    __nv_bfloat16* Cb = static_cast<__nv_bfloat16*>(args.C);
    // paired stores need an even row pitch and a base aligned to two elements (C and every
    // split-K slice C + z * split_stride)
    const uintptr_t cbase = OUT_BF16 ? reinterpret_cast<uintptr_t>(Cb) : reinterpret_cast<uintptr_t>(Cf);
    const bool vec2 = (args.ldc % 2) == 0 && (cbase & (OUT_BF16 ? 3u : 7u)) == 0;
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
          const float stored = OUT_BF16 ? __bfloat162float(__float2bfloat16_rn(x)) : x;
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
        if (OUT_BF16) {
          __nv_bfloat16* p = Cb + static_cast<size_t>(row) * args.ldc + col;
          if (both && vec2) {
            *reinterpret_cast<uint32_t*>(p) = pack_bf16(x0, x1);
          } else {
            p[0] = __float2bfloat16_rn(x0);
            if (both) p[1] = __float2bfloat16_rn(x1);
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
  }
  if (args.colsum_cols) {
    __syncwarp();
    float* dst = args.colsum + static_cast<size_t>(blockIdx.x * kWarps + warp) * args.colsum_stride;
    for (int c = lane; c < args.GN; c += 32) dst[c] = cacc[warp * args.colsum_cols + c];
  }
}

// Launches the persistent grid; *ctas receives its size (column-sum slots = 8 x ctas).
template <typename T, bool A_MN, bool B_MN, int PASSES, bool PRE_B, bool OUT_BF16>
int launch(Args a, cudaStream_t st, int* ctas) {
  a.m_tiles = (a.GM + BM - 1) / BM;
  a.n_tiles = (a.GN + BN - 1) / BN;
  if (a.splits < 1) a.splits = 1;
  const int nkb_total = (a.GK + Elem<T>::BK - 1) / Elem<T>::BK;
  a.kb_per_split = (nkb_total + a.splits - 1) / a.splits;
  const int total = a.m_tiles * a.n_tiles * a.splits;
  const int sms = num_sms();
  const int grid = total < sms ? total : sms;
  if (ctas) *ctas = grid;
  const size_t smem = smem_bytes(PASSES, a.colsum_cols);
  auto kern = gemm_kernel<T, A_MN, B_MN, PASSES, PRE_B, OUT_BF16>;
  TFR_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<grid, kThreads, smem, st>>>(a);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

}  // namespace wg
}  // namespace tfr
