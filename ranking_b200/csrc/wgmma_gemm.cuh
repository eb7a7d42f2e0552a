// Hopper (sm_90a) warpgroup-MMA GEMM core shared by the TF32 / 3xTF32 engine (tc_gemm.cu) and
// the bf16 engine (tc_gemm_bf16.cu).
//
//   * a CTA owns a 128 x 128 output tile: two consumer warpgroups of 64 rows, each issuing
//     wgmma.mma_async m64n64 instructions (two per k step for the full 128 columns);
//   * operands go global -> registers -> shared memory, always written K-major with the
//     128-byte swizzle that the wgmma descriptors address.  TF32 wgmma only reads K-major
//     operands, so MN-major storage (the dW GEMMs) is transposed on that way, and the 3xTF32
//     hi / lo split of A (and of B when it is not pre-split) happens there too;
//   * the next k block is loaded into registers while the tensor cores work on the current
//     one (two shared-memory stages);
//   * the epilogue runs on the accumulator registers: bias / activation, ReLU masks (from an
//     fp32 array or from 1-bit sign words), ReLU sign words out, per-warp column sums,
//     row-major, transposed or split-K partial stores, fp32 or bf16 output.
// The grid is persistent (at most one CTA per SM), so the column-sum slots are bounded by
// 8 x the SM count.
#pragma once

#include <cuda_bf16.h>
#include <stdint.h>

#include "common.cuh"

namespace tfr {
namespace wg {

constexpr int BM = 128;          // rows of an output tile (two warpgroups of 64)
constexpr int BN = 128;          // columns of an output tile (two m64n64 instructions)
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kTileBytes = 128 * 128;   // one operand tile: 128 rows x 128 bytes of k
constexpr int kStages = 2;

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

#define TFR_WG_D32                                                                           \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, "  \
  "%19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define TFR_WG_OUT32(d)                                                                      \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),       \
      "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]),             \
      "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),          \
      "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),          \
      "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])

// D[64 x 64] += A[64 x 8] B[8 x 64], TF32 operands (fp32 bits; the low 13 are ignored)
__device__ __forceinline__ void mma_tf32(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " TFR_WG_D32
               ", %32, %33, 1, 1, 1;"
               : TFR_WG_OUT32(d)
               : "l"(da), "l"(db));
}
// D[64 x 64] += A[64 x 16] B[16 x 64], bf16 operands, both K-major
__device__ __forceinline__ void mma_bf16(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " TFR_WG_D32
               ", %32, %33, 1, 1, 1, 0, 0;"
               : TFR_WG_OUT32(d)
               : "l"(da), "l"(db));
}
#undef TFR_WG_D32
#undef TFR_WG_OUT32

// Element traits: a 16-byte chunk holds EPC elements; a 128-byte swizzle row holds BK of k.
template <typename T> struct Elem;
template <> struct Elem<float> { static constexpr int EPC = 4; static constexpr int BK = 32; };
template <> struct Elem<__nv_bfloat16> { static constexpr int EPC = 8; static constexpr int BK = 64; };

// One 16-byte chunk of an operand tile, zero past the matrix edge.  `p` points at the first
// element; `n` elements of the chunk lie inside the matrix (the chunk is aligned when n == EPC).
template <typename T>
__device__ __forceinline__ uint4 load_chunk(const T* p, int n) {
  constexpr int EPC = Elem<T>::EPC;
  if (n >= EPC) return __ldg(reinterpret_cast<const uint4*>(p));
  union { uint4 v; T e[EPC]; } u;
  u.v = make_uint4(0u, 0u, 0u, 0u);
  for (int i = 0; i < n; ++i) u.e[i] = p[i];
  return u.v;
}

// Byte offset of element (row, k) in a K-major 128B-swizzled tile (row pitch 128 B).
template <typename T>
__device__ __forceinline__ int swz(int row, int k) {
  const int byte = k * static_cast<int>(sizeof(T));
  return row * 128 + ((((byte >> 4) ^ row) & 7) << 4) + (byte & 15);
}

// Chunk i (0..3) of this thread in an MN-major tile ([k][rows], rows contiguous): a warp takes
// 8 consecutive row chunks (one 128-byte line per k row) of 4 consecutive k rows.  Spreading a
// warp over k keeps the scalar K-major stores of the transpose on 4 (TF32) / 8 (bf16) ways of
// bank conflict instead of 16: within one k row every lane's rows share their swizzle phase.
template <typename T>
__device__ __forceinline__ void mn_chunk(int i, int& k, int& r) {
  constexpr int EPC = Elem<T>::EPC, RG = 128 / EPC / 8;   // groups of 8 row chunks
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  k = (lane >> 3) + 4 * (warp / RG) + (Elem<T>::BK / 4) * i;
  r = ((lane & 7) + 8 * (warp % RG)) * EPC;
}

// Register-staged operand tile: 128 rows (m or n) x BK of k, 4 chunks per thread.
//   MN == false: stored [rows][k] (k contiguous); chunk c = row * 8 + k chunk
//   MN == true : stored [k][rows] (rows contiguous); chunks as in mn_chunk
template <typename T, bool MN>
struct Tile {
  uint4 v[4];
  __device__ __forceinline__ void load(const T* base, int ld, int r0, int rows, int k0, int ks) {
    constexpr int EPC = Elem<T>::EPC;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = threadIdx.x + i * kThreads;
      if (!MN) {
        const int r = c >> 3, k = (c & 7) * EPC;
        const int n = (r < rows) ? min(EPC, ks - (k0 + k)) : 0;
        v[i] = n > 0 ? load_chunk(base + static_cast<size_t>(r0 + r) * ld + k0 + k, n)
                     : make_uint4(0u, 0u, 0u, 0u);
      } else {
        int k, r;
        mn_chunk<T>(i, k, r);
        const int n = (k0 + k < ks) ? min(EPC, rows - r) : 0;
        v[i] = n > 0 ? load_chunk(base + static_cast<size_t>(k0 + k) * ld + r0 + r, n)
                     : make_uint4(0u, 0u, 0u, 0u);
      }
    }
  }
  // Write into the K-major swizzled tile(s).  SPLIT: hi = RN-TF32(x) to `hi`, x - hi to `lo`.
  template <bool SPLIT>
  __device__ __forceinline__ void store(unsigned char* hi, unsigned char* lo) const {
    constexpr int EPC = Elem<T>::EPC;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = threadIdx.x + i * kThreads;
      union { uint4 v; T e[EPC]; } u;
      u.v = v[i];
      if (!MN) {
        const int r = c >> 3, k = (c & 7) * EPC;
        const int off = swz<T>(r, k);
        if (SPLIT) {
          float4 h, l;
          const float4 x = *reinterpret_cast<const float4*>(&u.v);
          h.x = tf32_rn(x.x); h.y = tf32_rn(x.y); h.z = tf32_rn(x.z); h.w = tf32_rn(x.w);
          l.x = x.x - h.x; l.y = x.y - h.y; l.z = x.z - h.z; l.w = x.w - h.w;
          *reinterpret_cast<float4*>(hi + off) = h;
          *reinterpret_cast<float4*>(lo + off) = l;
        } else {
          *reinterpret_cast<uint4*>(hi + off) = u.v;
        }
      } else {
        int k, r;
        mn_chunk<T>(i, k, r);
#pragma unroll
        for (int e = 0; e < EPC; ++e) {
          const int off = swz<T>(r + e, k);
          if (SPLIT) {
            const float x = static_cast<float>(u.e[e]);
            const float h = tf32_rn(x);
            *reinterpret_cast<float*>(hi + off) = h;
            *reinterpret_cast<float*>(lo + off) = x - h;
          } else {
            *reinterpret_cast<T*>(hi + off) = u.e[e];
          }
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
// Shared memory: kStages x {A hi, A lo, B hi, B lo} tiles, then [8][colsum_cols] floats.
template <typename T, bool A_MN, bool B_MN, int PASSES, bool PRE_B, bool OUT_BF16>
__global__ void __launch_bounds__(kThreads, 1) gemm_kernel(const Args args) {
  constexpr int BK = Elem<T>::BK;
  constexpr int KSTEP = sizeof(T) == 4 ? 8 : 16;   // k of one wgmma
  constexpr bool P3 = PASSES == 3;
  constexpr int kCopies = P3 ? 2 : 1;
  constexpr int kStageBytes = 2 * kCopies * kTileBytes;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  float* cacc = reinterpret_cast<float*>(smem + kStages * kStageBytes);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2, wq = warp & 3;   // warpgroup, warp within it
  const T* A = static_cast<const T*>(args.A);
  const T* B = static_cast<const T*>(args.B);
  const T* Blo = static_cast<const T*>(args.B_lo);
  const int nkb_total = (args.GK + BK - 1) / BK;
  const int tiles_mn = args.m_tiles * args.n_tiles;
  const int total = tiles_mn * args.splits;

  for (int c = threadIdx.x; c < kWarps * args.colsum_cols; c += kThreads) cacc[c] = 0.f;

  auto sA = [&](int s, int lo) { return smem + s * kStageBytes + lo * kTileBytes; };
  auto sB = [&](int s, int lo) { return smem + s * kStageBytes + (kCopies + lo) * kTileBytes; };

  for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
    const int z = tile / tiles_mn;
    const int r = tile - z * tiles_mn;
    const int m0 = (r / args.n_tiles) * BM, n0 = (r % args.n_tiles) * BN;
    const int kb0 = z * args.kb_per_split;
    const int nkb = max(min(nkb_total, kb0 + args.kb_per_split) - kb0, 0);
    const bool two_n = n0 + 64 < args.GN;   // the second 64-column half holds live columns

    float acc[2][32];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[h][j] = 0.f;

    Tile<T, A_MN> ta;
    Tile<T, B_MN> tb, tbl;
    auto load = [&](int kb) {
      const int k0 = (kb0 + kb) * BK;
      ta.load(A, args.lda, m0, args.GM - m0, k0, args.GK);
      tb.load(B, args.ldb, n0, args.GN - n0, k0, args.GK);
      if (PRE_B) tbl.load(Blo, args.ldb, n0, args.GN - n0, k0, args.GK);
    };
    if (nkb > 0) load(0);
    for (int kb = 0; kb < nkb; ++kb) {
      const int s = kb % kStages;
      // the wgmma groups that read this stage (issued kStages k blocks ago) have retired in
      // every warpgroup once all threads pass this barrier
      __syncthreads();
      ta.template store<P3>(sA(s, 0), sA(s, 1));
      if (PRE_B) {
        tb.template store<false>(sB(s, 0), nullptr);
        tbl.template store<false>(sB(s, 1), nullptr);
      } else {
        tb.template store<P3>(sB(s, 0), sB(s, 1));
      }
      fence_proxy_async();   // generic-proxy stores -> visible to the tensor cores
      __syncthreads();
      if (kb + 1 < nkb) load(kb + 1);   // in flight while the tensor cores run
      // a K tail that is no multiple of BK is zero-filled: skip its all-zero k steps
      const int krem = args.GK - (kb0 + kb) * BK;
      const int ksteps = krem >= BK ? BK / KSTEP : (krem + KSTEP - 1) / KSTEP;
      const uint32_t a_hi = smem_u32(sA(s, 0)) + wg * 64 * 128, a_lo = a_hi + kTileBytes;
      const uint32_t b_hi = smem_u32(sB(s, 0)), b_lo = b_hi + kTileBytes;
      wgmma_fence();
#pragma unroll 1
      for (int ks = 0; ks < ksteps; ++ks) {
        const uint32_t kofs = ks * 32;   // 32 bytes of k per wgmma
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (h == 1 && !two_n) break;
          const uint64_t dah = desc_sw128(a_hi + kofs);
          const uint64_t dbh = desc_sw128(b_hi + h * 64 * 128 + kofs);
          if (sizeof(T) == 4) {
            mma_tf32(acc[h], dah, dbh);
            if (P3) {
              mma_tf32(acc[h], desc_sw128(a_lo + kofs), dbh);
              mma_tf32(acc[h], dah, desc_sw128(b_lo + h * 64 * 128 + kofs));
            }
          } else {
            mma_bf16(acc[h], dah, dbh);
          }
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
    }
    wgmma_wait<0>();

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

// Shared memory of one instantiation (dynamic, including the 1 KB alignment slack).
inline size_t smem_bytes(int passes, int colsum_cols) {
  return (size_t)kStages * 2 * (passes == 3 ? 2 : 1) * kTileBytes +
         (size_t)kWarps * colsum_cols * sizeof(float) + 1024;
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
