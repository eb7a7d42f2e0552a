// 16-bit tensor-core attention core (TFR-BERT's TFR_PREC_BF16 and TFR_PREC_FP16 modes): the
// contractions of din.cu's SIMT kernels on wgmma m64nNk16 (bf16 or fp16 operands, fp32
// accumulate); softmax, masking and dropout in fp32 registers, as there.  qkv, O, dO and dqkv
// are 16-bit (T: bf16 or fp16, the same code on either); lse and dsum fp32.  The text below says
// bf16 for T.
//
// CTA and grid as din_tc.cu: one warpgroup owns 64 rows of one (list, head), the other side
// streams through shared memory in tiles of 64 items, head sizes padded to the buckets 16 / 32 /
// 64 / 128 (HP).  What bf16 changes:
//   * one shared copy of each operand.  Q, K, V and dO are copied as stored (item rows of HP
//     bf16, 128-byte swizzled, 64 columns per 8 KB block).  Read K-major (k = head dimension)
//     that is the A or B of S = Q K^T, dP = dO V^T and their transposes; the same bytes read
//     MN-major through the wgmma transpose bit (k = item, n = head dimension, 64 columns per
//     swizzle atom) are the B of O = P~ V, dQ = dS K, dV = P~^T dO and dK = dS^T Q.  Nothing is
//     transposed through registers;
//   * the first product's accumulators are the second product's A fragments as they lie: lane
//     t holds columns 2t, 2t + 1 (and + 8) of each group of 16, which is the bf16 A fragment
//     of that k step (frag_of_acc), so there is no perm_k reordering;
//   * P~ is rounded to bf16 after normalisation: the forward finds each row's max and sum in a
//     first pass over the key tiles (skipped when one tile holds every key: the scores are
//     still in registers), then P = exp(s - max) / sum, dropout, rounding and P~ V.  So the
//     rounded value is bf16(P~), the quantity the header's contract names, and the backward's
//     recomputed P is the forward's P.
// The backward keeps the two passes of the other cores (queries, then keys) and no atomics:
// two identical calls give identical bits.  D_i = dO_i . O_i over the stored bf16 values.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "common.cuh"
#include "din.cuh"
#include "wgmma_gemm.cuh"

namespace tfr {
namespace {

using wg::cp_async16;
using wg::desc_sw128;
using wg::desc_sw128_mn;
using wg::fence_proxy_async;
using wg::smem_u32;
using wg::swz_chunk;
using wg::wgmma_commit;
using wg::wgmma_fence;
using wg::wgmma_wait;

using bf16 = __nv_bfloat16;

constexpr int kT = 64;            // rows a CTA owns; items per streamed tile
constexpr int kThreads = 128;     // one warpgroup
constexpr int kBlock = kT * 128;  // 64 item rows x 128 B: 64 head columns of a tile

__host__ __device__ constexpr int bucket(int h) {
  return h <= 16 ? 16 : h <= 32 ? 32 : h <= 64 ? 64 : 128;
}
#define TFR_DIN16_DISPATCH(h, fn, T, ...)                                                   \
  (bucket(h) == 16 ? fn<16, T>(__VA_ARGS__) : bucket(h) == 32 ? fn<32, T>(__VA_ARGS__)        \
   : bucket(h) == 64 ? fn<64, T>(__VA_ARGS__) : fn<128, T>(__VA_ARGS__))

__host__ __device__ constexpr int tile_bytes(int hp) { return (hp < 64 ? 1 : hp / 64) * kBlock; }

// Items [0, kT) x head columns [0, HP) of src (row pitch ld): item r < n, column c < h; zero
// elsewhere.  cp.async; the caller commits and waits.  h % 8 == 0, so a 16-byte chunk is
// either wholly inside the head or wholly past it.
template <int HP, typename T>
__device__ __forceinline__ void load_tile(unsigned char* dst, const T* src, int ld, int n,
                                          int h) {
  constexpr int CPR = HP / 8;   // 16-byte chunks per item row
  for (int e = threadIdx.x; e < kT * CPR; e += kThreads) {
    const int r = e / CPR, kc = e % CPR;
    const bool ok = r < n && kc * 8 < h;
    cp_async16(smem_u32(dst + (kc >> 3) * kBlock + swz_chunk(r, kc & 7)),
               ok ? src + (size_t)r * ld + kc * 8 : src, ok ? 16 : 0);
  }
}

// K-major view, k step ks (16 head columns).
__device__ __forceinline__ uint64_t kdesc(const unsigned char* tile, int ks) {
  return desc_sw128(smem_u32(tile + (ks >> 2) * kBlock + (ks & 3) * 32));
}
// MN-major view, k step ks (16 items).
__device__ __forceinline__ uint64_t ndesc(const unsigned char* tile, int ks) {
  return desc_sw128_mn(smem_u32(tile + ks * 2048), kBlock);
}

// Accumulator element j of an m64nN product: row 16 warp + lane / 4 + 8 acc_half(j), column
// acc_col(j) (lane % 4 = t).
__device__ __forceinline__ int acc_half(int j) { return (j >> 1) & 1; }
__device__ __forceinline__ int acc_col(int j, int t) { return 8 * (j >> 2) + 2 * t + (j & 1); }

// Two elements of T, rounded to nearest even; the pair type of T.
template <typename T>
using pair_t = std::conditional_t<std::is_same_v<T, __half>, __half2, __nv_bfloat162>;
template <typename T>
__device__ __forceinline__ pair_t<T> pair_rn(float lo, float hi) {
  if constexpr (std::is_same_v<T, __half>) return __floats2half2_rn(lo, hi);
  else return __floats2bfloat162_rn(lo, hi);
}
template <typename T>
__device__ __forceinline__ uint32_t pack16(float lo, float hi) {
  const pair_t<T> v = pair_rn<T>(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&v);
}
template <typename T>
__device__ __forceinline__ float2 unpack16(const pair_t<T>& v) {
  if constexpr (std::is_same_v<T, __half>) return __half22float2(v);
  else return __bfloat1622float2(v);
}

// A fragment of k step ks (items 16 ks .. 16 ks + 15) from an m64n64 accumulator, rounded to
// nearest T.
template <typename T>
__device__ __forceinline__ void frag_of_acc(const float (&acc)[32], int ks, uint32_t (&a)[4]) {
  a[0] = pack16<T>(acc[8 * ks], acc[8 * ks + 1]);
  a[1] = pack16<T>(acc[8 * ks + 2], acc[8 * ks + 3]);
  a[2] = pack16<T>(acc[8 * ks + 4], acc[8 * ks + 5]);
  a[3] = pack16<T>(acc[8 * ks + 6], acc[8 * ks + 7]);
}

#define TFR_F8(d, o)                                                                         \
  "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), \
      "+f"(d[o + 6]), "+f"(d[o + 7])
#define TFR_F32(d, o) TFR_F8(d, o), TFR_F8(d, o + 8), TFR_F8(d, o + 16), TFR_F8(d, o + 24)
#define TFR_R32                                                                              \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, "  \
  "%19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"

// The products, with TY the wgmma operand type ("bf16" or "f16") of T.
// D[64 x 64] += A B, both K-major in shared memory.
#define TFR_MMA_SS64(TY)                                                                     \
  asm volatile("wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " " TFR_R32           \
               ", %32, %33, 1, 1, 1, 0, 0;"                                                  \
               : TFR_F32(d, 0)                                                               \
               : "l"(da), "l"(db))
template <typename T>
__device__ __forceinline__ void mma_ss64(float (&d)[32], uint64_t da, uint64_t db) {
  if constexpr (std::is_same_v<T, __half>) TFR_MMA_SS64("f16");
  else TFR_MMA_SS64("bf16");
}
// D[64 x N] += A B, A from registers, B MN-major (transpose bit).
#define TFR_MMA_RS(TY)                                                                       \
  if constexpr (N == 16) {                                                                   \
    asm volatile("wgmma.mma_async.sync.aligned.m64n16k16.f32." TY "." TY " "                 \
                 "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, 1, 1, 1, 1;"    \
                 : TFR_F8(d, 0)                                                              \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));                     \
  } else if constexpr (N == 32) {                                                            \
    asm volatile("wgmma.mma_async.sync.aligned.m64n32k16.f32." TY "." TY " "                 \
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "  \
                 "{%16, %17, %18, %19}, %20, 1, 1, 1, 1;"                                    \
                 : TFR_F8(d, 0), TFR_F8(d, 8)                                                \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));                     \
  } else if constexpr (N == 64) {                                                            \
    asm volatile("wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " " TFR_R32         \
                 ", {%32, %33, %34, %35}, %36, 1, 1, 1, 1;"                                  \
                 : TFR_F32(d, 0)                                                             \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));                     \
  } else {                                                                                   \
    static_assert(N == 128, "n width");                                                      \
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " "                \
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, " \
                 "%17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, " \
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, " \
                 "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, " \
                 "%62, %63}, {%64, %65, %66, %67}, %68, 1, 1, 1, 1;"                         \
                 : TFR_F32(d, 0), TFR_F32(d, 32)                                             \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));                     \
  }
template <int N, typename T>
__device__ __forceinline__ void mma_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t db) {
  if constexpr (std::is_same_v<T, __half>) {
    TFR_MMA_RS("f16")
  } else {
    TFR_MMA_RS("bf16")
  }
}
#undef TFR_MMA_SS64
#undef TFR_MMA_RS
#undef TFR_F8
#undef TFR_F32
#undef TFR_R32

// S (or S^T) = A B^T over the padded head dimension.
template <int HP, typename T>
__device__ __forceinline__ void mma_heads(float (&d)[32], const unsigned char* a,
                                          const unsigned char* b) {
#pragma unroll
  for (int ks = 0; ks < HP / 16; ++ks) mma_ss64<T>(d, kdesc(a, ks), kdesc(b, ks));
}
// D += A B over the kT items of a tile: A from the accumulator `p`, B a tile read MN-major.
template <int HP, typename T>
__device__ __forceinline__ void mma_items(float (&d)[HP / 2], const float (&p)[32],
                                          const unsigned char* b) {
#pragma unroll
  for (int ks = 0; ks < kT / 16; ++ks) {
    uint32_t a[4];
    frag_of_acc<T>(p, ks, a);
    mma_rs<HP, T>(d, a, ndesc(b, ks));
  }
}

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

__device__ __forceinline__ unsigned char* align1024(unsigned char* p) {
  return reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~(uintptr_t)1023);
}

// Writes this thread's accumulator elements of rows < n (relative to `base`, row pitch ld),
// columns < h, times `mul`, rounded to T.
template <int HP, typename T>
__device__ __forceinline__ void store_rows(const float (&acc)[HP / 2], T* base, int ld, int n,
                                           int h, float mul) {
  const int lane = threadIdx.x & 31, row = 16 * (threadIdx.x >> 5) + (lane >> 2);
#pragma unroll
  for (int j = 0; j < HP / 2; j += 2) {
    const int r = row + 8 * acc_half(j), c = acc_col(j, lane & 3);
    if (r < n && c < h)   // c even and h % 8 == 0: c + 1 < h too
      *reinterpret_cast<pair_t<T>*>(base + (size_t)r * ld + c) =
          pair_rn<T>(acc[j] * mul, acc[j + 1] * mul);
  }
}

// Scaled, masked scores of one tile in place (-inf past the list's nk items).
__device__ __forceinline__ void mask_scores(float (&s)[32], const uint8_t* vm, int nk, int t,
                                            float scale) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int c = acc_col(j, t);
    s[j] = c < nk ? (vm[c] ? s[j] * scale : s[j] * scale + kMaskAdder) : -INFINITY;
  }
}

// Forward: grid B H ceil(N / 64), CTA = 64 query rows of one (list, head).
template <int HP, typename T>
__global__ void __launch_bounds__(kThreads)
attn_fwd16_kernel(const T* __restrict__ qkv, const uint8_t* __restrict__ lmask, int N,
                     int H, int h, float scale, float drop, unsigned long long dseed,
                     T* __restrict__ O, float* __restrict__ lse) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* Qs = align1024(smem_raw);
  unsigned char* Ks = Qs + tile_bytes(HP);
  unsigned char* Vs = Ks + tile_bytes(HP);
  uint8_t* vm = Vs + tile_bytes(HP);
  const int tiles = (N + kT - 1) / kT;
  const int bh = blockIdx.x / tiles, i0 = (blockIdx.x % tiles) * kT;
  const int hd = bh % H, HH = H * h, ld = 3 * HH;
  const size_t row0 = (size_t)(bh / H) * N;
  const T* Qg = qkv + row0 * ld + hd * h;
  const T* Kg = Qg + HH;
  const T* Vg = Qg + 2 * HH;
  const int lane = threadIdx.x & 31, t = lane & 3;
  const int row = 16 * (threadIdx.x >> 5) + (lane >> 2);   // + 8 * half
  const float kscale = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  const unsigned long long ebase = (unsigned long long)bh * N;
  const int n = min(kT, N - i0);
  load_tile<HP, T>(Qs, Qg + (size_t)i0 * ld, ld, n, h);
  // Streams key tile j0 (and its values when `with_v`) into shared memory, then S.
  auto scores = [&](int j0, bool with_v, float (&s)[32]) {
    const int nk = min(kT, N - j0);
    __syncthreads();   // every warpgroup product of the previous tile has completed
    load_tile<HP, T>(Ks, Kg + (size_t)j0 * ld, ld, nk, h);
    if (with_v) load_tile<HP, T>(Vs, Vg + (size_t)j0 * ld, ld, nk, h);
    wg::cp_async_commit();
    if (threadIdx.x < kT)
      vm[threadIdx.x] = threadIdx.x < nk && (lmask == nullptr || lmask[row0 + j0 + threadIdx.x]);
    wg::cp_async_wait<0>();
    fence_proxy_async();
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 32; ++j) s[j] = 0.f;
    wgmma_fence();
    mma_heads<HP, T>(s, Qs, Ks);
    wgmma_commit();
    wgmma_wait<0>();
    mask_scores(s, vm, nk, t, scale);
  };
  // Row max and sum over every key: online over the tiles, or from the one tile's scores.
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  auto absorb = [&](const float (&s)[32]) {
    float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 32; ++j) tmax[acc_half(j)] = fmaxf(tmax[acc_half(j)], s[j]);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float mn = fmaxf(m[r], quad_max(tmax[r]));
      l[r] *= expf(m[r] - mn);
      m[r] = mn;
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) l[acc_half(j)] += expf(s[j] - m[acc_half(j)]);
  };
  float s[32];
  if (tiles > 1)
    for (int j0 = 0; j0 < N; j0 += kT) {
      scores(j0, false, s);
      absorb(s);
    }
  float inv[2];
  float o[HP / 2];
#pragma unroll
  for (int j = 0; j < HP / 2; ++j) o[j] = 0.f;
  for (int j0 = 0; j0 < N; j0 += kT) {
    const int nk = min(kT, N - j0);
    scores(j0, true, s);
    if (j0 == 0) {
      if (tiles == 1) absorb(s);
#pragma unroll
      for (int r = 0; r < 2; ++r) inv[r] = 1.f / quad_sum(l[r]);
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int r = acc_half(j), c = acc_col(j, t);
      float pr = expf(s[j] - m[r]) * inv[r];   // 0 past the list
      if (drop > 0.f && c < nk)
        pr = din_uniform(dseed, (ebase + i0 + row + 8 * r) * N + j0 + c) >= drop ? pr * kscale
                                                                                : 0.f;
      s[j] = pr;
    }
    wgmma_fence();
    mma_items<HP, T>(o, s, Vs);
    wgmma_commit();
    wgmma_wait<0>();
  }
  store_rows<HP, T>(o, O + (row0 + i0) * HH + hd * h, HH, n, h, 1.f);
  if (t == 0) {   // max and 1 / sum: exact for a list with no valid item (all -1e9)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int i = row + 8 * r;
      if (i < n) {
        lse[((row0 + i0 + i) * H + hd) * 2] = m[r];
        lse[((row0 + i0 + i) * H + hd) * 2 + 1] = inv[r];
      }
    }
  }
}

// Backward, query-owning pass: D_i = rowsum(dO_i O_i); S = Q K^T and dP = dO V^T per key tile;
// dS = bf16(P (dP keep / (1 - rate) - D_i)); dQ = scale dS K.
template <int HP, typename T>
__global__ void __launch_bounds__(kThreads)
attn_bwd_dq16_kernel(const T* __restrict__ qkv, const uint8_t* __restrict__ lmask, int N,
                        int H, int h, float scale, float drop, unsigned long long dseed,
                        const T* __restrict__ O, const float* __restrict__ lse,
                        const T* __restrict__ dO, float* __restrict__ dsum,
                        T* __restrict__ dqkv) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* Qs = align1024(smem_raw);
  unsigned char* Gs = Qs + tile_bytes(HP);
  unsigned char* Ks = Gs + tile_bytes(HP);
  unsigned char* Vs = Ks + tile_bytes(HP);
  float* Dsm = reinterpret_cast<float*>(Vs + tile_bytes(HP));
  uint8_t* vm = reinterpret_cast<uint8_t*>(Dsm + kT);
  const int tiles = (N + kT - 1) / kT;
  const int bh = blockIdx.x / tiles, i0 = (blockIdx.x % tiles) * kT;
  const int hd = bh % H, HH = H * h, ld = 3 * HH;
  const size_t row0 = (size_t)(bh / H) * N;
  const T* Qg = qkv + row0 * ld + hd * h;
  const T* Kg = Qg + HH;
  const T* Vg = Qg + 2 * HH;
  const int lane = threadIdx.x & 31, t = lane & 3;
  const int row = 16 * (threadIdx.x >> 5) + (lane >> 2);
  const float kscale = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  const unsigned long long ebase = (unsigned long long)bh * N;
  const int n = min(kT, N - i0);
  const T* Gg = dO + (row0 + i0) * HH + hd * h;
  load_tile<HP, T>(Qs, Qg + (size_t)i0 * ld, ld, n, h);
  load_tile<HP, T>(Gs, Gg, HH, n, h);
  wg::cp_async_commit();
  {   // D_i: two threads per row, 8 columns of every 16 each
    const int r = threadIdx.x >> 1;
    float d = 0.f;
    if (r < n)
      for (int c = (threadIdx.x & 1) * 8; c < h; c += 16) {
        const uint4 gv = *reinterpret_cast<const uint4*>(Gg + (size_t)r * HH + c);
        const uint4 xv = *reinterpret_cast<const uint4*>(O + (row0 + i0 + r) * HH + hd * h + c);
        const pair_t<T>* g2 = reinterpret_cast<const pair_t<T>*>(&gv);
        const pair_t<T>* x2 = reinterpret_cast<const pair_t<T>*>(&xv);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 g = unpack16<T>(g2[q]), x = unpack16<T>(x2[q]);
          d += g.x * x.x + g.y * x.y;
        }
      }
    d += __shfl_xor_sync(0xffffffffu, d, 1);
    if ((threadIdx.x & 1) == 0) {
      Dsm[r] = d;
      if (r < n) dsum[(row0 + i0 + r) * H + hd] = d;
    }
  }
  float mi[2], il[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = row + 8 * r;
    mi[r] = i < n ? lse[((row0 + i0 + i) * H + hd) * 2] : 0.f;
    il[r] = i < n ? lse[((row0 + i0 + i) * H + hd) * 2 + 1] : 0.f;
  }
  float dq[HP / 2];
#pragma unroll
  for (int j = 0; j < HP / 2; ++j) dq[j] = 0.f;
  for (int j0 = 0; j0 < N; j0 += kT) {
    const int nk = min(kT, N - j0);
    __syncthreads();
    load_tile<HP, T>(Ks, Kg + (size_t)j0 * ld, ld, nk, h);
    load_tile<HP, T>(Vs, Vg + (size_t)j0 * ld, ld, nk, h);
    wg::cp_async_commit();
    if (threadIdx.x < kT)
      vm[threadIdx.x] = threadIdx.x < nk && (lmask == nullptr || lmask[row0 + j0 + threadIdx.x]);
    wg::cp_async_wait<0>();
    fence_proxy_async();
    __syncthreads();
    const float Di[2] = {Dsm[row], Dsm[row + 8]};
    float s[32], dp[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) s[j] = dp[j] = 0.f;
    wgmma_fence();
    mma_heads<HP, T>(s, Qs, Ks);
    mma_heads<HP, T>(dp, Gs, Vs);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int r = acc_half(j), c = acc_col(j, t);
      float ds = 0.f;
      if (c < nk) {
        const float x = vm[c] ? s[j] * scale : s[j] * scale + kMaskAdder;
        const float pr = expf(x - mi[r]) * il[r];
        float kf = 1.f;
        if (drop > 0.f)
          kf = din_uniform(dseed, (ebase + i0 + row + 8 * r) * N + j0 + c) >= drop ? kscale : 0.f;
        ds = pr * (dp[j] * kf - Di[r]);
      }
      s[j] = ds;
    }
    wgmma_fence();
    mma_items<HP, T>(dq, s, Ks);
    wgmma_commit();
    wgmma_wait<0>();
  }
  store_rows<HP, T>(dq, dqkv + (row0 + i0) * ld + hd * h, ld, n, h, scale);
}

// Backward, key-owning pass: S^T = K Q^T and dP^T = V dO^T per query tile; dV = bf16(P~)^T dO
// and dK = scale bf16(dS)^T Q.
template <int HP, typename T>
__global__ void __launch_bounds__(kThreads)
attn_bwd_dkv16_kernel(const T* __restrict__ qkv, const uint8_t* __restrict__ lmask, int N,
                         int H, int h, float scale, float drop, unsigned long long dseed,
                         const float* __restrict__ lse, const float* __restrict__ dsum,
                         const T* __restrict__ dO, T* __restrict__ dqkv) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* Ks = align1024(smem_raw);
  unsigned char* Vs = Ks + tile_bytes(HP);
  unsigned char* Qs = Vs + tile_bytes(HP);
  unsigned char* Gs = Qs + tile_bytes(HP);
  float* ms = reinterpret_cast<float*>(Gs + tile_bytes(HP));
  float* ls = ms + kT;
  float* dd = ls + kT;
  const int tiles = (N + kT - 1) / kT;
  const int bh = blockIdx.x / tiles, j0 = (blockIdx.x % tiles) * kT;
  const int hd = bh % H, HH = H * h, ld = 3 * HH;
  const size_t row0 = (size_t)(bh / H) * N;
  const T* Qg = qkv + row0 * ld + hd * h;
  const T* Kg = Qg + HH;
  const T* Vg = Qg + 2 * HH;
  const T* Gg = dO + row0 * HH + hd * h;
  const int lane = threadIdx.x & 31, t = lane & 3;
  const int row = 16 * (threadIdx.x >> 5) + (lane >> 2);
  const float kscale = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  const unsigned long long ebase = (unsigned long long)bh * N;
  const int n = min(kT, N - j0);
  load_tile<HP, T>(Ks, Kg + (size_t)j0 * ld, ld, n, h);
  load_tile<HP, T>(Vs, Vg + (size_t)j0 * ld, ld, n, h);
  bool valid[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int j = row + 8 * r;
    valid[r] = j < n && (lmask == nullptr || lmask[row0 + j0 + j]);
  }
  float dk[HP / 2], dv[HP / 2];
#pragma unroll
  for (int j = 0; j < HP / 2; ++j) dk[j] = dv[j] = 0.f;
  for (int i0 = 0; i0 < N; i0 += kT) {
    const int nq = min(kT, N - i0);
    __syncthreads();
    load_tile<HP, T>(Qs, Qg + (size_t)i0 * ld, ld, nq, h);
    load_tile<HP, T>(Gs, Gg + (size_t)i0 * HH, HH, nq, h);
    wg::cp_async_commit();
    if (threadIdx.x < kT) {
      const bool ok = threadIdx.x < nq;
      const size_t q = row0 + i0 + threadIdx.x;
      ms[threadIdx.x] = ok ? lse[(q * H + hd) * 2] : 0.f;
      ls[threadIdx.x] = ok ? lse[(q * H + hd) * 2 + 1] : 0.f;
      dd[threadIdx.x] = ok ? dsum[q * H + hd] : 0.f;
    }
    wg::cp_async_wait<0>();
    fence_proxy_async();
    __syncthreads();
    float s[32], dp[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) s[j] = dp[j] = 0.f;
    wgmma_fence();
    mma_heads<HP, T>(s, Ks, Qs);
    mma_heads<HP, T>(dp, Vs, Gs);
    wgmma_commit();
    wgmma_wait<0>();
    const unsigned long long e0 = (ebase + i0) * N + j0 + row;   // element of (query 0, row)
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int r = acc_half(j), c = acc_col(j, t);   // key row + 8 r, query c
      float ds = 0.f, pt = 0.f;
      if (c < nq) {
        const float x = valid[r] ? s[j] * scale : s[j] * scale + kMaskAdder;
        const float pr = expf(x - ms[c]) * ls[c];
        float kf = 1.f;
        if (drop > 0.f && row + 8 * r < n)
          kf = din_uniform(dseed, e0 + (unsigned long long)c * N + 8 * r) >= drop ? kscale : 0.f;
        ds = pr * (dp[j] * kf - dd[c]);
        pt = pr * kf;
      }
      s[j] = ds;
      dp[j] = pt;
    }
    wgmma_fence();
    mma_items<HP, T>(dv, dp, Gs);
    mma_items<HP, T>(dk, s, Qs);
    wgmma_commit();
    wgmma_wait<0>();
  }
  T* base = dqkv + (row0 + j0) * ld + hd * h;
  store_rows<HP, T>(dk, base + HH, ld, n, h, scale);
  store_rows<HP, T>(dv, base + 2 * HH, ld, n, h, 1.f);
}

template <int HP>
constexpr size_t fwd_smem() { return 1024 + 3 * tile_bytes(HP) + kT; }
template <int HP>
constexpr size_t dq_smem() { return 1024 + 4 * tile_bytes(HP) + kT * sizeof(float) + kT; }
template <int HP>
constexpr size_t dkv_smem() { return 1024 + 4 * tile_bytes(HP) + 3 * kT * sizeof(float); }
static_assert(dkv_smem<128>() <= wg::kSmemLimit, "the key pass fits one CTA per SM");

int set_smem(const void* fn, size_t bytes) {
  TFR_CUDA_OK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return TFR_OK;
}

template <int HP, typename T>
int fwd(const T* qkv, const uint8_t* lmask, int B, int N, int H, int h, float drop,
        unsigned long long s, T* O, float* lse, cudaStream_t st) {
  int rc = set_smem((const void*)attn_fwd16_kernel<HP, T>, fwd_smem<HP>());
  if (rc) return rc;
  const unsigned grid = (unsigned)B * H * ((N + kT - 1) / kT);
  attn_fwd16_kernel<HP, T><<<grid, kThreads, fwd_smem<HP>(), st>>>(
      qkv, lmask, N, H, h, 1.f / sqrtf((float)h), drop, s, O, lse);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

template <int HP, typename T>
int bwd(const T* qkv, const uint8_t* lmask, int B, int N, int H, int h, float drop,
        unsigned long long s, const T* O, const float* lse, const T* dO, float* dsum,
        T* dqkv, cudaStream_t st) {
  const float scale = 1.f / sqrtf((float)h);
  const unsigned grid = (unsigned)B * H * ((N + kT - 1) / kT);
  int rc = set_smem((const void*)attn_bwd_dq16_kernel<HP, T>, dq_smem<HP>());
  if (rc) return rc;
  attn_bwd_dq16_kernel<HP, T><<<grid, kThreads, dq_smem<HP>(), st>>>(
      qkv, lmask, N, H, h, scale, drop, s, O, lse, dO, dsum, dqkv);
  TFR_LAUNCH_OK();
  rc = set_smem((const void*)attn_bwd_dkv16_kernel<HP, T>, dkv_smem<HP>());
  if (rc) return rc;
  attn_bwd_dkv16_kernel<HP, T><<<grid, kThreads, dkv_smem<HP>(), st>>>(
      qkv, lmask, N, H, h, scale, drop, s, lse, dsum, dO, dqkv);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

}  // namespace

int din16_attn_fwd(const __nv_bfloat16* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                   float drop, unsigned long long dseed, __nv_bfloat16* O, float* lse,
                   cudaStream_t st) {
  return TFR_DIN16_DISPATCH(h, fwd, bf16, qkv, lmask, B, N, H, h, drop, dseed, O, lse, st);
}
int din16_attn_fwd(const __half* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                   float drop, unsigned long long dseed, __half* O, float* lse, cudaStream_t st) {
  return TFR_DIN16_DISPATCH(h, fwd, __half, qkv, lmask, B, N, H, h, drop, dseed, O, lse, st);
}

int din16_attn_bwd(const __nv_bfloat16* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                   float drop, unsigned long long dseed, const __nv_bfloat16* O,
                   const float* lse, const __nv_bfloat16* dO, float* dsum,
                   __nv_bfloat16* dqkv, cudaStream_t st) {
  return TFR_DIN16_DISPATCH(h, bwd, bf16, qkv, lmask, B, N, H, h, drop, dseed, O, lse, dO,
                               dsum, dqkv, st);
}
int din16_attn_bwd(const __half* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                   float drop, unsigned long long dseed, const __half* O, const float* lse,
                   const __half* dO, float* dsum, __half* dqkv, cudaStream_t st) {
  return TFR_DIN16_DISPATCH(h, bwd, __half, qkv, lmask, B, N, H, h, drop, dseed, O, lse, dO,
                               dsum, dqkv, st);
}

namespace {

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// The parity entries' limits: those of TFR-BERT's 16-bit modes (tfr_bert_*), checked before any
// CUDA call.  ty names the element type in the messages.
int check_attn(const char* ty, const void* qkv, int B, int N, int H, int h, float drop) {
  TFR_REQUIRE(qkv, "%s attention: NULL qkv", ty);
  TFR_REQUIRE(h >= 8 && h <= 128 && h % 8 == 0,
              "%s attention: head size %d must be a multiple of 8 in [8, 128]", ty, h);
  TFR_REQUIRE(N >= 1 && N <= TFR_DIN_MAX_LIST, "%s attention: N %d must be in [1, %d]", ty, N,
              TFR_DIN_MAX_LIST);
  TFR_REQUIRE(H >= 1 && (long long)H * h <= TFR_BERT_MAX_HIDDEN,
              "%s attention: %d heads of %d exceed %d columns", ty, H, h, TFR_BERT_MAX_HIDDEN);
  TFR_REQUIRE(B >= 0 && (long long)B * H * ((N + kT - 1) / kT) <= 0x7fffffffLL,
              "%s attention: batch %d out of range", ty, B);
  TFR_REQUIRE(drop >= 0.f && drop < 1.f, "%s attention: dropout rate must be in [0, 1)", ty);
  return TFR_OK;
}

template <typename T>
int parity_fwd(const char* ty, const void* qkv, const uint8_t* lmask, int B, int N, int H, int h,
               float drop, unsigned long long dseed, void* O, float* lse, void* stream) {
  int rc = check_attn(ty, qkv, B, N, H, h, drop);
  if (rc) return rc;
  TFR_REQUIRE(O && lse, "%s attention: NULL output", ty);
  TFR_REQUIRE(aligned16(qkv) && aligned16(O) && aligned16(lse),
              "%s attention: operands must be 16-byte aligned", ty);
  if (B == 0) return TFR_OK;
  return din16_attn_fwd(static_cast<const T*>(qkv), lmask, B, N, H, h, drop, dseed,
                        static_cast<T*>(O), lse, (cudaStream_t)stream);
}

template <typename T>
int parity_bwd(const char* ty, const void* qkv, const uint8_t* lmask, int B, int N, int H, int h,
               float drop, unsigned long long dseed, const void* O, const float* lse,
               const void* dO, float* dsum, void* dqkv, void* stream) {
  int rc = check_attn(ty, qkv, B, N, H, h, drop);
  if (rc) return rc;
  TFR_REQUIRE(O && lse && dO && dsum && dqkv, "%s attention: NULL operand", ty);
  TFR_REQUIRE(aligned16(qkv) && aligned16(O) && aligned16(lse) && aligned16(dO) &&
                  aligned16(dsum) && aligned16(dqkv),
              "%s attention: operands must be 16-byte aligned", ty);
  if (B == 0) return TFR_OK;
  return din16_attn_bwd(static_cast<const T*>(qkv), lmask, B, N, H, h, drop, dseed,
                        static_cast<const T*>(O), lse, static_cast<const T*>(dO), dsum,
                        static_cast<T*>(dqkv), (cudaStream_t)stream);
}

}  // namespace
}  // namespace tfr

// Parity entries: the 16-bit attention core alone (see include/tfr_b200.h).
extern "C" int tfr_attn_bf16_fwd(const void* qkv, const uint8_t* lmask, int B, int N, int H,
                                 int h, float drop, unsigned long long dseed, void* O, float* lse,
                                 void* stream) {
  return tfr::parity_fwd<__nv_bfloat16>("bf16", qkv, lmask, B, N, H, h, drop, dseed, O, lse,
                                        stream);
}

extern "C" int tfr_attn_bf16_bwd(const void* qkv, const uint8_t* lmask, int B, int N, int H,
                                 int h, float drop, unsigned long long dseed, const void* O,
                                 const float* lse, const void* dO, float* dsum, void* dqkv,
                                 void* stream) {
  return tfr::parity_bwd<__nv_bfloat16>("bf16", qkv, lmask, B, N, H, h, drop, dseed, O, lse, dO,
                                        dsum, dqkv, stream);
}

extern "C" int tfr_attn_f16_fwd(const void* qkv, const uint8_t* lmask, int B, int N, int H,
                                int h, float drop, unsigned long long dseed, void* O, float* lse,
                                void* stream) {
  return tfr::parity_fwd<__half>("fp16", qkv, lmask, B, N, H, h, drop, dseed, O, lse, stream);
}

extern "C" int tfr_attn_f16_bwd(const void* qkv, const uint8_t* lmask, int B, int N, int H,
                                int h, float drop, unsigned long long dseed, const void* O,
                                const float* lse, const void* dO, float* dsum, void* dqkv,
                                void* stream) {
  return tfr::parity_bwd<__half>("fp16", qkv, lmask, B, N, H, h, drop, dseed, O, lse, dO, dsum,
                                 dqkv, stream);
}
