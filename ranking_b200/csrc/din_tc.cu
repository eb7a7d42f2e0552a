// K11 DocumentInteractionAttention, TF32 tensor-core attention core (tfr_din_cfg precision
// TFR_PREC_TF32): the contractions of din.cu's SIMT kernels on wgmma m64nNk8 (TF32 operands,
// fp32 accumulate); softmax, masking and dropout in fp32 registers, as there.
//
// A CTA is one warpgroup and owns 64 rows of one (list, head): query rows in the forward and
// the backward's query pass, key rows in its key pass.  The other side streams through shared
// memory in tiles of 64 items.  Every shared tile is 128-byte swizzled and K-major (k
// contiguous), in blocks of 32 floats of k:
//   * an operand whose contraction runs over the head dimension (Q, K, V, dO as stored in
//     qkv / dO) is copied as is, by cp.async, columns past h and rows past N zero-filled; both
//     A and B of S = Q K^T, dP = dO V^T, S^T = K Q^T and dP^T = V dO^T are read from there by
//     descriptor;
//   * an operand whose contraction runs over items (V in O = P~ V, K in dQ = dS K, dO and Q in
//     dV = P~^T dO and dK = dS^T Q) is MN-major as stored, and TF32 wgmma reads only K-major B,
//     so it is transposed on its way into shared memory: row = head dimension (zero past h),
//     k = item (zero past N).
// The A operand of the second product (P~, dS, their transposes) comes from the first product's
// accumulators, in registers, without a shuffle: lane t's accumulator holds items 2t and 2t + 1
// of each group of 8, while its A fragment covers k = t and t + 4.  So item 2t + c of a group is
// stored at k = t + 4c of the transposed tile (perm_k), and the fragment is the accumulator's
// registers in another order (frag_of_acc).
//
// The backward keeps the SIMT kernels' two passes and grid: no atomics, so two identical calls
// give identical bits.  The head dimension is padded to a bucket HP (tc_bucket, the one table),
// the n width of the O / dQ / dK / dV products and the padded k of the S products.
#include "common.cuh"
#include "din.cuh"
#include "wgmma_gemm.cuh"

namespace tfr {
namespace {

using wg::cp_async16;
using wg::desc_sw128;
using wg::fence_proxy_async;
using wg::smem_u32;
using wg::swz_chunk;
using wg::tf32_rn;
using wg::wgmma_commit;
using wg::wgmma_fence;
using wg::wgmma_wait;

constexpr int kT = 64;             // rows a CTA owns; items per streamed tile
constexpr int kTcThreads = 128;    // one warpgroup

// Head-size buckets: HP = the padded head size a kernel is instantiated for.
__host__ __device__ constexpr int tc_bucket(int h) {
  return h <= 16 ? 16 : h <= 32 ? 32 : h <= 64 ? 64 : 128;
}
#define TFR_DIN_TC_DISPATCH(h, fn, ...)                                                  \
  (tc_bucket(h) == 16 ? fn<16>(__VA_ARGS__) : tc_bucket(h) == 32 ? fn<32>(__VA_ARGS__) \
   : tc_bucket(h) == 64 ? fn<64>(__VA_ARGS__) : fn<128>(__VA_ARGS__))

// Shared tiles: kT rows x HP of k (blocks of kT x 128 B), and HP rows x kT items of k (two
// blocks of HP x 128 B).  Every block starts 1024-aligned, as the swizzle atoms need.
__host__ __device__ constexpr int kmajor_bytes(int hp) { return (hp < 32 ? 1 : hp / 32) * kT * 128; }
__host__ __device__ constexpr int trans_bytes(int hp) { return 2 * hp * 128; }

// Descriptor of k step ks (8 floats) of a tile whose k blocks are `block` bytes apart.
__device__ __forceinline__ uint64_t kdesc(const unsigned char* tile, int block, int ks) {
  return desc_sw128(smem_u32(tile + (ks >> 2) * block + (ks & 3) * 32));
}

// Rows [0, kT) x k [0, HP) of a K-major tile: row r < n, column c < h from src[r ld + c], zero
// elsewhere.  cp.async; the caller commits and waits.
template <int HP>
__device__ __forceinline__ void load_kmajor(unsigned char* dst, const float* src, int ld, int n,
                                            int h) {
  constexpr int CPR = (HP < 32 ? 32 : HP) / 4;   // 16-byte chunks per row
  for (int e = threadIdx.x; e < kT * CPR; e += kTcThreads) {
    const int r = e / CPR, kc = e % CPR;
    const bool ok = r < n && kc * 4 < h;
    cp_async16(smem_u32(dst + (kc >> 3) * (kT * 128) + swz_chunk(r, kc & 7)),
               ok ? src + (size_t)r * ld + kc * 4 : src, ok ? 16 : 0);
  }
}

// k position of item jj in a transposed tile (see the top of the file).
__device__ __forceinline__ int perm_k(int jj) {
  return (jj & ~7) | ((jj & 7) >> 1) | ((jj & 1) << 2);
}

// The transposed tile of items [0, kT) of src (row pitch ld): row c < h, k = perm_k(item) holds
// src[item ld + c] for item < n; zero elsewhere.  Like the tiles copied as stored, it is
// truncated to TF32 by the tensor core, so V enters O (forward) and dP (backward) alike.
template <int HP>
__device__ __forceinline__ void load_trans(unsigned char* dst, const float* src, int ld, int n,
                                           int h) {
  constexpr int CPR = HP / 4;
  for (int e = threadIdx.x; e < kT * CPR; e += kTcThreads) {
    const int jj = e / CPR, c = (e % CPR) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (jj < n && c < h) v = *reinterpret_cast<const float4*>(src + (size_t)jj * ld + c);
    const int k = perm_k(jj);
    unsigned char* b = dst + (k >> 5) * (HP * 128) + ((k & 3) << 2);
    const int kc = (k & 31) >> 2;
    *reinterpret_cast<float*>(b + swz_chunk(c, kc)) = v.x;
    *reinterpret_cast<float*>(b + swz_chunk(c + 1, kc)) = v.y;
    *reinterpret_cast<float*>(b + swz_chunk(c + 2, kc)) = v.z;
    *reinterpret_cast<float*>(b + swz_chunk(c + 3, kc)) = v.w;
  }
}

// Accumulator element j of an m64nN product: row 16 warp + lane / 4 + 8 acc_half(j), column
// acc_col(j) (lane % 4 = t).
__device__ __forceinline__ int acc_half(int j) { return (j >> 1) & 1; }
__device__ __forceinline__ int acc_col(int j, int t) { return 8 * (j >> 2) + 2 * t + (j & 1); }

// A fragment of k step ks (items 8 ks .. 8 ks + 7, in perm_k order) from an m64n64 accumulator,
// rounded to nearest TF32: truncation would shrink every P~ and dS by 2^-11 on average, a
// one-sided error that no longer averages out over the items.
__device__ __forceinline__ void frag_of_acc(const float (&acc)[32], int ks, uint32_t (&a)[4]) {
  a[0] = __float_as_uint(tf32_rn(acc[4 * ks]));
  a[1] = __float_as_uint(tf32_rn(acc[4 * ks + 2]));
  a[2] = __float_as_uint(tf32_rn(acc[4 * ks + 1]));
  a[3] = __float_as_uint(tf32_rn(acc[4 * ks + 3]));
}

#define TFR_F8(d, o)                                                                         \
  "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), \
      "+f"(d[o + 6]), "+f"(d[o + 7])
#define TFR_F32(d, o) TFR_F8(d, o), TFR_F8(d, o + 8), TFR_F8(d, o + 16), TFR_F8(d, o + 24)
#define TFR_R32                                                                              \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, "  \
  "%19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"

// D[64 x 64] += A B, both from shared memory.
__device__ __forceinline__ void mma_ss64(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " TFR_R32
               ", %32, %33, 1, 1, 1;"
               : TFR_F32(d, 0)
               : "l"(da), "l"(db));
}
// D[64 x N] += A B, A from registers.
template <int N>
__device__ __forceinline__ void mma_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t db) {
  if constexpr (N == 16) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, 1, 1, 1;"
                 : TFR_F8(d, 0)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
  } else if constexpr (N == 32) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
                 "{%16, %17, %18, %19}, %20, 1, 1, 1;"
                 : TFR_F8(d, 0), TFR_F8(d, 8)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
  } else if constexpr (N == 64) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " TFR_R32
                 ", {%32, %33, %34, %35}, %36, 1, 1, 1;"
                 : TFR_F32(d, 0)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
  } else {
    static_assert(N == 128, "n width");
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, "
                 "%17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, "
                 "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, "
                 "%62, %63}, {%64, %65, %66, %67}, %68, 1, 1, 1;"
                 : TFR_F32(d, 0), TFR_F32(d, 32)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
  }
}
#undef TFR_F8
#undef TFR_F32
#undef TFR_R32

// S (or S^T) = A B^T over the padded head dimension, both K-major tiles of kT rows.
template <int HP>
__device__ __forceinline__ void mma_heads(float (&d)[32], const unsigned char* a,
                                          const unsigned char* b) {
#pragma unroll
  for (int ks = 0; ks < HP / 8; ++ks)
    mma_ss64(d, kdesc(a, kT * 128, ks), kdesc(b, kT * 128, ks));
}
// D += A B over the kT items of a tile: A from the accumulator `p`, B a transposed tile.
template <int HP>
__device__ __forceinline__ void mma_items(float (&d)[HP / 2], const float (&p)[32],
                                          const unsigned char* bt) {
#pragma unroll
  for (int ks = 0; ks < kT / 8; ++ks) {
    uint32_t a[4];
    frag_of_acc(p, ks, a);
    mma_rs<HP>(d, a, kdesc(bt, HP * 128, ks));
  }
}

// What the tensor core reads of an fp32 operand: the low 13 mantissa bits cleared.
__device__ __forceinline__ float tf32_trunc(float x) {
  return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
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
// columns < h, times `mul`.
template <int HP>
__device__ __forceinline__ void store_rows(const float (&acc)[HP / 2], float* base, int ld, int n,
                                           int h, const float (&mul)[2]) {
  const int lane = threadIdx.x & 31, row = 16 * (threadIdx.x >> 5) + (lane >> 2);
#pragma unroll
  for (int j = 0; j < HP / 2; j += 2) {
    const int r = row + 8 * acc_half(j), c = acc_col(j, lane & 3);
    if (r < n && c < h)   // h % 4 == 0: c even, so c + 1 < h too
      *reinterpret_cast<float2*>(base + (size_t)r * ld + c) =
          make_float2(acc[j] * mul[acc_half(j)], acc[j + 1] * mul[acc_half(j)]);
  }
}

// Forward: grid B H ceil(N / 64), CTA = 64 query rows of one (list, head).
template <int HP>
__global__ void __launch_bounds__(kTcThreads)
attn_fwd_tc_kernel(const float* __restrict__ qkv, const uint8_t* __restrict__ lmask, int N,
                   int H, int h, float scale, float drop, unsigned long long dseed,
                   float* __restrict__ O, float* __restrict__ lse) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* Qs = align1024(smem_raw);
  unsigned char* Ks = Qs + kmajor_bytes(HP);
  unsigned char* Vt = Ks + kmajor_bytes(HP);
  uint8_t* vm = Vt + trans_bytes(HP);
  const int tiles = (N + kT - 1) / kT;
  const int bh = blockIdx.x / tiles, i0 = (blockIdx.x % tiles) * kT;
  const int hd = bh % H, HH = H * h, ld = 3 * HH;
  const size_t row0 = (size_t)(bh / H) * N;
  const float* Qg = qkv + row0 * ld + hd * h;
  const float* Kg = Qg + HH;
  const float* Vg = Qg + 2 * HH;
  const int lane = threadIdx.x & 31, t = lane & 3;
  const int row = 16 * (threadIdx.x >> 5) + (lane >> 2);   // + 8 * half
  const float kscale = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  const unsigned long long ebase = (unsigned long long)bh * N;
  load_kmajor<HP>(Qs, Qg + (size_t)i0 * ld, ld, min(kT, N - i0), h);
  float o[HP / 2];
#pragma unroll
  for (int j = 0; j < HP / 2; ++j) o[j] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  for (int j0 = 0; j0 < N; j0 += kT) {
    const int nk = min(kT, N - j0);
    __syncthreads();   // every warpgroup product of the previous tile has completed
    load_kmajor<HP>(Ks, Kg + (size_t)j0 * ld, ld, nk, h);
    wg::cp_async_commit();
    load_trans<HP>(Vt, Vg + (size_t)j0 * ld, ld, nk, h);
    if (threadIdx.x < kT)
      vm[threadIdx.x] = threadIdx.x < nk && (lmask == nullptr || lmask[row0 + j0 + threadIdx.x]);
    wg::cp_async_wait<0>();
    fence_proxy_async();
    __syncthreads();
    float s[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) s[j] = 0.f;
    wgmma_fence();
    mma_heads<HP>(s, Qs, Ks);
    wgmma_commit();
    wgmma_wait<0>();
    float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int c = acc_col(j, t);
      s[j] = c < nk ? (vm[c] ? s[j] * scale : s[j] * scale + kMaskAdder) : -INFINITY;
      tmax[acc_half(j)] = fmaxf(tmax[acc_half(j)], s[j]);
    }
    float corr[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float mn = fmaxf(m[r], quad_max(tmax[r]));
      corr[r] = expf(m[r] - mn);
      l[r] *= corr[r];
      m[r] = mn;
    }
#pragma unroll
    for (int j = 0; j < HP / 2; ++j) o[j] *= corr[acc_half(j)];
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int r = acc_half(j), c = acc_col(j, t);
      float pr = expf(s[j] - m[r]);   // 0 past the list
      l[r] += pr;
      if (drop > 0.f && c < nk)
        pr = din_uniform(dseed, (ebase + i0 + row + 8 * r) * N + j0 + c) >= drop ? pr * kscale
                                                                                : 0.f;
      s[j] = pr;
    }
    wgmma_fence();
    mma_items<HP>(o, s, Vt);
    wgmma_commit();
    wgmma_wait<0>();
  }
  float inv[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) inv[r] = 1.f / quad_sum(l[r]);
  const int n = min(kT, N - i0);
  store_rows<HP>(o, O + (row0 + i0) * HH + hd * h, HH, n, h, inv);
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
// dS = P (dP keep / (1 - rate) - D_i); dQ = scale dS K.
template <int HP>
__global__ void __launch_bounds__(kTcThreads)
attn_bwd_dq_tc_kernel(const float* __restrict__ qkv, const uint8_t* __restrict__ lmask, int N,
                      int H, int h, float scale, float drop, unsigned long long dseed,
                      const float* __restrict__ O, const float* __restrict__ lse,
                      const float* __restrict__ dO, float* __restrict__ dsum,
                      float* __restrict__ dqkv) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* Qs = align1024(smem_raw);
  unsigned char* Gs = Qs + kmajor_bytes(HP);
  unsigned char* Ks = Gs + kmajor_bytes(HP);
  unsigned char* Vs = Ks + kmajor_bytes(HP);
  unsigned char* Kt = Vs + kmajor_bytes(HP);
  float* Dsm = reinterpret_cast<float*>(Kt + trans_bytes(HP));
  uint8_t* vm = reinterpret_cast<uint8_t*>(Dsm + kT);
  const int tiles = (N + kT - 1) / kT;
  const int bh = blockIdx.x / tiles, i0 = (blockIdx.x % tiles) * kT;
  const int hd = bh % H, HH = H * h, ld = 3 * HH;
  const size_t row0 = (size_t)(bh / H) * N;
  const float* Qg = qkv + row0 * ld + hd * h;
  const float* Kg = Qg + HH;
  const float* Vg = Qg + 2 * HH;
  const int lane = threadIdx.x & 31, t = lane & 3;
  const int row = 16 * (threadIdx.x >> 5) + (lane >> 2);
  const float kscale = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  const unsigned long long ebase = (unsigned long long)bh * N;
  const int n = min(kT, N - i0);
  const float* Gg = dO + (row0 + i0) * HH + hd * h;
  load_kmajor<HP>(Qs, Qg + (size_t)i0 * ld, ld, n, h);
  load_kmajor<HP>(Gs, Gg, HH, n, h);
  wg::cp_async_commit();
  {   // D_i: two threads per row, 4 columns of every 8 each.  dO is truncated to TF32 here as
      // the tensor core truncates it in dP = dO V^T: sum_j P_ij dP_ij then matches D_i but for
      // unbiased rounding, and sum_j dS_ij = 0 holds without a one-sided 2^-11 D_i offset
      // (which would carry the keys' shared component into dQ).
    const int r = threadIdx.x >> 1;
    float d = 0.f;
    if (r < n)
      for (int c = (threadIdx.x & 1) * 4; c < h; c += 8) {
        const float4 g = *reinterpret_cast<const float4*>(Gg + (size_t)r * HH + c);
        const float4 x = *reinterpret_cast<const float4*>(O + (row0 + i0 + r) * HH + hd * h + c);
        d += tf32_trunc(g.x) * x.x + tf32_trunc(g.y) * x.y + tf32_trunc(g.z) * x.z +
             tf32_trunc(g.w) * x.w;
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
    load_kmajor<HP>(Ks, Kg + (size_t)j0 * ld, ld, nk, h);
    load_kmajor<HP>(Vs, Vg + (size_t)j0 * ld, ld, nk, h);
    wg::cp_async_commit();
    load_trans<HP>(Kt, Kg + (size_t)j0 * ld, ld, nk, h);
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
    mma_heads<HP>(s, Qs, Ks);
    mma_heads<HP>(dp, Gs, Vs);
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
    mma_items<HP>(dq, s, Kt);
    wgmma_commit();
    wgmma_wait<0>();
  }
  const float mul[2] = {scale, scale};
  store_rows<HP>(dq, dqkv + (row0 + i0) * ld + hd * h, ld, n, h, mul);
}

// Backward, key-owning pass: S^T = K Q^T and dP^T = V dO^T per query tile; dV = P~^T dO and
// dK = scale dS^T Q.
template <int HP>
__global__ void __launch_bounds__(kTcThreads)
attn_bwd_dkv_tc_kernel(const float* __restrict__ qkv, const uint8_t* __restrict__ lmask, int N,
                       int H, int h, float scale, float drop, unsigned long long dseed,
                       const float* __restrict__ lse, const float* __restrict__ dsum,
                       const float* __restrict__ dO, float* __restrict__ dqkv) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* Ks = align1024(smem_raw);
  unsigned char* Vs = Ks + kmajor_bytes(HP);
  unsigned char* Qs = Vs + kmajor_bytes(HP);
  unsigned char* Gs = Qs + kmajor_bytes(HP);
  unsigned char* Qt = Gs + kmajor_bytes(HP);
  unsigned char* Gt = Qt + trans_bytes(HP);
  float* ms = reinterpret_cast<float*>(Gt + trans_bytes(HP));
  float* ls = ms + kT;
  float* dd = ls + kT;
  const int tiles = (N + kT - 1) / kT;
  const int bh = blockIdx.x / tiles, j0 = (blockIdx.x % tiles) * kT;
  const int hd = bh % H, HH = H * h, ld = 3 * HH;
  const size_t row0 = (size_t)(bh / H) * N;
  const float* Qg = qkv + row0 * ld + hd * h;
  const float* Kg = Qg + HH;
  const float* Vg = Qg + 2 * HH;
  const float* Gg = dO + row0 * HH + hd * h;
  const int lane = threadIdx.x & 31, t = lane & 3;
  const int row = 16 * (threadIdx.x >> 5) + (lane >> 2);
  const float kscale = drop > 0.f ? 1.f / (1.f - drop) : 1.f;
  const unsigned long long ebase = (unsigned long long)bh * N;
  const int n = min(kT, N - j0);
  load_kmajor<HP>(Ks, Kg + (size_t)j0 * ld, ld, n, h);
  load_kmajor<HP>(Vs, Vg + (size_t)j0 * ld, ld, n, h);
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
    load_kmajor<HP>(Qs, Qg + (size_t)i0 * ld, ld, nq, h);
    load_kmajor<HP>(Gs, Gg + (size_t)i0 * HH, HH, nq, h);
    wg::cp_async_commit();
    load_trans<HP>(Qt, Qg + (size_t)i0 * ld, ld, nq, h);
    load_trans<HP>(Gt, Gg + (size_t)i0 * HH, HH, nq, h);
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
    mma_heads<HP>(s, Ks, Qs);
    mma_heads<HP>(dp, Vs, Gs);
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
    mma_items<HP>(dv, dp, Gt);
    mma_items<HP>(dk, s, Qt);
    wgmma_commit();
    wgmma_wait<0>();
  }
  const float kmul[2] = {scale, scale}, vmul[2] = {1.f, 1.f};
  float* base = dqkv + (row0 + j0) * ld + hd * h;
  store_rows<HP>(dk, base + HH, ld, n, h, kmul);
  store_rows<HP>(dv, base + 2 * HH, ld, n, h, vmul);
}

template <int HP>
constexpr size_t fwd_smem() { return 1024 + 2 * kmajor_bytes(HP) + trans_bytes(HP) + kT; }
template <int HP>
constexpr size_t dq_smem() {
  return 1024 + 4 * kmajor_bytes(HP) + trans_bytes(HP) + kT * sizeof(float) + kT;
}
template <int HP>
constexpr size_t dkv_smem() {
  return 1024 + 4 * kmajor_bytes(HP) + 2 * trans_bytes(HP) + 3 * kT * sizeof(float);
}
static_assert(dkv_smem<128>() <= wg::kSmemLimit, "the key pass fits one CTA per SM");

int set_smem(const void* fn, size_t bytes) {
  TFR_CUDA_OK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return TFR_OK;
}

template <int HP>
int fwd(const float* qkv, const uint8_t* lmask, int B, int N, int H, int h, float drop,
        unsigned long long s, float* O, float* lse, cudaStream_t st) {
  int rc = set_smem((const void*)attn_fwd_tc_kernel<HP>, fwd_smem<HP>());
  if (rc) return rc;
  const unsigned grid = (unsigned)B * H * ((N + kT - 1) / kT);
  attn_fwd_tc_kernel<HP><<<grid, kTcThreads, fwd_smem<HP>(), st>>>(
      qkv, lmask, N, H, h, 1.f / sqrtf((float)h), drop, s, O, lse);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

template <int HP>
int bwd(const float* qkv, const uint8_t* lmask, int B, int N, int H, int h, float drop,
        unsigned long long s, const float* O, const float* lse, const float* dO, float* dsum,
        float* dqkv, cudaStream_t st) {
  const float scale = 1.f / sqrtf((float)h);
  const unsigned grid = (unsigned)B * H * ((N + kT - 1) / kT);
  int rc = set_smem((const void*)attn_bwd_dq_tc_kernel<HP>, dq_smem<HP>());
  if (rc) return rc;
  attn_bwd_dq_tc_kernel<HP><<<grid, kTcThreads, dq_smem<HP>(), st>>>(
      qkv, lmask, N, H, h, scale, drop, s, O, lse, dO, dsum, dqkv);
  TFR_LAUNCH_OK();
  rc = set_smem((const void*)attn_bwd_dkv_tc_kernel<HP>, dkv_smem<HP>());
  if (rc) return rc;
  attn_bwd_dkv_tc_kernel<HP><<<grid, kTcThreads, dkv_smem<HP>(), st>>>(
      qkv, lmask, N, H, h, scale, drop, s, lse, dsum, dO, dqkv);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

}  // namespace

int din_tc_attn_fwd(const float* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                    float drop, unsigned long long dseed, float* O, float* lse, cudaStream_t st) {
  return TFR_DIN_TC_DISPATCH(h, fwd, qkv, lmask, B, N, H, h, drop, dseed, O, lse, st);
}

int din_tc_attn_bwd(const float* qkv, const uint8_t* lmask, int B, int N, int H, int h,
                    float drop, unsigned long long dseed, const float* O, const float* lse,
                    const float* dO, float* dsum, float* dqkv, cudaStream_t st) {
  return TFR_DIN_TC_DISPATCH(h, bwd, qkv, lmask, B, N, H, h, drop, dseed, O, lse, dO, dsum, dqkv,
                             st);
}

}  // namespace tfr
