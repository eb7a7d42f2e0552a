// K5/K6 fused 3xTF32 forward of the scorer tower: every hidden Dense layer from
// `first_layer` on, plus the output layer, in one persistent kernel.
//
// A CTA (one per SM) owns a 128-row tile of M at a time and walks the tower depth-first on
// it.  Only the first fused layer reads its A operand (X) from HBM, through the stage ring;
// every later layer takes its A fragments from Hbuf, a 128 x 128 fp32 tile in shared memory
// that the previous layer's epilogue wrote.  A first layer wider than 128 runs in two
// 128-column chunks, and the next layer consumes each chunk as soon as its epilogue has
// written it (k 0..127, then 128..255), its accumulator kept in registers meanwhile.
//
// Every operand tile in shared memory has one layout, that of a TMA box of 32 fp32 columns x
// 128 rows with the 128-byte swizzle: row r at r * 128 bytes, its 16-byte chunk c at chunk
// c ^ (r % 8).  The wgmma descriptors read the W^T tiles in it, the A fragment loads of a warp
// hit 32 different banks in it, and Hbuf is four such panels (columns 0-31, ..., 96-127), so
// the epilogue warpgroup stores H_d from Hbuf with TMA.
//
// Threads 0-255 are the two MMA warpgroups (setmaxnreg 208): the k loop, and the half of each
// epilogue the next layer needs, bias + activation into Hbuf.  Thread 0 also issues the ring's
// TMA loads.  Threads 256-383 are the epilogue warpgroup (setmaxnreg 88): after each such Hbuf
// write it stores H_d from Hbuf by TMA and forms the ReLU sign words from it (the backward
// reads both), and after a tile's last hidden layer it computes the output layer from Hbuf,
// while the MMA warps run the next layer's k loop.  The hand-off is the GEMM engine's
// (wgmma_gemm.cuh): the MMA warps arrive at kBarFull once Hbuf is written and wait at kBarFree
// before they overwrite it; the epilogue warpgroup waits at kBarFull and arrives at kBarFree
// once it, and its TMA stores, have read it.
//
// The k blocks of a tile form one linear sequence (config 2: 5 + 4 + 5 + 4 + 4 blocks), block
// g in stage g mod kStages.  A block always brings the layer's pre-split W^T hi / lo tile;
// blocks of the first layer also bring the X tile.  TMA zero-fills what lies past K, N or M,
// as the engine's copies do.  Each stage has a `full` mbarrier (the TMA transactions) and an
// `empty` one (one arrival per MMA warp once the block's wgmma group has retired); thread 0
// refills a stage with the block kStages further on as soon as it is empty, across layer
// boundaries, epilogues and into the next tile.
//
// Results are those of the per-layer path bit for bit: every output element sees the same
// wgmma shapes (m64n128, or m64n64 when the tile's live columns fit in 64), the same k-block
// order, the same skipped all-zero k steps and the same hi.hi, lo.hi, hi.lo pass order as
// wg::gemm_kernel, and the scores are summed in out_layer_fwd_kernel's order (per-lane fma
// chains over k = lane, lane + 32, ..., then warp_sum).
//
// Between an MMA warp's Hbuf write and its next layer's fragment loads only __syncwarp is
// needed: the accumulator rows of warp w (16 w .. 16 w + 15) are the rows its A fragments
// read.  Hbuf is not warp-private as a whole, though: the epilogue warpgroup reads every row,
// hence kBarFree before every Hbuf write but a CTA's first.
#include <cuda.h>

#include "common.cuh"
#include "mlp.h"
#include "wgmma_gemm.cuh"

namespace tfr {
namespace fused {

constexpr int kPanel = wg::kTileBytes;                     // one 32-column swizzled box: 16 KB
constexpr int kStages = 3;
constexpr int kStage = 3 * kPanel;                         // W^T hi + W^T lo + X: 48 KB
constexpr int kAOff = 2 * kPanel;
constexpr int kHbufOff = kStages * kStage;                 // four panels: 64 KB
constexpr int kBarOff = kHbufOff + 4 * kPanel;             // full[kStages], empty[kStages]
constexpr int kSmem = kBarOff + 2 * kStages * 8 + 1024;    // + alignment slack
static_assert(kSmem == 214064, "fused forward shared memory: 3 stages + Hbuf + barriers + slack");
static_assert(kSmem <= wg::kSmemLimit, "fused forward exceeds the shared memory of a CTA");
constexpr int kMaxSegs = 4 + TFR_MLP_MAX_LAYERS;
constexpr int kMaxHidden = TFR_MLP_MAX_LAYERS - 1;
// kBarFull / kBarFree: the 256 MMA threads and the 128 epilogue threads, once per Hbuf write.
// Both sides walk the same (tile, segment with epi) sequence, so every wait has its arrive.
constexpr int kHandoff = wg::kThreads + wg::kEpiThreads;

// Float index of (row, column) in a stack of swizzled 32-column panels.
__device__ __forceinline__ int panel_idx(int row, int col) {
  const int c = col & 31;
  return (col >> 5) * (kPanel / 4) + row * 32 + ((((c >> 2) ^ row) & 7) << 2) + (c & 3);
}

// A run of k blocks of one layer that accumulates into one accumulator.
struct Seg {
  const float* bias;
  uint32_t* bits;                       // ReLU sign words [(col / 32) * M + row], or null
  int layer;                            // Dense layer d: tensor maps whi / wlo / h [d]
  int K, N;
  int n0;                               // first output column (tile of 128)
  int kb0, nkb;                         // k blocks [kb0, kb0 + nkb) of the layer
  int a_x;                              // A is X, streamed through the ring; else Hbuf
  int hoff;                             // Hbuf column 0 is layer k index hoff
  int acc;                              // accumulator 0 or 1
  int zero, epi;                        // clear the accumulator first / run the epilogue after
};

// TMA maps (boxes of 32 columns x 128 rows, 128-byte swizzle): X [M][K0]; per hidden layer d,
// W_d^T hi / lo [N][K] and H_d [M][N].
struct FusedArgs {
  CUtensorMap x;
  CUtensorMap whi[kMaxHidden], wlo[kMaxHidden], h[kMaxHidden];
  int M, m_tiles;
  int act;
  int nseg;
  Seg seg[kMaxSegs];
  const float* Wout; const float* bout;  // output layer [Kout, O], [O] (fp32)
  int Kout, O;
  const uint8_t* mask;
  float* scores;
};

// One wgmma group over a k block: NK k steps, each hi.hi, lo.hi, hi.lo (as wg::gemm_kernel).
template <bool W, int NK>
__device__ __forceinline__ void mma_block(float (&acc)[2][32], uint32_t (&ahi)[4][4],
                                          uint32_t (&alo)[4][4], uint32_t st) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      asm volatile("" : "+r"(ahi[ks][i]));
      asm volatile("" : "+r"(alo[ks][i]));
    }
  wg::wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < NK; ++ks) {
    const uint64_t dbh = wg::desc_sw128(st + ks * 32);
    const uint64_t dbl = wg::desc_sw128(st + kPanel + ks * 32);
    if (W) {
      wg::mma_tf32_n128(acc, ahi[ks], dbh);
      wg::mma_tf32_n128(acc, alo[ks], dbh);
      wg::mma_tf32_n128(acc, ahi[ks], dbl);
    } else {
      wg::mma_tf32_n64(acc, ahi[ks], dbh);
      wg::mma_tf32_n64(acc, alo[ks], dbh);
      wg::mma_tf32_n64(acc, ahi[ks], dbl);
    }
  }
  wg::wgmma_commit();
}

template <bool W>
__device__ __forceinline__ void mma_block_k(float (&acc)[2][32], uint32_t (&ahi)[4][4],
                                            uint32_t (&alo)[4][4], uint32_t st, int ksteps) {
  if (ksteps == 4) mma_block<W, 4>(acc, ahi, alo, st);
  else if (ksteps == 3) mma_block<W, 3>(acc, ahi, alo, st);
  else if (ksteps == 2) mma_block<W, 2>(acc, ahi, alo, st);
  else mma_block<W, 1>(acc, ahi, alo, st);
}

struct FusedCta {
  const FusedArgs& a;
  unsigned char* smem;
  uint32_t sbase;
  int lane, wrow;   // wrow: first of this warp's 16 tile rows
  int n;            // blocks consumed so far; block n sits in stage n % kStages
  int p_tile, p_seg, p_kb;   // thread 0: the block the next TMA fetches
  bool handed;      // Hbuf has been handed to the epilogue warpgroup before

  // The stage's mbarriers: full (the block's TMA bytes have landed) and empty (every MMA warp
  // is done with the block: 8 arrivals).
  __device__ __forceinline__ uint64_t* full(int s) {
    return reinterpret_cast<uint64_t*>(smem + kBarOff) + s;
  }
  __device__ __forceinline__ uint64_t* empty(int s) {
    return reinterpret_cast<uint64_t*>(smem + kBarOff) + kStages + s;
  }

  // Thread 0: once its stage is empty, loads the next block of the sequence, block number pn
  // (nothing past the last tile).
  __device__ __forceinline__ void produce(int pn) {
    if (p_tile >= a.m_tiles) return;
    const Seg& sg = a.seg[p_seg];
    const int s = pn % kStages;
    wg::mbar_wait(empty(s), ((pn / kStages) & 1) ^ 1);
    const uint32_t st = sbase + s * kStage;
    const int k0 = (sg.kb0 + p_kb) * 32;
    wg::mbar_expect_tx(full(s), (sg.a_x ? 3 : 2) * kPanel);
    wg::tma_load_2d(st, &a.whi[sg.layer], k0, sg.n0, full(s));
    wg::tma_load_2d(st + kPanel, &a.wlo[sg.layer], k0, sg.n0, full(s));
    if (sg.a_x) wg::tma_load_2d(st + kAOff, &a.x, k0, p_tile * wg::BM, full(s));
    if (++p_kb == sg.nkb) {
      p_kb = 0;
      if (++p_seg == a.nseg) {
        p_seg = 0;
        p_tile += gridDim.x;
      }
    }
  }

  __device__ __forceinline__ void run_seg(float (&acc)[2][32], const Seg& sg, int m0) {
    if (sg.zero) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[h][j] = 0.f;
    }
    const bool two_n = sg.n0 + 64 < sg.N;   // the second 64 columns hold live columns
    const int g = lane >> 2, t = lane & 3;
    for (int kb = 0; kb < sg.nkb; ++kb) {
      const int s = n % kStages;
      const uint32_t st = sbase + s * kStage;
      const int kg = (sg.kb0 + kb) * 32;   // first k of the block within the layer
      const int krem = sg.K - kg;
      const int ksteps = krem >= 32 ? 4 : (krem + 7) / 8;
      const unsigned char* sa =
          sg.a_x ? smem + s * kStage + kAOff : smem + kHbufOff + ((kg - sg.hoff) >> 5) * kPanel;
      wg::mbar_wait(full(s), (n / kStages) & 1);
      // A fragments (m64 x k, per warp 16 rows): register i holds row g + 8 (i % 2),
      // k t + 4 (i / 2), at chunk (k / 4) ^ (row % 8) = (2 ks + i / 2) ^ g of its row; split
      // into hi / lo in registers
      uint32_t ahi[4][4], alo[4][4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int rr = wrow + g + 8 * (i & 1);
          const float x = *reinterpret_cast<const float*>(
              sa + rr * 128 + (((2 * ks + (i >> 1)) ^ g) << 4) + t * 4);
          const float h = wg::tf32_rn(x);
          ahi[ks][i] = __float_as_uint(h);
          alo[ks][i] = __float_as_uint(x - h);
        }
      if (two_n) mma_block_k<true>(acc, ahi, alo, st, ksteps);
      else mma_block_k<false>(acc, ahi, alo, st, ksteps);
      wg::wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) wg::mbar_arrive(empty(s));
      ++n;
      if (threadIdx.x == 0) produce(n - 1 + kStages);   // into the stage just freed
    }
    if (sg.epi) epilogue(acc, sg, m0, two_n);
  }

  // The MMA warps' half of an epilogue: bias and activation as wg::gemm_kernel's EPI_BIAS_ACT,
  // zero past M and N (the next layer's zero-filled k tail), into Hbuf; then Hbuf goes to the
  // epilogue warpgroup, which stores it.
  __device__ __forceinline__ void epilogue(float (&acc)[2][32], const Seg& sg, int m0, bool two_n) {
    // accumulator element j of half h: row = lane / 4 + 8 ((j / 2) % 2),
    // column = 64 h + 8 (j / 4) + 2 (lane % 4) + j % 2
    float* hb = reinterpret_cast<float*>(smem + kHbufOff);
    // the epilogue warpgroup is done with the last Hbuf (this warp's own reads of it are too)
    if (handed) wg::bar_sync(wg::kBarFree, kHandoff);
    else __syncwarp();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (h == 1 && !two_n) break;
#pragma unroll
      for (int j = 0; j < 32; j += 2) {
        const int cin = h * 64 + 8 * (j >> 2) + 2 * (lane & 3);
        const int rl = wrow + (lane >> 2) + 8 * ((j >> 1) & 1);
        float x[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = sg.n0 + cin + e;
          float v = acc[h][j + e];
          v += col < sg.N ? __ldg(sg.bias + col) : 0.f;
          if (a.act == TFR_ACT_RELU) v = fmaxf(v, 0.f);
          if (m0 + rl >= a.M || col >= sg.N) v = 0.f;
          x[e] = v;
        }
        *reinterpret_cast<float2*>(hb + panel_idx(rl, cin)) = make_float2(x[0], x[1]);
      }
    }
    // Hbuf written before any lane of the warp reads it, and visible to the TMA stores
    wg::fence_proxy_async();
    __syncwarp();
    wg::bar_arrive(wg::kBarFull, kHandoff);
    handed = true;
  }
};

// H_d and the ReLU sign words of one segment's columns, from Hbuf.  One thread stores the live
// panels by TMA (clipped to M and N).  The sign words: a job is one 32-column plane of 32 rows,
// and the warps take jobs round-robin.  Lane c reads column c of a row, __ballot_sync forms
// the row's word, lane r keeps the word of row r and stores it after the 32 rows: one 128-byte
// line per job.  Columns past N are zero in Hbuf, so their bits are clear.
__device__ __forceinline__ void store_seg(const FusedArgs& a, const Seg& sg, const float* hb,
                                          uint32_t hb_s, int m0, int ew, int lane) {
  const int planes = min(4, (sg.N - sg.n0 + 31) >> 5);
  if (ew == 0 && lane == 0) {
    for (int p = 0; p < planes; ++p)
      wg::tma_store_2d(&a.h[sg.layer], hb_s + p * kPanel, sg.n0 + 32 * p, m0);
    wg::bulk_commit();
  }
  if (!sg.bits) return;
  for (int job = ew; job < 4 * planes; job += 4) {
    const int p = job >> 2, r0 = 32 * (job & 3);
    uint32_t keep = 0u;
#pragma unroll 8
    for (int i = 0; i < 32; ++i) {
      const uint32_t w = __ballot_sync(0xffffffffu, hb[panel_idx(r0 + i, 32 * p + lane)] > 0.f);
      if (i == lane) keep = w;
    }
    const int row = m0 + r0 + lane;
    if (row < a.M) sg.bits[static_cast<size_t>((sg.n0 >> 5) + p) * a.M + row] = keep;
  }
}

// Scores of tile rows 32 ew .. 32 ew + 31 from the last hidden layer in Hbuf, in
// out_layer_fwd_kernel's order; RestoreList fill for masked rows.  kPlanar: task-major
// scores[o * M + row] with the fill on every plane, as out_layer_fwd_kernel<true>.
template <bool kPlanar>
__device__ __forceinline__ void out_rows(const FusedArgs& a, const float* hb, int m0, int ew,
                                         int lane) {
  for (int r0 = 32 * ew; r0 < 32 * ew + 32; r0 += 4) {
    for (int o = 0; o < a.O; ++o) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int k = lane; k < a.Kout; k += 32) {
        const float w = __ldg(a.Wout + static_cast<size_t>(k) * a.O + o);
#pragma unroll
        for (int r = 0; r < 4; ++r) acc[r] = fmaf(hb[panel_idx(r0 + r, k)], w, acc[r]);
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[r] = warp_sum(acc[r]);
      const int row = m0 + r0 + lane;
      if (lane < 4 && row < a.M) {
        float v = (lane == 0 ? acc[0] : lane == 1 ? acc[1] : lane == 2 ? acc[2] : acc[3]) +
                  __ldg(a.bout + o);
        if (a.mask && (kPlanar || a.O == 1) && !a.mask[row]) v = kLogEpsilon;
        a.scores[kPlanar ? static_cast<size_t>(o) * a.M + row : static_cast<size_t>(row) * a.O + o] =
            v;
      }
    }
  }
}

// The epilogue warpgroup walks the CTA's tiles and segments as the MMA warps do and takes
// every Hbuf they hand over; the last segment with an epilogue is the last hidden layer, whose
// Hbuf also feeds the output layer.  It frees Hbuf after every pass but the CTA's last, which
// nobody would wait for; the thread that issued the pass's TMA stores first waits until they
// have read Hbuf.
template <bool kPlanar>
__device__ __forceinline__ void epilogue_warpgroup(const FusedArgs& a, const float* hb) {
  const int lane = threadIdx.x & 31, ew = (threadIdx.x - wg::kThreads) >> 5;
  const uint32_t hb_s = wg::smem_u32(hb);
  int last = 0;
  for (int q = 0; q < a.nseg; ++q)
    if (a.seg[q].epi) last = q;
  for (int tile = blockIdx.x; tile < a.m_tiles; tile += gridDim.x) {
    const int m0 = tile * wg::BM;
    for (int q = 0; q <= last; ++q) {
      const Seg& sg = a.seg[q];
      if (!sg.epi) continue;
      wg::bar_sync(wg::kBarFull, kHandoff);
      store_seg(a, sg, hb, hb_s, m0, ew, lane);
      if (q == last) out_rows<kPlanar>(a, hb, m0, ew, lane);
      if (q != last || tile + static_cast<int>(gridDim.x) < a.m_tiles) {
        if (ew == 0 && lane == 0) wg::bulk_wait_read<0>();
        wg::bar_arrive(wg::kBarFree, kHandoff);
      }
    }
  }
  if (ew == 0 && lane == 0) wg::bulk_wait<0>();
}

template <bool kPlanar>
__device__ __forceinline__ void tower_fused_fwd(const FusedArgs& args) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (wg::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kBarOff);
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      wg::mbar_init(&bars[s], 1);
      wg::mbar_init(&bars[kStages + s], wg::kWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x >= wg::kThreads) {
    wg::setmaxnreg_dec<wg::kEpiRegs>();
    epilogue_warpgroup<kPlanar>(args, reinterpret_cast<const float*>(smem + kHbufOff));
    return;
  }
  wg::setmaxnreg_inc<wg::kMmaRegs>();
  FusedCta cta{args, smem, wg::smem_u32(smem), static_cast<int>(threadIdx.x & 31),
               static_cast<int>(threadIdx.x >> 5) * 16, 0, static_cast<int>(blockIdx.x), 0, 0,
               false};
  if (threadIdx.x == 0)
    for (int p = 0; p < kStages; ++p) cta.produce(p);
  float acc0[2][32], acc1[2][32];
  for (int tile = blockIdx.x; tile < args.m_tiles; tile += gridDim.x) {
    const int m0 = tile * wg::BM;
    for (int q = 0; q < args.nseg; ++q) {
      if (args.seg[q].acc == 0) cta.run_seg(acc0, args.seg[q], m0);
      else cta.run_seg(acc1, args.seg[q], m0);
    }
  }
}

__global__ void __launch_bounds__(kHandoff, 1)
tower_fused_fwd_kernel(const __grid_constant__ FusedArgs args) {
  tower_fused_fwd<false>(args);
}

// tfr_mlp_fwd_tasks: the same kernel with task-major score planes (out_rows<true>).
__global__ void __launch_bounds__(kHandoff, 1)
tower_fused_fwd_tasks_kernel(const __grid_constant__ FusedArgs args) {
  tower_fused_fwd<true>(args);
}

// cuTensorMapEncodeTiled from the driver the runtime has loaded (no link dependency on it).
using EncodeTiled = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                 const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                 const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiled encode_tiled() {
  static EncodeTiled fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) !=
            cudaSuccess ||
        q != cudaDriverEntryPointSuccess) {
      (void)cudaGetLastError();
      p = nullptr;
    }
    return reinterpret_cast<EncodeTiled>(p);
  }();
  return fn;
}

// The map of a row-major fp32 [rows][cols] array (cols a multiple of 4, base 16-byte aligned):
// boxes of 32 columns x 128 rows, 128-byte swizzle, zero fill outside.
static bool encode_panels(CUtensorMap* m, const float* base, int cols, int rows) {
  const EncodeTiled fn = encode_tiled();
  if (!fn) return false;
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(cols) * 4};
  const cuuint32_t box[2] = {32, static_cast<cuuint32_t>(wg::BM)};
  const cuuint32_t elem[2] = {1, 1};
  return fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box,
            elem, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace fused

bool mlp_tc_fused_fwd_ok(int first_layer, const float* X, int M, const MlpPlan& p, int passes,
                         const float* ws) {
  const int L = p.n_dense - 1;
  if (passes != 3 || p.post() || p.input_bn) return false;
  if (p.activation != TFR_ACT_RELU && p.activation != TFR_ACT_NONE) return false;
  if (L - first_layer < 1 || p.dims[first_layer + 1] > 256 || p.dims[L] > 128) return false;
  for (int d = first_layer + 2; d <= L; ++d)
    if (p.dims[d] > 128) return false;
  if (p.dims[L + 1] > 8) return false;
  // the per-layer path reports these cases; TMA needs 16-byte aligned tensors
  return M >= 1 && (reinterpret_cast<uintptr_t>(X) & 15) == 0 &&
         (reinterpret_cast<uintptr_t>(ws) & 15) == 0;
}

int mlp_tc_fused_fwd(int first_layer, const float* X, int M, const MlpPlan& p,
                     const float* params, const uint8_t* mask, float* ws, float* scores,
                     cudaStream_t st, bool planar) {
  const int L = p.n_dense - 1, f = first_layer;
  fused::FusedArgs a{};
  TFR_REQUIRE(fused::encode_panels(&a.x, X, p.dims[f], M),
              "fused tower forward: cannot encode the TMA map of X");
  for (int d = f; d < L; ++d)
    TFR_REQUIRE(fused::encode_panels(&a.whi[d], ws + p.wthi_off + p.w_off[d], p.dims[d],
                                     p.dims[d + 1]) &&
                    fused::encode_panels(&a.wlo[d], ws + p.wtlo_off + p.w_off[d], p.dims[d],
                                         p.dims[d + 1]) &&
                    fused::encode_panels(&a.h[d], ws + p.act_off[d], p.dims[d + 1], M),
                "fused tower forward: cannot encode the TMA maps of layer %d", d);
  a.M = M; a.m_tiles = (M + wg::BM - 1) / wg::BM;
  a.act = p.activation;
  auto layer = [&](int d, int n0, int kb0, int nkb, int hoff, int acc, int zero, int epi) {
    fused::Seg& s = a.seg[a.nseg++];
    s.bias = params + p.b_off[d];
    s.bits = p.activation == TFR_ACT_RELU ? reinterpret_cast<uint32_t*>(ws + p.bits_off[d]) : nullptr;
    s.layer = d;
    s.K = p.dims[d]; s.N = p.dims[d + 1];
    s.n0 = n0; s.kb0 = kb0; s.nkb = nkb;
    s.a_x = d == f; s.hoff = hoff;
    s.acc = acc; s.zero = zero; s.epi = epi;
  };
  const int chunks = (p.dims[f + 1] + 127) / 128;
  for (int c = 0; c < chunks; ++c) {
    layer(f, 128 * c, 0, (p.dims[f] + 31) / 32, 0, 0, 1, 1);
    if (f + 1 < L) {   // Dense f + 1 over this chunk of its k range
      const int nkb = (p.dims[f + 1] + 31) / 32;
      layer(f + 1, 0, 4 * c, min(nkb, 4 * c + 4) - 4 * c, 128 * c, 1, c == 0, c == chunks - 1);
    }
  }
  for (int d = f + 2; d < L; ++d) layer(d, 0, 0, (p.dims[d] + 31) / 32, 0, 0, 1, 1);
  a.Wout = params + p.w_off[L]; a.bout = params + p.b_off[L];
  a.Kout = p.dims[L]; a.O = p.dims[L + 1];
  a.mask = mask; a.scores = scores;

  const int sms = num_sms();
  const int grid = a.m_tiles < sms ? a.m_tiles : sms;
  auto kernel = planar ? fused::tower_fused_fwd_tasks_kernel : fused::tower_fused_fwd_kernel;
  TFR_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   fused::kSmem));
  kernel<<<grid, fused::kHandoff, fused::kSmem, st>>>(a);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

}  // namespace tfr
