// K5/K6 fused 3xTF32 forward of the scorer tower: every hidden Dense layer from
// `first_layer` on, plus the output layer, in one persistent kernel.
//
// A CTA (two consumer warpgroups, one per SM) owns a 128-row tile of M at a time and walks
// the tower depth-first on it.  Only the first fused layer reads its A operand (X) from
// HBM, through the cp.async ring; every later layer takes its A fragments from Hbuf, a
// padded 128 x 128 fp32 tile in shared memory that the previous layer's epilogue wrote.  A
// first layer wider than 128 runs in two 128-column chunks, and the next layer consumes
// each chunk as soon as its epilogue has written it (k 0..127, then 128..255), its
// accumulator kept in registers meanwhile.  Each epilogue still stores H_d and the ReLU
// sign words to the workspace, as the backward reads them; the output layer then reads the
// last hidden layer from Hbuf.
//
// The k blocks of a tile form one linear sequence (config 2: 5 + 4 + 5 + 4 + 4 blocks), and
// the ring prefetches stages - 1 blocks ahead along it, across layer boundaries, epilogues
// and into the next tile.  A block always brings the layer's pre-split W^T hi / lo tile;
// blocks of the first layer also bring the X tile.
//
// Results are those of the per-layer path bit for bit: every output element sees the same
// wgmma shapes (m64n128, or m64n64 when the tile's live columns fit in 64), the same k-block
// order, the same skipped all-zero k steps and the same hi.hi, lo.hi, hi.lo pass order as
// wg::gemm_kernel, and the scores are summed in out_layer_fwd_kernel's order (per-lane fma
// chains over k = lane, lane + 32, ..., then warp_sum).
//
// Hbuf rows are private to a warp: the accumulator rows of warp w (16 w .. 16 w + 15) are
// the rows its A fragments read and the rows it scores, so Hbuf needs only __syncwarp.
#include "common.cuh"
#include "mlp.h"
#include "wgmma_gemm.cuh"

namespace tfr {
namespace fused {

constexpr int kStages = 3;
constexpr int kStage = wg::stage_bytes(3);                 // B hi + B lo + A: 51,200 B
constexpr int kAOff = 2 * wg::kTileBytes;
constexpr int kHPitch = 4 * (128 + 4);                     // 528 B: fragment loads conflict-free
constexpr int kHbufOff = kStages * kStage;
constexpr int kSmem = kStages * kStage + wg::BM * kHPitch + 1024;   // + alignment slack
static_assert(kSmem == 222208, "fused forward shared memory: 3 stages + Hbuf + slack");
static_assert(kSmem <= wg::kSmemLimit, "fused forward exceeds the shared memory of a CTA");
constexpr int kMaxSegs = 4 + TFR_MLP_MAX_LAYERS;

// A run of k blocks of one layer that accumulates into one accumulator.
struct Seg {
  const float* bhi; const float* blo;   // W_d^T hi / lo [N, K], K-major
  const float* bias;
  float* C;                             // H_d [M, N]
  uint32_t* bits;                       // ReLU sign words [(col / 32) * M + row], or null
  int K, N;
  int n0;                               // first output column (tile of 128)
  int kb0, nkb;                         // k blocks [kb0, kb0 + nkb) of the layer
  int a_x;                              // A is X, streamed through the ring; else Hbuf
  int hoff;                             // Hbuf column 0 is layer k index hoff
  int acc;                              // accumulator 0 or 1
  int zero, epi;                        // clear the accumulator first / run the epilogue after
};

struct FusedArgs {
  const float* X; int ldx;
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
    const uint64_t dbl = wg::desc_sw128(st + wg::kTileBytes + ks * 32);
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
  int s;            // stage of the block being consumed
  int p_tile, p_seg, p_kb, p_s;   // the block the next copy fetches, and its stage

  // Copies the next block of the sequence into its stage (nothing past the last tile) and
  // commits one cp.async group either way.
  __device__ __forceinline__ void produce() {
    if (p_tile < a.m_tiles) {
      const Seg& sg = a.seg[p_seg];
      const uint32_t st = sbase + p_s * kStage;
      const int k0 = (sg.kb0 + p_kb) * 32;
#pragma unroll
      for (int i = 0; i < 4; ++i) {   // W^T tile: [128 rows of n][8 chunks of k], swizzled
        const int c = threadIdx.x + i * wg::kThreads;
        const int r = c >> 3, kc = c & 7, k = k0 + kc * 4;
        const int n = (sg.n0 + r < sg.N && k < sg.K) ? min(4, sg.K - k) : 0;
        const size_t off = n > 0 ? static_cast<size_t>(sg.n0 + r) * sg.K + k : 0;
        wg::cp_async16(st + wg::swz_chunk(r, kc), sg.bhi + off, n * 4);
        wg::cp_async16(st + wg::kTileBytes + wg::swz_chunk(r, kc), sg.blo + off, n * 4);
      }
      if (sg.a_x) {
        const int m0 = p_tile * wg::BM;
#pragma unroll
        for (int i = 0; i < 4; ++i) {   // X tile: [128 rows of m][8 chunks of k], padded
          const int c = threadIdx.x + i * wg::kThreads;
          const int r = c >> 3, kc = c & 7, k = k0 + kc * 4;
          const int n = (m0 + r < a.M && k < sg.K) ? min(4, sg.K - k) : 0;
          const float* src = n > 0 ? a.X + static_cast<size_t>(m0 + r) * a.ldx + k : a.X;
          wg::cp_async16(st + kAOff + r * wg::kAPitchK + kc * 16, src, n * 4);
        }
      }
      if (++p_kb == sg.nkb) {
        p_kb = 0;
        if (++p_seg == a.nseg) {
          p_seg = 0;
          p_tile += gridDim.x;
        }
      }
    }
    wg::cp_async_commit();
    p_s = p_s + 1 == kStages ? 0 : p_s + 1;
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
      const uint32_t st = sbase + s * kStage;
      wg::cp_async_wait<kStages - 2>();
      wg::fence_proxy_async();   // cp.async writes -> visible to the tensor cores
      __syncthreads();
      // refill the stage of the previous block, whose MMAs every warpgroup retired
      produce();
      const int kg = (sg.kb0 + kb) * 32;   // first k of the block within the layer
      const int krem = sg.K - kg;
      const int ksteps = krem >= 32 ? 4 : (krem + 7) / 8;
      const unsigned char* sa =
          sg.a_x ? smem + s * kStage + kAOff : smem + kHbufOff + (kg - sg.hoff) * 4;
      const int pitch = sg.a_x ? wg::kAPitchK : kHPitch;
      // A fragments (m64 x k, per warp 16 rows): register i holds row g + 8 (i % 2),
      // k t + 4 (i / 2); split into hi / lo in registers
      uint32_t ahi[4][4], alo[4][4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int rr = wrow + g + 8 * (i & 1);
          const int k = ks * 8 + t + 4 * (i >> 1);
          const float x = *reinterpret_cast<const float*>(sa + rr * pitch + k * 4);
          const float h = wg::tf32_rn(x);
          ahi[ks][i] = __float_as_uint(h);
          alo[ks][i] = __float_as_uint(x - h);
        }
      if (two_n) mma_block_k<true>(acc, ahi, alo, st, ksteps);
      else mma_block_k<false>(acc, ahi, alo, st, ksteps);
      wg::wgmma_wait<0>();
      s = s + 1 == kStages ? 0 : s + 1;
    }
    if (sg.epi) epilogue(acc, sg, m0, two_n);
  }

  // bias / activation / sign words / H_d store as wg::gemm_kernel's EPI_BIAS_ACT, plus the
  // tile's columns into Hbuf (zero past N: the next layer's zero-filled k tail).
  __device__ __forceinline__ void epilogue(float (&acc)[2][32], const Seg& sg, int m0, bool two_n) {
    // accumulator element j of half h: row = lane / 4 + 8 ((j / 2) % 2),
    // column = 64 h + 8 (j / 4) + 2 (lane % 4) + j % 2
    const int rbase = m0 + wrow + (lane >> 2);
    const bool vec2 = (sg.N % 2) == 0 && (reinterpret_cast<uintptr_t>(sg.C) & 7u) == 0;
    float* hb = reinterpret_cast<float*>(smem + kHbufOff);
    __syncwarp();   // this warp's earlier Hbuf reads are done
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (h == 1 && !two_n) break;
#pragma unroll
      for (int c32 = 0; c32 < 2; ++c32) {   // 32-column chunks of this half
        const int chunk_col = sg.n0 + h * 64 + c32 * 32;
        if (chunk_col >= sg.N) break;
        uint32_t bits_out[2] = {0u, 0u};
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          const int j = c32 * 16 + jj;
          const int rr = (j >> 1) & 1;
          const int cin = 8 * (j >> 2) + 2 * (lane & 3) + (j & 1);
          const int col = sg.n0 + h * 64 + cin;
          const int row = rbase + 8 * rr;
          float x = acc[h][j];
          x += col < sg.N ? __ldg(sg.bias + col) : 0.f;
          if (a.act == TFR_ACT_RELU) x = fmaxf(x, 0.f);
          if (row >= a.M || col >= sg.N) x = 0.f;
          acc[h][j] = x;
          bits_out[rr] |= (x > 0.f ? 1u : 0u) << (cin & 31);
        }
        if (sg.bits) {
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            uint32_t w = bits_out[rr];
            w |= __shfl_xor_sync(0xffffffffu, w, 1);
            w |= __shfl_xor_sync(0xffffffffu, w, 2);
            const int row = rbase + 8 * rr;
            if ((lane & 3) == 0 && row < a.M)
              sg.bits[static_cast<size_t>(chunk_col >> 5) * a.M + row] = w;
          }
        }
      }
#pragma unroll
      for (int j = 0; j < 32; j += 2) {
        const int cin = h * 64 + 8 * (j >> 2) + 2 * (lane & 3);
        const int col = sg.n0 + cin;
        const int rl = wrow + (lane >> 2) + 8 * ((j >> 1) & 1);
        const int row = m0 + rl;
        const bool live = col < sg.N;
        *reinterpret_cast<float2*>(hb + rl * (kHPitch / 4) + cin) =
            make_float2(live ? acc[h][j] : 0.f, live && col + 1 < sg.N ? acc[h][j + 1] : 0.f);
        if (row >= a.M || !live) continue;
        const float x0 = acc[h][j], x1 = acc[h][j + 1];
        const bool both = col + 1 < sg.N;
        float* p = sg.C + static_cast<size_t>(row) * sg.N + col;
        if (both && vec2) {
          *reinterpret_cast<float2*>(p) = make_float2(x0, x1);
        } else {
          p[0] = x0;
          if (both) p[1] = x1;
        }
      }
    }
    __syncwarp();   // Hbuf written before any lane of the warp reads it
  }

  // scores of this warp's 16 rows from the last hidden layer in Hbuf, in
  // out_layer_fwd_kernel's order; RestoreList fill for masked rows
  __device__ __forceinline__ void out_layer(int m0) {
    const float* hb = reinterpret_cast<const float*>(smem + kHbufOff);
    for (int r0 = 0; r0 < 16; r0 += 4) {
      for (int o = 0; o < a.O; ++o) {
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        for (int k = lane; k < a.Kout; k += 32) {
          const float w = __ldg(a.Wout + static_cast<size_t>(k) * a.O + o);
#pragma unroll
          for (int r = 0; r < 4; ++r)
            acc[r] = fmaf(hb[(wrow + r0 + r) * (kHPitch / 4) + k], w, acc[r]);
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) acc[r] = warp_sum(acc[r]);
        const int row = m0 + wrow + r0 + lane;
        if (lane < 4 && row < a.M) {
          float v = (lane == 0 ? acc[0] : lane == 1 ? acc[1] : lane == 2 ? acc[2] : acc[3]) +
                    __ldg(a.bout + o);
          if (a.mask && a.O == 1 && !a.mask[row]) v = kLogEpsilon;
          a.scores[static_cast<size_t>(row) * a.O + o] = v;
        }
      }
    }
  }
};

__global__ void __launch_bounds__(wg::kThreads, 1)
tower_fused_fwd_kernel(const __grid_constant__ FusedArgs args) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (wg::smem_u32(smem_raw) & 1023u)) & 1023u);
  FusedCta cta{args, smem, wg::smem_u32(smem), static_cast<int>(threadIdx.x & 31),
               static_cast<int>(threadIdx.x >> 5) * 16, 0, static_cast<int>(blockIdx.x), 0, 0, 0};
  // cp.async groups: stages - 1 up front, then one per consumed block (empty past the end),
  // so a block's group is complete once at most stages - 2 younger groups are pending
  for (int p = 0; p < kStages - 1; ++p) cta.produce();
  float acc0[2][32], acc1[2][32];
  for (int tile = blockIdx.x; tile < args.m_tiles; tile += gridDim.x) {
    const int m0 = tile * wg::BM;
    for (int q = 0; q < args.nseg; ++q) {
      if (args.seg[q].acc == 0) cta.run_seg(acc0, args.seg[q], m0);
      else cta.run_seg(acc1, args.seg[q], m0);
    }
    cta.out_layer(m0);
  }
}

}  // namespace fused

bool mlp_tc_fused_fwd_ok(int first_layer, const float* X, int M, const MlpPlan& p, int passes) {
  const int L = p.n_dense - 1;
  if (passes != 3 || p.post() || p.input_bn) return false;
  if (p.activation != TFR_ACT_RELU && p.activation != TFR_ACT_NONE) return false;
  if (L - first_layer < 1 || p.dims[first_layer + 1] > 256 || p.dims[L] > 128) return false;
  for (int d = first_layer + 2; d <= L; ++d)
    if (p.dims[d] > 128) return false;
  if (p.dims[L + 1] > 8) return false;
  // the per-layer path reports these cases
  return M >= 1 && (reinterpret_cast<uintptr_t>(X) & 15) == 0;
}

int mlp_tc_fused_fwd(int first_layer, const float* X, int M, const MlpPlan& p,
                     const float* params, const uint8_t* mask, float* ws, float* scores,
                     cudaStream_t st) {
  const int L = p.n_dense - 1, f = first_layer;
  fused::FusedArgs a{};
  a.X = X; a.ldx = p.dims[f];
  a.M = M; a.m_tiles = (M + wg::BM - 1) / wg::BM;
  a.act = p.activation;
  auto layer = [&](int d, int n0, int kb0, int nkb, int hoff, int acc, int zero, int epi) {
    fused::Seg& s = a.seg[a.nseg++];
    s.bhi = ws + p.wthi_off + p.w_off[d];
    s.blo = ws + p.wtlo_off + p.w_off[d];
    s.bias = params + p.b_off[d];
    s.C = ws + p.act_off[d];
    s.bits = p.activation == TFR_ACT_RELU ? reinterpret_cast<uint32_t*>(ws + p.bits_off[d]) : nullptr;
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
  TFR_CUDA_OK(cudaFuncSetAttribute(fused::tower_fused_fwd_kernel,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, fused::kSmem));
  fused::tower_fused_fwd_kernel<<<grid, wg::kThreads, fused::kSmem, st>>>(a);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

}  // namespace tfr
