// Fused 3xTF32 backward of the scorer tower's first Dense layer: dZ_0 and dW_0 in one
// persistent kernel, so that dZ_0 = (dZ_1 W_1^T) * relu'(H_0) never goes through HBM.
//
// It replaces the per-layer pair mlp_tc_dense_dgrad(d = 1) + mlp_tc_weight_grad(d = 0) of
// towers within mlp_tc_fused_bwd_ok, where dW_0 runs in the swapped orientation
// (dW_0^T = dZ_0^T X, dZ_0 the MN-major A operand) as one column tile of at most 136.  A work
// unit is one row split s of that GEMM (k blocks s * kb_per_split ..., the same split-K) times
// one 128-column half h of dZ_0; units 2 s and 2 s + 1 run on neighbouring CTAs of one wave,
// so the second half reads dZ_1 and X from L2.  Per 128-row tile of the split:
//   phase 1: acc = dZ_1[rows, :] W_1[half, :]^T, the dZ GEMM's k blocks (32 of dims[2]) in its
//            order, wgmma m64n128 (m64n64 when the half's live columns fit in 64), hi.hi,
//            lo.hi, hi.lo; then masked by H_0's sign words and zeroed past the split's rows and
//            dims[1], written to Dbuf and summed by column (db_0);
//   phase 2: accW += Dbuf^T X[rows, :], the dW GEMM's k blocks (32 rows) in its order, A
//            fragments from Dbuf, X^T from the ring, wgmma m64n136 / m64n128 / m64n64 as the
//            engine picks for dims[0], hi.hi, lo.hi, hi.lo.
// accW stays in registers over the split and is stored transposed into partial slot s, as the
// engine's split-K epilogue stores it; the column sums go to bias slot s.  mlp_reduce2 then
// sums both as before.  dZ_0, dW_0's partials and so dW_0 are bit-identical to the per-layer
// path (same shapes, k blocks, skipped zero k steps, operand splits and pass order); db_0 is
// summed in another order.
//
// Dbuf: the 128 x 128 fp32 dZ_0 tile, [row][column] with rows padded to 136 floats: the float2
// accumulator stores of a half warp and the MN-major A fragment loads of a warp (row = k,
// column = m, as the engine's MN-major A tile of pitch kAPitchMN) both hit 32 different banks.
//
// Threads 0-255 are the two MMA warpgroups (setmaxnreg 208); threads 256-383 the producer
// warpgroup (88), which runs one stage ring of kStages stages for both phases: a phase-1 block
// brings the dZ_1 tile (K-major, pitch kAPitchK) and W_1's rows of the half, pre-split hi / lo
// (K-major, swizzled); a phase-2 block brings X's 32-row slab, transposed and split in place
// as the dW GEMMs' producer does (wg::copy_slab, wg::transpose_slab).  The ring's mbarriers are
// the engine's: full[s] (one arrival per producer warp), empty[s] (one per MMA warp).
#include "common.cuh"
#include "mlp.h"
#include "wgmma_gemm.cuh"

namespace tfr {
namespace fused_bwd {

constexpr int kStages = 3;
constexpr int kBLo1 = wg::kTileBytes;            // phase 1: W_1 hi at 0, lo here
constexpr int kAOff = 2 * wg::kTileBytes;        //          dZ_1 tile here
constexpr int kBLo2 = wg::b_tile_bytes(true);    // phase 2: X^T hi at 0 (136 rows), lo here
constexpr int kStage = kAOff + wg::kATileBytes;  // 50 KB
static_assert(2 * kBLo2 <= kStage, "a phase-2 block fits in a stage");
constexpr int kBufPitch = wg::kAPitchMN / 4;     // floats per Dbuf row
constexpr int kBufOff = kStages * kStage;
constexpr int kSumOff = kBufOff + wg::BM * kBufPitch * 4;   // [8 warps][128] column sums
constexpr int kBarOff = kSumOff + wg::kWarps * wg::BN * 4;  // full[kStages], empty[kStages]
constexpr int kSmem = kBarOff + 2 * kStages * 8 + 1024;     // + alignment slack
static_assert(kSmem == 228400, "fused dW_0 shared memory: 3 stages + Dbuf + column sums + barriers + slack");
static_assert(kSmem <= wg::kSmemLimit, "fused dW_0 exceeds the shared memory of a CTA");
constexpr int kThreads = wg::kThreads + wg::kEpiThreads;

struct Dw0Args {
  const float* X;          // [M, N0]: what Dense 0 consumed
  const float* dz1;        // dZ_1 [M, N2]
  const float* whi;        // W_1 [N1, N2], pre-split hi / lo
  const float* wlo;
  const uint32_t* bits;    // H_0's ReLU sign words [(col / 32) * M + row], or null (no mask)
  float* partial; size_t pstride;   // dW_0 partial slot s: [N0][N1] at partial + s * pstride
  float* bsum; size_t bstride;      // db_0 bias slot s: [N1] at bsum + s * bstride
  int M, N0, N1, N2;
  int nkb, kb_per_split;   // 32-row k blocks of M, and per split (as wg::launch_grid)
  int halves, units;
};

struct Unit {
  int split, half, kb0, kb_end;   // k blocks [kb0, kb_end) of M; none when kb_end <= kb0
};
__device__ __forceinline__ Unit unit_of(const Dw0Args& a, int u) {
  Unit r;
  r.split = u / a.halves;
  r.half = u - r.split * a.halves;
  r.kb0 = r.split * a.kb_per_split;
  r.kb_end = min(a.nkb, r.kb0 + a.kb_per_split);
  return r;
}

// The producer warpgroup: walks the (unit, tile, block) sequence of the MMA warps.  Block g
// goes to stage g mod kStages; its copies are finished (landed, X transposed, full[s]) just
// before block g + 2 is issued, so two blocks' copies run while the MMA warps take the one
// before them.
template <bool FOLD>
__device__ __forceinline__ void producer(const Dw0Args& a, unsigned char* smem, uint64_t* full,
                                         uint64_t* empty) {
  const int pt = threadIdx.x - wg::kThreads;
  const uint32_t sbase = wg::smem_u32(smem);
  const int nkb1 = (a.N2 + 31) / 32;
  const int tail = FOLD ? a.N0 - wg::BN : 0;
  int is = 0, fs = 0;
  uint32_t eph = 1;     // parity of the empty phase the issue waits for
  int pending = 0;      // blocks issued but not finished (at most 2)
  uint32_t slabs = 0;   // bit i: the i-th oldest pending block is an X slab
  // finishes the oldest pending block; `younger`: cp.async groups committed after its own
  auto finish = [&](int younger) {
    if (younger > 0) wg::cp_async_wait<1>();
    else wg::cp_async_wait<0>();
    wg::bar_sync(wg::kBarProd, wg::kEpiThreads);   // the copies of every producer thread have landed
    if (slabs & 1u) {
      unsigned char* sb = smem + fs * kStage;
      wg::transpose_slab<true, FOLD>(sb, sb + kBLo2, pt);
    }
    wg::fence_proxy_async();   // cp.async and st.shared writes -> visible to the tensor cores
    __syncwarp();
    if ((pt & 31) == 0) wg::mbar_arrive(full + fs);
    fs = fs + 1 == kStages ? 0 : fs + 1;
    slabs >>= 1;
    --pending;
  };
  // Two blocks' copies stay in flight.  The MMA warps hold at most two stages, the block they
  // take and the one whose wgmma group may still run, and release the older once the block
  // after it is full, so the wait for an empty stage never waits on an unfinished block.
  auto begin = [&] {
    if (pending == 2) finish(1);
    wg::mbar_wait(empty + is, eph);
    return sbase + is * kStage;
  };
  auto end = [&](bool x) {
    wg::cp_async_commit();
    if (++is == kStages) {
      is = 0;
      eph ^= 1u;
    }
    slabs |= static_cast<uint32_t>(x) << pending;
    ++pending;
  };
  for (int u = blockIdx.x; u < a.units; u += gridDim.x) {
    const Unit un = unit_of(a, u);
    const int rend = min(a.M, un.kb_end * 32);
    const int n0 = wg::BN * un.half;
    for (int kt = un.kb0; kt < un.kb_end; kt += 4) {
      const int m0 = kt * 32;
      for (int j = 0; j < nkb1; ++j) {
        const uint32_t st = begin();
        // [128 rows][8 chunks of k] of dZ_1 and of W_1 hi / lo: a thread's chunk kc and its rows'
        // swizzle phase (row mod 8) are the same for all 8 of its rows, 16 apart, so every
        // address steps by a constant and the copies go out four at a time (eight spill)
        const int r0 = pt >> 3, kc = pt & 7, k = 32 * j + kc * 4;   // N2 is a multiple of 4
        const bool kin = k < a.N2;
        const size_t rstep = static_cast<size_t>(16) * a.N2;
        const float* pa = a.dz1 + static_cast<size_t>(m0 + r0) * a.N2 + k;
        const size_t wo = static_cast<size_t>(n0 + r0) * a.N2 + k;
        const uint32_t da = st + kAOff + r0 * wg::kAPitchK + kc * 16;
        const uint32_t db = st + wg::swz_chunk(r0, kc);
#pragma unroll 4
        for (int i = 0; i < 8; ++i) {
          const int na = kin && m0 + r0 + 16 * i < rend ? 16 : 0;
          const int nb = kin && n0 + r0 + 16 * i < a.N1 ? 16 : 0;
          wg::cp_async16(da + i * 16 * wg::kAPitchK, na ? pa + i * rstep : a.dz1, na);
          wg::cp_async16(db + i * 16 * 128, nb ? a.whi + wo + i * rstep : a.whi, nb);
          wg::cp_async16(db + kBLo1 + i * 16 * 128, nb ? a.wlo + wo + i * rstep : a.wlo, nb);
        }
        end(false);
      }
      const int cnt = min(4, un.kb_end - kt);
      for (int j = 0; j < cnt; ++j) {
        const uint32_t st = begin();
        wg::copy_slab<FOLD>(a.X, a.N0, a.M, a.N0, st, 0, m0 + 32 * j, tail, pt);
        end(true);
      }
    }
  }
  while (pending > 0) finish(pending - 1);
}

// One wgmma group over a block: NK k steps, each hi.hi, lo.hi, hi.lo (as wg::gemm_kernel),
// B hi at st and lo at st + LO.  N: 136 (acc, then the folded columns into acc_t), 128 or 64.
template <int N, int NK, int LO, int KS>
__device__ __forceinline__ void mma_group(float (&acc)[2][32], float (&acc_t)[4],
                                          uint32_t (&ahi)[KS][4], uint32_t (&alo)[KS][4],
                                          uint32_t st) {
  // the fragments are final before the fence (as in wg::gemm_kernel)
#pragma unroll
  for (int ks = 0; ks < KS; ++ks)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      asm volatile("" : "+r"(ahi[ks][i]));
      asm volatile("" : "+r"(alo[ks][i]));
    }
  wg::wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < NK; ++ks) {
    const uint64_t dbh = wg::desc_sw128(st + ks * 32);
    const uint64_t dbl = wg::desc_sw128(st + LO + ks * 32);
    if constexpr (N == 136) {
      wg::mma_tf32_n136(acc, acc_t, ahi[ks], dbh);
      wg::mma_tf32_n136(acc, acc_t, alo[ks], dbh);
      wg::mma_tf32_n136(acc, acc_t, ahi[ks], dbl);
    } else if constexpr (N == 128) {
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
// the first min(ksteps, KS) k steps: those not wholly past K
template <int N, int LO, int KS>
__device__ __forceinline__ void mma_group_k(float (&acc)[2][32], float (&acc_t)[4],
                                            uint32_t (&ahi)[KS][4], uint32_t (&alo)[KS][4],
                                            uint32_t st, int ksteps) {
  if (KS == 4 && ksteps >= 4) mma_group<N, KS == 4 ? 4 : 1, LO>(acc, acc_t, ahi, alo, st);
  else if (KS == 4 && ksteps == 3) mma_group<N, KS == 4 ? 3 : 1, LO>(acc, acc_t, ahi, alo, st);
  else if (KS >= 2 && ksteps >= 2) mma_group<N, KS >= 2 ? 2 : 1, LO>(acc, acc_t, ahi, alo, st);
  else mma_group<N, 1, LO>(acc, acc_t, ahi, alo, st);
}

// The two MMA warpgroups.  NW: the dW_0 wgmma width, 136 / 128 / 64 (wg::launch's choice for
// GN = dims[0]).
template <int NW>
__device__ __forceinline__ void mma_warps(const Dw0Args& a, unsigned char* smem, uint64_t* full,
                                          uint64_t* empty) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int row = (warp >> 2) * 64 + (warp & 3) * 16 + g;   // fragment / accumulator row
  const uint32_t sbase = wg::smem_u32(smem);
  float* buf = reinterpret_cast<float*>(smem + kBufOff);
  float* sums = reinterpret_cast<float*>(smem + kSumOff) + warp * wg::BN;   // this warp's
  const int nkb1 = (a.N2 + 31) / 32;
  int s = 0;          // stage of the next block
  uint32_t fph = 0;   // parity of its full phase
  int held = -1;      // the stage of the last block issued, whose last group may still run
  auto release = [&](int stage) {   // each MMA warp arrives for itself (wait_group is warp-wide)
    if (lane == 0) wg::mbar_arrive(empty + stage);
  };
  auto advance = [&] {
    if (++s == kStages) {
      s = 0;
      fph ^= 1u;
    }
  };
  // A fragment register i of k step ks0 + ks: row + 8 (i % 2), k 8 (ks0 + ks) + t + 4 (i / 2),
  // split hi / lo
  auto frags = [&](auto& ahi, auto& alo, int ks0, auto at) {
    constexpr int KS = sizeof(ahi) / sizeof(ahi[0]);
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float x = at(row + 8 * (i & 1), (ks0 + ks) * 8 + t + 4 * (i >> 1));
        const float h = wg::tf32_rn(x);
        ahi[ks][i] = __float_as_uint(h);
        alo[ks][i] = __float_as_uint(x - h);
      }
  };

  float accw[2][32], accw_t[4];
  for (int u = blockIdx.x; u < a.units; u += gridDim.x) {
    const Unit un = unit_of(a, u);
    const int rend = min(a.M, un.kb_end * 32);
    const int n0 = wg::BN * un.half;
    const bool two_n = n0 + 64 < a.N1;   // the second 64 columns of the half hold live columns
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 32; ++j) accw[h][j] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) accw_t[j] = 0.f;
    for (int c = lane; c < wg::BN; c += 32) sums[c] = 0.f;

    for (int kt = un.kb0; kt < un.kb_end; kt += 4) {
      const int m0 = kt * 32;
      // ---- phase 1: the dZ_0 half tile, one wgmma group of two k steps at a time.  Its
      // accumulator lives beside accW; with a group in flight here as well as in phase 2,
      // ptxas serialises the wgmmas.
      float acc[2][32];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[h][j] = 0.f;
      for (int j = 0; j < nkb1; ++j) {
        const int krem = a.N2 - 32 * j;
        const int ksteps = krem >= 32 ? 4 : (krem + 7) / 8;
        const unsigned char* sa = smem + s * kStage + kAOff;
        wg::mbar_wait(full + s, fph);
        for (int ks0 = 0; ks0 < ksteps; ks0 += 2) {
          uint32_t ahi[2][4], alo[2][4];
          frags(ahi, alo, ks0, [&](int r, int k) {
            return *reinterpret_cast<const float*>(sa + r * wg::kAPitchK + k * 4);
          });
          const uint32_t st = sbase + s * kStage + ks0 * 32;
          if (two_n) mma_group_k<128, kBLo1>(acc, accw_t, ahi, alo, st, ksteps - ks0);
          else mma_group_k<64, kBLo1>(acc, accw_t, ahi, alo, st, ksteps - ks0);
          wg::wgmma_wait<0>();
        }
        release(s);
        advance();
      }
      // ---- the mask epilogue into Dbuf: accumulator element j of half h is tile row
      // row + 8 ((j / 2) % 2), column 64 h + 8 (j / 4) + 2 t + j % 2
      wg::bar_sync(wg::kBarMma, wg::kThreads);   // every warp is done reading the last Dbuf
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int c32 = 0; c32 < 2; ++c32) {
          const int chunk_col = n0 + h * 64 + c32 * 32;
          uint32_t keep[2];
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const int r = m0 + row + 8 * rr;
            keep[rr] = r >= rend || chunk_col >= a.N1 ? 0u
                       : a.bits ? __ldg(a.bits + static_cast<size_t>(chunk_col >> 5) * a.M + r)
                                : ~0u;
          }
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) {
            const int j = c32 * 16 + jj;
            const int cin = 8 * (j >> 2) + 2 * t + (j & 1);   // column within the 64
            const bool on = (keep[(j >> 1) & 1] >> (cin & 31)) & 1u && chunk_col + (cin & 31) < a.N1;
            acc[h][j] = on ? acc[h][j] : 0.f;
          }
        }
#pragma unroll
        for (int j = 0; j < 32; j += 2) {
          const int col = h * 64 + 8 * (j >> 2) + 2 * t;
          const int rl = row + 8 * ((j >> 1) & 1);
          *reinterpret_cast<float2*>(buf + rl * kBufPitch + col) = make_float2(acc[h][j], acc[h][j + 1]);
        }
        // column sums of this warp's 16 rows: over the 8 lanes that share t
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          float s0 = acc[h][j] + acc[h][j + 2], s1 = acc[h][j + 1] + acc[h][j + 3];
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            s0 += __shfl_xor_sync(0xffffffffu, s0, o);
            s1 += __shfl_xor_sync(0xffffffffu, s1, o);
          }
          if (lane < 4) {
            const int col = h * 64 + 8 * (j >> 2) + 2 * t;
            sums[col] += s0;
            sums[col + 1] += s1;
          }
        }
      }
      wg::bar_sync(wg::kBarMma, wg::kThreads);   // Dbuf is whole
      // ---- phase 2: accW += Dbuf^T X over the tile's k blocks, in wgmma groups of two k
      // steps, one in flight while the next one's fragments load (two sets of 16 registers)
      const int cnt = min(4, un.kb_end - kt);
      for (int j = 0; j < cnt; ++j) {
        const int krem = a.M - (kt + j) * 32;
        const int ksteps = krem >= 32 ? 4 : (krem + 7) / 8;
        const uint32_t st = sbase + s * kStage;
        wg::mbar_wait(full + s, fph);
        uint32_t ahi[2][2][4], alo[2][2][4];
        auto half_block = [&](int ks0, auto set) {
          constexpr int F = decltype(set)::value;
          frags(ahi[F], alo[F], ks0, [&](int r, int k) { return buf[(32 * j + k) * kBufPitch + r]; });
          mma_group_k<NW, kBLo2>(accw, accw_t, ahi[F], alo[F], st + ks0 * 32, ksteps - ks0);
          wg::wgmma_wait<1>();
          if (ks0 == 0 && held >= 0) release(held);
        };
        half_block(0, std::integral_constant<int, 0>{});
        if (ksteps > 2) half_block(2, std::integral_constant<int, 1>{});
        held = s;
        advance();
      }
      wg::wgmma_wait<0>();
      if (held >= 0) release(held);
      held = -1;
    }

    // ---- the unit's results: accW transposed into partial slot s (element (m, n) of dW_0^T,
    // m a dZ_0 column, n an X column, at partial[n * N1 + m]), column sums into bias slot s
    float* P = a.partial + static_cast<size_t>(un.split) * a.pstride;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int m = n0 + row + 8 * ((j >> 1) & 1);
        const int n = h * 64 + 8 * (j >> 2) + 2 * t + (j & 1);
        if (m < a.N1 && n < a.N0) P[static_cast<size_t>(n) * a.N1 + m] = accw[h][j];
      }
    }
    if (NW == 136) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int m = n0 + row + 8 * (j >> 1);
        const int n = wg::BN + 2 * t + (j & 1);
        if (m < a.N1 && n < a.N0) P[static_cast<size_t>(n) * a.N1 + m] = accw_t[j];
      }
    }
    wg::bar_sync(wg::kBarMma, wg::kThreads);   // every warp's column sums are in
    if (threadIdx.x < wg::BN && n0 + static_cast<int>(threadIdx.x) < a.N1) {
      const float* sp = reinterpret_cast<const float*>(smem + kSumOff) + threadIdx.x;
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < wg::kWarps; ++w) v += sp[w * wg::BN];
      a.bsum[static_cast<size_t>(un.split) * a.bstride + n0 + threadIdx.x] = v;
    }
    wg::bar_sync(wg::kBarMma, wg::kThreads);   // ... and read before the next unit clears them
  }
}

template <int NW>
__global__ void __launch_bounds__(kThreads, 1)
tower_fused_dw0_kernel(const __grid_constant__ Dw0Args args) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (wg::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kBarOff);
  uint64_t* empty = full + kStages;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      wg::mbar_init(full + i, wg::kEpiThreads / 32);
      wg::mbar_init(empty + i, wg::kWarps);
    }
  }
  __syncthreads();
  if (threadIdx.x >= wg::kThreads) {
    wg::setmaxnreg_dec<wg::kEpiRegs>();
    producer<NW == 136>(args, smem, full, empty);
    return;
  }
  wg::setmaxnreg_inc<wg::kMmaRegs>();
  mma_warps<NW>(args, smem, full, empty);
}

}  // namespace fused_bwd

int mlp_tc_fused_dw0(const float* X, const float* dz1, int M, const MlpPlan& p, float* ws,
                     cudaStream_t st) {
  TFR_REQUIRE((reinterpret_cast<uintptr_t>(X) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(dz1) & 15) == 0,
              "tc gemm: operands must be 16-byte aligned");
  fused_bwd::Dw0Args a{};
  a.X = X; a.dz1 = dz1;
  a.whi = ws + p.whi_off + p.w_off[1];
  a.wlo = ws + p.wlo_off + p.w_off[1];
  a.bits = p.activation == TFR_ACT_RELU ? reinterpret_cast<const uint32_t*>(ws + p.bits_off[0])
                                        : nullptr;
  a.partial = ws + p.partial_off; a.pstride = p.partial_stride;
  a.bsum = ws + p.tile_off; a.bstride = p.tile_stride;
  a.M = M; a.N0 = p.dims[0]; a.N1 = p.dims[1]; a.N2 = p.dims[2];
  a.nkb = (M + 31) / 32;
  a.kb_per_split = (a.nkb + p.splits - 1) / p.splits;   // wg::launch_grid's split of the k range
  a.halves = (p.dims[1] + wg::BN - 1) / wg::BN;
  a.units = p.splits * a.halves;
  const int sms = num_sms();
  const int grid = a.units < sms ? a.units : sms;
  // the dW_0 width wg::launch takes for GN = dims[0] (it folds 129..136)
  auto kernel = a.N0 > wg::BN ? fused_bwd::tower_fused_dw0_kernel<136>
                : a.N0 > 64   ? fused_bwd::tower_fused_dw0_kernel<128>
                              : fused_bwd::tower_fused_dw0_kernel<64>;
  TFR_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   fused_bwd::kSmem));
  kernel<<<grid, fused_bwd::kThreads, fused_bwd::kSmem, st>>>(a);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

}  // namespace tfr
