// K12: pooled embedding bags (tf.feature_column.embedding_column over a categorical column,
// feature_column.py `_safe_embedding_lookup_sparse` with combiner sum / mean / sqrtn; Keras
// Embedding followed by a reduction over the token axis, examples/keras/antique_kpl_din.py).
//
// Forward: one warp per bag; lane c accumulates column c (then c + 32, ...) over the bag's
// tokens in slot order, scales by the combiner and stores the pooled row rows_per_bag times.
//
// Backward, without float atomics (two identical calls give identical bits):
//   1. one warp per bag: g_r = scale_r * sum_k dout[r * rows_per_bag + k] (fixed k order), and
//      the (key, bag) pair of every slot, key = id for ids in [0, V), V otherwise
//   2. stable LSD radix sort of the pairs by key, 8 bits per pass: per-warp tile digit counts,
//      one exclusive scan over (digit, tile), then a stable scatter in which each warp ranks
//      its 32 items with __match_any_sync; every (id, bag) occurrence stays in bag order
//   3. segment bounds of every id from the sorted keys, then ceil(count / 128) chunks per id;
//      one warp sums one chunk's g rows in order into a partial row
//   4. one thread per table element adds its id's partials in chunk order
// An id present in every bag therefore spreads over R * T / 128 warps instead of one.
#include <utility>

#include "common.cuh"

namespace tfr {
namespace {

constexpr int kWarps = 8;               // warps per block of the warp-per-item kernels
constexpr int kTile = 8192;             // radix sort: items per warp tile
constexpr int kRadix = 256;             // 8 bits per pass
constexpr int kChunk = 128;             // occurrences per segment-sum chunk
constexpr int kMaxE = 1024;

__device__ __forceinline__ bool in_table(int id, int V) { return id >= 0 && id < V; }

__device__ __forceinline__ float combiner_scale(int combiner, int count) {
  if (count == 0) return 0.f;
  if (combiner == TFR_COMBINER_MEAN) return 1.f / static_cast<float>(count);
  if (combiner == TFR_COMBINER_SQRTN) return rsqrtf(static_cast<float>(count));
  return 1.f;
}

// Number of ids of bag `row` inside the table; counts the out-of-range ones into *bad.
__device__ __forceinline__ int bag_count(const int32_t* row, int T, int V, int* bad, int lane) {
  int count = 0, nbad = 0;
  for (int t0 = 0; t0 < T; t0 += 32) {
    const int t = t0 + lane;
    const int id = t < T ? row[t] : -1;
    count += __popc(__ballot_sync(0xffffffffu, in_table(id, V)));
    nbad += __popc(__ballot_sync(0xffffffffu, id < -1 || id >= V));
  }
  if (bad && nbad && lane == 0) atomicAdd(bad, nbad);
  return count;
}

__global__ void __launch_bounds__(kWarps * 32)
embed_fwd_kernel(const int32_t* __restrict__ ids, int R, int T, const float* __restrict__ table,
                 int V, int E, int combiner, int rpb, float* __restrict__ out, int ldo, int* bad) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (r >= R) return;
  const int32_t* row = ids + static_cast<size_t>(r) * T;
  const float scale = combiner_scale(combiner, bag_count(row, T, V, bad, lane));
  for (int c0 = 0; c0 < E; c0 += 32) {
    const int c = c0 + lane;
    float acc = 0.f;
    for (int t0 = 0; t0 < T; t0 += 32) {
      const int mine = t0 + lane < T ? row[t0 + lane] : -1;
      const int n = min(32, T - t0);
      for (int q = 0; q < n; ++q) {
        const int id = __shfl_sync(0xffffffffu, mine, q);
        if (in_table(id, V) && c < E) acc += __ldg(table + static_cast<size_t>(id) * E + c);
      }
    }
    if (c < E) {
      const float v = acc * scale;
      for (int k = 0; k < rpb; ++k) out[(static_cast<size_t>(r) * rpb + k) * ldo + c] = v;
    }
  }
}

// Step 1 of the backward: scaled per-bag gradient rows and the (key, bag) pairs.
__global__ void __launch_bounds__(kWarps * 32)
bag_grad_kernel(const int32_t* __restrict__ ids, int R, int T, const float* __restrict__ dout,
                int lddo, int rpb, int V, int E, int combiner, float* __restrict__ g,
                int32_t* __restrict__ keys, int32_t* __restrict__ vals, int* bad) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (r >= R) return;
  const int32_t* row = ids + static_cast<size_t>(r) * T;
  const float scale = combiner_scale(combiner, bag_count(row, T, V, bad, lane));
  for (int t = lane; t < T; t += 32) {
    const int id = row[t];
    keys[static_cast<size_t>(r) * T + t] = in_table(id, V) ? id : V;
    vals[static_cast<size_t>(r) * T + t] = r;
  }
  for (int c = lane; c < E; c += 32) {
    float s = 0.f;
    for (int k = 0; k < rpb; ++k) s += dout[(static_cast<size_t>(r) * rpb + k) * lddo + c];
    g[static_cast<size_t>(r) * E + c] = s * scale;
  }
}

// Radix pass, counting: hist[d * n_tiles + tile] = number of items of the warp's tile whose
// digit is d.
__global__ void __launch_bounds__(kWarps * 32)
radix_hist_kernel(const int32_t* __restrict__ keys, int n, int shift, int n_tiles,
                  int32_t* __restrict__ hist) {
  __shared__ int32_t cnt[kWarps][kRadix];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int tile = blockIdx.x * kWarps + w;
  for (int d = lane; d < kRadix; d += 32) cnt[w][d] = 0;
  __syncwarp();
  if (tile >= n_tiles) return;
  const int lo = tile * kTile, hi = min(lo + kTile, n);
  for (int base = lo; base < hi; base += 32) {
    const int i = base + lane;
    const int d = i < hi ? (keys[i] >> shift) & (kRadix - 1) : kRadix;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    if (d < kRadix && lane == 31 - __clz(peers)) cnt[w][d] += __popc(peers);
    __syncwarp();
  }
  for (int d = lane; d < kRadix; d += 32) hist[d * n_tiles + tile] = cnt[w][d];
}

// Radix pass, stable scatter: items of a tile keep their order among equal digits.
__global__ void __launch_bounds__(kWarps * 32)
radix_scatter_kernel(const int32_t* __restrict__ keys, const int32_t* __restrict__ vals, int n,
                     int shift, int n_tiles, const int32_t* __restrict__ offsets,
                     int32_t* __restrict__ keys_out, int32_t* __restrict__ vals_out) {
  __shared__ int32_t pos[kWarps][kRadix];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int tile = blockIdx.x * kWarps + w;
  if (tile >= n_tiles) return;
  for (int d = lane; d < kRadix; d += 32) pos[w][d] = offsets[d * n_tiles + tile];
  __syncwarp();
  const int lo = tile * kTile, hi = min(lo + kTile, n);
  const unsigned below = (1u << lane) - 1u;
  for (int base = lo; base < hi; base += 32) {
    const int i = base + lane;
    const int key = i < hi ? keys[i] : 0;
    const int d = i < hi ? (key >> shift) & (kRadix - 1) : kRadix;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    int p = 0;
    if (d < kRadix) p = pos[w][d] + __popc(peers & below);
    __syncwarp();
    if (d < kRadix) {
      keys_out[p] = key;
      vals_out[p] = vals[i];
      if (lane == 31 - __clz(peers)) pos[w][d] += __popc(peers);
    }
    __syncwarp();
  }
}

// In-place exclusive prefix sum of data[0, n) by one block.
__global__ void __launch_bounds__(1024) exclusive_scan_kernel(int32_t* data, int n) {
  __shared__ int32_t sums[1024];
  const int tid = threadIdx.x;
  const int per = (n + 1023) / 1024;
  const int lo = min(tid * per, n), hi = min(lo + per, n);
  int32_t s = 0;
  for (int i = lo; i < hi; ++i) s += data[i];
  sums[tid] = s;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {
    const int32_t v = tid >= off ? sums[tid - off] : 0;
    __syncthreads();
    sums[tid] += v;
    __syncthreads();
  }
  int32_t run = tid ? sums[tid - 1] : 0;
  for (int i = lo; i < hi; ++i) {
    const int32_t v = data[i];
    data[i] = run;
    run += v;
  }
}

// [start, end) of every id's run in the sorted keys (ids that never occur keep 0, 0).
__global__ void segment_bounds_kernel(const int32_t* __restrict__ keys, int n, int V,
                                      int32_t* __restrict__ start, int32_t* __restrict__ end) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int k = keys[i];
    if (k >= V) continue;
    if (i == 0 || keys[i - 1] != k) start[k] = i;
    if (i == n - 1 || keys[i + 1] != k) end[k] = i + 1;
  }
}

__global__ void chunk_count_kernel(const int32_t* __restrict__ start,
                                   const int32_t* __restrict__ end, int V,
                                   int32_t* __restrict__ chunks) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v <= V; v += gridDim.x * blockDim.x)
    chunks[v] = v < V ? (end[v] - start[v] + kChunk - 1) / kChunk : 0;
}

// One warp per chunk: partial[j] = sum of g[bag] over the chunk's occurrences, in order.
__global__ void __launch_bounds__(kWarps * 32)
chunk_sum_kernel(const int32_t* __restrict__ vals, const int32_t* __restrict__ start,
                 const int32_t* __restrict__ end, const int32_t* __restrict__ chunk_off, int V,
                 int max_chunks, const float* __restrict__ g, int E,
                 float* __restrict__ partial) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (j >= max_chunks || j >= chunk_off[V]) return;
  int lo = 0, hi = V - 1;               // the largest v with chunk_off[v] <= j
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (chunk_off[mid] <= j) lo = mid; else hi = mid - 1;
  }
  const int v = lo;
  const int begin = start[v] + (j - chunk_off[v]) * kChunk;
  const int stop = min(begin + kChunk, end[v]);
  for (int c0 = 0; c0 < E; c0 += 32) {
    const int c = c0 + lane;
    float acc = 0.f;
    for (int b0 = begin; b0 < stop; b0 += 32) {
      const int mine = b0 + lane < stop ? vals[b0 + lane] : 0;
      const int cnt = min(32, stop - b0);
      for (int q = 0; q < cnt; ++q) {
        const int r = __shfl_sync(0xffffffffu, mine, q);
        if (c < E) acc += g[static_cast<size_t>(r) * E + c];
      }
    }
    if (c < E) partial[static_cast<size_t>(j) * E + c] = acc;
  }
}

__global__ void table_grad_kernel(const int32_t* __restrict__ chunk_off,
                                  const float* __restrict__ partial, int V, int E,
                                  int accumulate, float* __restrict__ dtable) {
  const size_t total = static_cast<size_t>(V) * E;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i / E), c = static_cast<int>(i % E);
    float s = 0.f;
    for (int j = chunk_off[v]; j < chunk_off[v + 1]; ++j)
      s += partial[static_cast<size_t>(j) * E + c];
    dtable[i] = accumulate ? dtable[i] + s : s;
  }
}

struct EmbedWs {
  size_t g, keys_a, vals_a, keys_b, vals_b, hist, start, end, chunk_off, partial, total;
  int n_tiles, max_chunks;
};

size_t align_up(size_t x) { return (x + 255) & ~static_cast<size_t>(255); }

EmbedWs plan_ws(int R, int T, int V, int E) {
  EmbedWs w;
  const size_t ne = static_cast<size_t>(R) * T;
  w.n_tiles = static_cast<int>((ne + kTile - 1) / kTile);
  w.max_chunks = static_cast<int>((ne + kChunk - 1) / kChunk) + V;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += align_up(bytes); return o; };
  w.g = take(static_cast<size_t>(R) * E * 4);
  w.keys_a = take(ne * 4);
  w.vals_a = take(ne * 4);
  w.keys_b = take(ne * 4);
  w.vals_b = take(ne * 4);
  w.hist = take(static_cast<size_t>(kRadix) * w.n_tiles * 4);
  w.start = take(static_cast<size_t>(V) * 4);
  w.end = take(static_cast<size_t>(V) * 4);
  w.chunk_off = take((static_cast<size_t>(V) + 1) * 4);
  w.partial = take(static_cast<size_t>(w.max_chunks) * E * 4);
  w.total = off;
  return w;
}

int check_sizes(int R, int T, int V, int E, int rows_per_bag, int combiner) {
  TFR_REQUIRE(R >= 0 && T >= 1 && rows_per_bag >= 1, "embedding: bad sizes (R=%d T=%d "
              "rows_per_bag=%d)", R, T, rows_per_bag);
  TFR_REQUIRE(static_cast<long long>(R) * T < (1ll << 31) &&
                  static_cast<long long>(R) * rows_per_bag < (1ll << 31),
              "embedding: R * T = %lld exceeds the int32 index range",
              static_cast<long long>(R) * T);
  TFR_REQUIRE(V >= 1 && V < (1 << 30), "embedding: vocabulary size %d out of range", V);
  TFR_REQUIRE(E >= 1 && E <= kMaxE, "embedding: dimension %d must be in [1, %d]", E, kMaxE);
  TFR_REQUIRE(combiner >= TFR_COMBINER_SUM && combiner <= TFR_COMBINER_SQRTN,
              "embedding: combiner %d is not a tfr_combiner", combiner);
  return TFR_OK;
}

unsigned grid_of(long long items, int per_block) {
  return static_cast<unsigned>((items + per_block - 1) / per_block);
}

}  // namespace
}  // namespace tfr

using namespace tfr;

extern "C" size_t tfr_embedding_workspace_bytes(int R, int T, int V, int E) {
  if (check_sizes(R, T, V, E, 1, TFR_COMBINER_SUM)) return 0;
  return plan_ws(R, T, V, E).total;
}

extern "C" int tfr_embedding_fwd(const int32_t* ids, int R, int T, const float* table, int V,
                                 int E, int combiner, int rows_per_bag, float* out, int ldo,
                                 int* bad_ids, void* stream) {
  if (int rc = check_sizes(R, T, V, E, rows_per_bag, combiner)) return rc;
  TFR_REQUIRE(ids && table && out, "NULL argument");
  TFR_REQUIRE(ldo >= E, "ldo %d must be >= the embedding dimension %d", ldo, E);
  if (R == 0) return TFR_OK;
  embed_fwd_kernel<<<grid_of(R, kWarps), kWarps * 32, 0, (cudaStream_t)stream>>>(
      ids, R, T, table, V, E, combiner, rows_per_bag, out, ldo, bad_ids);
  TFR_LAUNCH_OK();
  return TFR_OK;
}

extern "C" int tfr_embedding_bwd(const int32_t* ids, int R, int T, const float* dout, int lddo,
                                 int rows_per_bag, int V, int E, int combiner, int accumulate,
                                 void* workspace, float* dtable, int* bad_ids, void* stream) {
  if (int rc = check_sizes(R, T, V, E, rows_per_bag, combiner)) return rc;
  TFR_REQUIRE(dtable && workspace && (R == 0 || (ids && dout)), "NULL argument");
  TFR_REQUIRE(lddo >= E, "lddo %d must be >= the embedding dimension %d", lddo, E);
  cudaStream_t st = (cudaStream_t)stream;
  if (R == 0) {
    if (!accumulate)
      TFR_CUDA_OK(cudaMemsetAsync(dtable, 0, static_cast<size_t>(V) * E * sizeof(float), st));
    return TFR_OK;
  }
  const EmbedWs w = plan_ws(R, T, V, E);
  char* base = static_cast<char*>(workspace);
  float* g = reinterpret_cast<float*>(base + w.g);
  int32_t* keys = reinterpret_cast<int32_t*>(base + w.keys_a);
  int32_t* vals = reinterpret_cast<int32_t*>(base + w.vals_a);
  int32_t* keys2 = reinterpret_cast<int32_t*>(base + w.keys_b);
  int32_t* vals2 = reinterpret_cast<int32_t*>(base + w.vals_b);
  int32_t* hist = reinterpret_cast<int32_t*>(base + w.hist);
  int32_t* start = reinterpret_cast<int32_t*>(base + w.start);
  int32_t* end = reinterpret_cast<int32_t*>(base + w.end);
  int32_t* chunk_off = reinterpret_cast<int32_t*>(base + w.chunk_off);
  float* partial = reinterpret_cast<float*>(base + w.partial);
  const int ne = R * T;

  bag_grad_kernel<<<grid_of(R, kWarps), kWarps * 32, 0, st>>>(
      ids, R, T, dout, lddo, rows_per_bag, V, E, combiner, g, keys, vals, bad_ids);
  TFR_LAUNCH_OK();
  int bits = 0;                         // keys lie in [0, V]
  while ((1ll << bits) <= V) ++bits;
  for (int shift = 0; shift < bits; shift += 8) {
    radix_hist_kernel<<<grid_of(w.n_tiles, kWarps), kWarps * 32, 0, st>>>(keys, ne, shift,
                                                                          w.n_tiles, hist);
    TFR_LAUNCH_OK();
    exclusive_scan_kernel<<<1, 1024, 0, st>>>(hist, kRadix * w.n_tiles);
    TFR_LAUNCH_OK();
    radix_scatter_kernel<<<grid_of(w.n_tiles, kWarps), kWarps * 32, 0, st>>>(
        keys, vals, ne, shift, w.n_tiles, hist, keys2, vals2);
    TFR_LAUNCH_OK();
    std::swap(keys, keys2);
    std::swap(vals, vals2);
  }
  TFR_CUDA_OK(cudaMemsetAsync(start, 0, static_cast<size_t>(V) * 4, st));
  TFR_CUDA_OK(cudaMemsetAsync(end, 0, static_cast<size_t>(V) * 4, st));
  const unsigned cap = 16u * static_cast<unsigned>(num_sms());
  segment_bounds_kernel<<<min(grid_of(ne, 256), cap), 256, 0, st>>>(keys, ne, V, start, end);
  TFR_LAUNCH_OK();
  chunk_count_kernel<<<min(grid_of(V + 1ll, 256), cap), 256, 0, st>>>(start, end, V, chunk_off);
  TFR_LAUNCH_OK();
  exclusive_scan_kernel<<<1, 1024, 0, st>>>(chunk_off, V + 1);
  TFR_LAUNCH_OK();
  chunk_sum_kernel<<<grid_of(w.max_chunks, kWarps), kWarps * 32, 0, st>>>(
      vals, start, end, chunk_off, V, w.max_chunks, g, E, partial);
  TFR_LAUNCH_OK();
  table_grad_kernel<<<min(grid_of(static_cast<long long>(V) * E, 256), cap), 256, 0, st>>>(
      chunk_off, partial, V, E, accumulate, dtable);
  TFR_LAUNCH_OK();
  return TFR_OK;
}
