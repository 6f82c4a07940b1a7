// radix_sort.cuh -- the stable LSD radix sort of 64-bit keys with a u32 row payload, and the scan of the sorted keys'
// heads (hand-written CUDA for sm_90a).  Shared by libtloam_b200_gmm.so (map_merge.cu, the merged map's voxels),
// libtloam_b200_loc.so (localize.cu, the prior map's cells), libtloam_b200_mapu.so (map_update.cu) and
// libtloam_b200_frontier.so (frontier.cu, each frontier's cells), so that all order rows by the same rule:
//   k_gmm_hist     \
//   k_gmm_offsets   |   one pass per 8-bit digit: per-tile digit counts, per-digit offsets, a stable scatter; rows with
//   k_gmm_scatter  /    equal keys stay in row order
//   k_gmm_head_count \  the positions whose key differs from the previous one, numbered in order: the j-th distinct
//   k_gmm_head_scatter/ key's first position at start[j], their count in st->n_vox and start[count] = n
// The kernels keep the names the merge gave them.  This header is included by those libraries only; including it in
// libtloam_b200.so would add its kernels there.
#pragma once
#include <cuda_runtime.h>

#include "map_merge.h"

namespace tloam {

constexpr unsigned kGmmT = 256;
constexpr unsigned kGmmItems = 8;                          // rows per thread of a radix tile
constexpr unsigned kGmmTile = kGmmT * kGmmItems;           // rows per block of the radix sort
constexpr unsigned kGmmMaxBlocks = 1024;                   // blocks of the head scan

static inline unsigned gmm_tiles(unsigned long long n) { return (unsigned)((n + kGmmTile - 1) / kGmmTile); }

// per-tile counts of digit (key >> sh) & 255 at hist[digit * tiles + tile]
__global__ void __launch_bounds__(kGmmT) k_gmm_hist(const unsigned long long* key, unsigned long long n, int sh,
                                                    unsigned* hist, unsigned tiles) {
  __shared__ unsigned s_h[256];
  const unsigned t = threadIdx.x, lane = t & 31u;
  s_h[t] = 0u;
  __syncthreads();
  const unsigned long long base = (unsigned long long)blockIdx.x * kGmmTile;
  for (unsigned q = 0; q < kGmmItems; ++q) {
    const unsigned long long i = base + q * kGmmT + t;
    const unsigned d = i < n ? (unsigned)(key[i] >> sh) & 255u : 256u;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    if (d < 256u && (peers & ((1u << lane) - 1u)) == 0u) atomicAdd(&s_h[d], (unsigned)__popc(peers));
  }
  __syncthreads();
  hist[(size_t)t * tiles + blockIdx.x] = s_h[t];
}

// the exclusive scan of a block's values in thread order, and their total
__device__ __forceinline__ unsigned gmm_block_scan(unsigned v, unsigned* total) {
  __shared__ unsigned s_w[kGmmT / 32];
  const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  unsigned inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= (unsigned)o) inc += u;
  }
  __syncthreads();
  if (lane == 31u) s_w[warp] = inc;
  __syncthreads();
  unsigned before = 0u, all = 0u;
#pragma unroll
  for (unsigned w = 0; w < kGmmT / 32; ++w) {
    before += w < warp ? s_w[w] : 0u;
    all += s_w[w];
  }
  *total = all;
  return before + inc - v;
}

// block d: the exclusive offsets of digit d's tiles within the digit, and the digit's total
__global__ void __launch_bounds__(kGmmT) k_gmm_offsets(unsigned* hist, unsigned tiles, unsigned* totals) {
  unsigned* row = hist + (size_t)blockIdx.x * tiles;
  unsigned run = 0u;
  for (unsigned b0 = 0; b0 < tiles; b0 += kGmmT) {
    const unsigned b = b0 + threadIdx.x;
    const unsigned c = b < tiles ? row[b] : 0u;
    unsigned chunk;
    const unsigned ex = gmm_block_scan(c, &chunk);
    if (b < tiles) row[b] = run + ex;
    run += chunk;
  }
  if (threadIdx.x == 0) totals[blockIdx.x] = run;
}

// stable scatter by digit: a tile's rows go in row order to the digit's base + the tile's offset (within a warp by lane,
// across warps by a per-digit prefix, across the tile's sub-tiles by a running offset)
__global__ void __launch_bounds__(kGmmT) k_gmm_scatter(const unsigned long long* key_in, const unsigned* row_in,
                                                       unsigned long long n, int sh, const unsigned* hist, unsigned tiles,
                                                       const unsigned* totals, unsigned long long* key_out,
                                                       unsigned* row_out) {
  __shared__ unsigned s_off[256];
  __shared__ unsigned s_w[kGmmT / 32][256];
  const unsigned t = threadIdx.x, lane = t & 31u, warp = t >> 5;
  unsigned all;
  const unsigned digit_base = gmm_block_scan(totals[t], &all);
  s_off[t] = digit_base + hist[(size_t)t * tiles + blockIdx.x];
  const unsigned long long base = (unsigned long long)blockIdx.x * kGmmTile;
  for (unsigned q = 0; q < kGmmItems; ++q) {
#pragma unroll
    for (unsigned w = 0; w < kGmmT / 32; ++w) s_w[w][t] = 0u;
    __syncthreads();
    const unsigned long long i = base + q * kGmmT + t;
    const bool ok = i < n;
    unsigned long long k = 0ull;
    unsigned r = 0u, d = 256u;
    if (ok) { k = key_in[i]; r = row_in[i]; d = (unsigned)(k >> sh) & 255u; }
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const unsigned rank = __popc(peers & ((1u << lane) - 1u));
    if (ok && rank == 0u) s_w[warp][d] = __popc(peers);
    __syncthreads();
    unsigned run = s_off[t];
#pragma unroll
    for (unsigned w = 0; w < kGmmT / 32; ++w) { const unsigned c = s_w[w][t]; s_w[w][t] = run; run += c; }
    s_off[t] = run;
    __syncthreads();
    if (ok) {
      const unsigned pos = s_w[warp][d] + rank;
      key_out[pos] = k;
      row_out[pos] = r;
    }
    __syncthreads();
  }
}

__device__ __forceinline__ bool gmm_head(const unsigned long long* key, unsigned long long p) {
  return p == 0ull || key[p] != key[p - 1];
}

// the sum of one value per thread, the same for every thread of the block
__device__ __forceinline__ unsigned gmm_block_sum(unsigned v) {
  unsigned all;
  gmm_block_scan(v, &all);
  return all;
}

// block b: the heads among sorted positions [b chunk, (b + 1) chunk) of the n_sel selected ones
__global__ void __launch_bounds__(kGmmT) k_gmm_head_count(const unsigned long long* key, unsigned long long n_sel,
                                                          unsigned long long chunk, unsigned* block_counts) {
  const unsigned long long lo = blockIdx.x * chunk, hi = lo + chunk < n_sel ? lo + chunk : n_sel;
  unsigned c = 0u;
  for (unsigned long long p = lo + threadIdx.x; p < hi; p += kGmmT) c += gmm_head(key, p) ? 1u : 0u;
  c = gmm_block_sum(c);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = c;
}

// block b: its base = the heads of blocks 0 .. b - 1, then its chunk tile by tile: the j-th head's position at start[j].
// The last block writes the voxel count and start[n_vox] = n_sel.
__global__ void __launch_bounds__(kGmmT) k_gmm_head_scatter(const unsigned long long* key, unsigned long long n_sel,
                                                            unsigned long long chunk, const unsigned* block_counts,
                                                            unsigned* start, tloam_gmm_state* st) {
  __shared__ unsigned warp_n[kGmmT / 32];
  unsigned before = 0u;
  for (unsigned k = threadIdx.x; k < blockIdx.x; k += kGmmT) before += block_counts[k];
  unsigned base = gmm_block_sum(before);
  const unsigned long long lo = blockIdx.x * chunk, hi = lo + chunk < n_sel ? lo + chunk : n_sel;
  const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  for (unsigned long long t = lo; t < hi; t += kGmmT) {
    const unsigned long long p = t + threadIdx.x;
    const bool head = p < hi && gmm_head(key, p);
    const unsigned ballot = __ballot_sync(0xffffffffu, head);
    if (lane == 0) warp_n[warp] = __popc(ballot);
    __syncthreads();
    unsigned off = 0u, tile = 0u;
    for (unsigned w = 0; w < kGmmT / 32; ++w) {
      off += w < warp ? warp_n[w] : 0u;
      tile += warp_n[w];
    }
    if (head) start[base + off + __popc(ballot & ((1u << lane) - 1u))] = (unsigned)p;
    base += tile;
    __syncthreads();
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
    st->n_vox = base;
    start[base] = (unsigned)n_sel;
  }
}

// `passes` 8-bit digit passes over the n keys of key[0] / row[0], ping-ponging through key[1] / row[1]; the sorted
// order ends in buffer (passes & 1).  hist holds 256 x gmm_tiles(n) counters, totals 256.
static inline int gmm_radix_sort(unsigned long long* const key[2], unsigned* const row[2], unsigned long long n, int passes,
                                 unsigned* hist, unsigned* totals, cudaStream_t stream) {
  const unsigned tiles = gmm_tiles(n);
  int cur = 0;
  for (int p = 0; p < passes; ++p, cur ^= 1) {
    k_gmm_hist<<<tiles, kGmmT, 0, stream>>>(key[cur], n, 8 * p, hist, tiles);
    k_gmm_offsets<<<256, kGmmT, 0, stream>>>(hist, tiles, totals);
    k_gmm_scatter<<<tiles, kGmmT, 0, stream>>>(key[cur], row[cur], n, 8 * p, hist, tiles, totals, key[cur ^ 1], row[cur ^ 1]);
  }
  return 3 * passes;
}

static inline unsigned long long gmm_chunk(unsigned long long n, unsigned blocks) {
  const unsigned long long c = (n + blocks - 1) / blocks;
  return (c + kGmmT - 1) / kGmmT * kGmmT;
}

// the heads of the first n sorted keys: start[j] for every distinct key j, start[count] = n and st->n_vox = count
static inline int gmm_heads(const unsigned long long* key, unsigned long long n, unsigned* block_counts, unsigned* start,
                            tloam_gmm_state* st, cudaStream_t stream) {
  unsigned long long b = (n + kGmmT - 1) / kGmmT;
  if (b > kGmmMaxBlocks) b = kGmmMaxBlocks;
  const unsigned long long chunk = gmm_chunk(n, (unsigned)b);
  const unsigned blocks = (unsigned)((n + chunk - 1) / chunk);
  k_gmm_head_count<<<blocks, kGmmT, 0, stream>>>(key, n, chunk, block_counts);
  k_gmm_head_scatter<<<blocks, kGmmT, 0, stream>>>(key, n, chunk, block_counts, start, st);
  return 2;
}

}  // namespace tloam
