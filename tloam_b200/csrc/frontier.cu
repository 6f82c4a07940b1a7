// frontier.cu -- libtloam_b200_frontier.so: the frontier cells of a costmap, their 8-connected components and each
// component's statistics and approach cell, on the device (hand-written CUDA for sm_90a).  The full definition is in
// include/tloam_b200.h ("Frontiers"); tests/frontier_oracle.py restates it in numpy bit for bit.
//
// Labelling is union-find over parent indices that always point to a smaller cell index (Playne & Hawick's lock-free
// scheme: a root is linked under a smaller one by atomicMin, and a link that lost a race is retried from the value it
// found), so every component's root is its least cell index whatever the order of the unions:
//   - k_fr_tile: one block per TLOAM_FR_TILE^2-cell tile.  It stages the tile's codes with a one-cell halo, marks the
//     frontier cells, unions each with its W, NW, N and NE neighbours inside the tile in shared memory and writes every
//     cell's label: the global index of its tile root, TLOAM_FR_NONE for other cells.  A tile with no frontier cell
//     writes TLOAM_FR_NONE and stops.
//   - k_fr_border: one block per tile that holds a frontier cell; each cell of its top row and its left and right
//     columns unions, in global memory, with its W, NW, N and NE neighbours that lie in another tile.  Every 8-edge
//     across tiles is such a pair.
//   - k_fr_flatten: every frontier cell's label becomes its root; per block the frontier cells of its chunk, and their
//     total for the host, which sizes the grouping's buffers by it.
//   - k_fr_compact: the frontier cells in index order (root as key, cell as row), for the stable radix sort of
//     radix_sort.cuh and its head scan: each component's cells contiguous and ascending, components ascending by root.
//   - k_fr_stats: one warp per component over its cells: size, sums, bounding box, the approach cell by the least
//     (P, index), and the cells' labels set to the component's id.  Integer reductions only, so the result is exact.
//
// A separate library so that the kernels of libtloam_b200.so and of the other side libraries keep their SASS.
#include <cuda_runtime.h>

#include "frontier.h"
#include "radix_sort.cuh"

namespace tloam {

constexpr unsigned kFrT = 256;                             // a tile block: 32 x 8 threads, 4 rows each
constexpr unsigned kFrRows = TLOAM_FR_TILE * TLOAM_FR_TILE / kFrT;
constexpr unsigned kFrS = TLOAM_FR_TILE + 2;               // the staged tile's side, halo included
constexpr unsigned kFrBorderT = 128;                       // a border block: the 94 cells of a tile's top row and sides
constexpr unsigned char kFrOutside = 254;                  // the staged code of a cell outside the grid: never a frontier
                                                           // cell, never free (free_max <= 252)
static_assert(TLOAM_FR_TILE == 32 && kFrRows * 8 == TLOAM_FR_TILE, "a warp is one row of a tile");

__device__ __forceinline__ unsigned ldg_relaxed(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// the root of x: follow the parents (each one smaller) to the index that is its own parent
__device__ __forceinline__ unsigned fr_find_shared(volatile unsigned* L, unsigned x) {
  unsigned p = L[x];
  while (p != x) { x = p; p = L[x]; }
  return x;
}
__device__ __forceinline__ unsigned fr_find_global(const unsigned* L, unsigned x) {
  unsigned p = ldg_relaxed(L + x);
  while (p != x) { x = p; p = ldg_relaxed(L + x); }
  return x;
}

// the union of the sets of a and b: the larger root is linked under the smaller; when the larger one stopped being a
// root in the meantime, atomicMin still leaves it a smaller parent and the union goes on from the parent it had
__device__ __forceinline__ void fr_union_shared(unsigned* L, unsigned a, unsigned b) {
  for (;;) {
    a = fr_find_shared(L, a);
    b = fr_find_shared(L, b);
    if (a == b) return;
    if (a > b) { const unsigned t = a; a = b; b = t; }
    const unsigned old = atomicMin(L + b, a);
    if (old == b) return;
    b = old;
  }
}
__device__ __forceinline__ void fr_union_global(unsigned* L, unsigned a, unsigned b) {
  for (;;) {
    a = fr_find_global(L, a);
    b = fr_find_global(L, b);
    if (a == b) return;
    if (a > b) { const unsigned t = a; a = b; b = t; }
    const unsigned old = atomicMin(L + b, a);
    if (old == b) return;
    b = old;
  }
}

// one block per tile: the frontier flag, the tile's own components and every cell's label
__global__ void __launch_bounds__(kFrT) k_fr_tile(tloam_fr_args a) {
  __shared__ unsigned char s_code[kFrS * kFrS];
  __shared__ unsigned s_lab[TLOAM_FR_TILE * TLOAM_FR_TILE];
  const unsigned ntx = (a.width + TLOAM_FR_TILE - 1) / TLOAM_FR_TILE;
  const unsigned ti = blockIdx.x % ntx, tj = blockIdx.x / ntx;
  const long long x0 = (long long)ti * TLOAM_FR_TILE - 1, y0 = (long long)tj * TLOAM_FR_TILE - 1;
  for (unsigned k = threadIdx.x; k < kFrS * kFrS; k += kFrT) {
    const long long x = x0 + (long long)(k % kFrS), y = y0 + (long long)(k / kFrS);
    const bool in = x >= 0 && y >= 0 && x < (long long)a.width && y < (long long)a.height;
    s_code[k] = in ? a.costs[(unsigned long long)y * a.width + (unsigned long long)x] : kFrOutside;
  }
  __syncthreads();
  const unsigned tx = threadIdx.x % TLOAM_FR_TILE, ty = threadIdx.x / TLOAM_FR_TILE;
  const unsigned fm = a.free_max;
  unsigned flags = 0;                                      // bit q: cell (tx, ty + 8 q) is a frontier cell
  for (unsigned q = 0; q < kFrRows; ++q) {
    const unsigned ly = ty + 8 * q, s = (ly + 1) * kFrS + tx + 1;
    const bool f = s_code[s] == 255 &&
                   (s_code[s + 1] <= fm || s_code[s - 1] <= fm || s_code[s + kFrS] <= fm || s_code[s - kFrS] <= fm);
    s_lab[ly * TLOAM_FR_TILE + tx] = f ? ly * TLOAM_FR_TILE + tx : TLOAM_FR_NONE;
    flags |= (f ? 1u : 0u) << q;
  }
  const bool any = __syncthreads_or(flags != 0);
  if (threadIdx.x == 0) a.tile_any[blockIdx.x] = any ? 1 : 0;
  if (any) {
    for (unsigned q = 0; q < kFrRows; ++q) {
      if (!((flags >> q) & 1u)) continue;
      const unsigned ly = ty + 8 * q, k = ly * TLOAM_FR_TILE + tx;
      const volatile unsigned* V = s_lab;
      if (tx > 0 && V[k - 1] != TLOAM_FR_NONE) fr_union_shared(s_lab, k, k - 1);
      if (ly > 0) {
        if (tx > 0 && V[k - TLOAM_FR_TILE - 1] != TLOAM_FR_NONE) fr_union_shared(s_lab, k, k - TLOAM_FR_TILE - 1);
        if (V[k - TLOAM_FR_TILE] != TLOAM_FR_NONE) fr_union_shared(s_lab, k, k - TLOAM_FR_TILE);
        if (tx + 1 < TLOAM_FR_TILE && V[k - TLOAM_FR_TILE + 1] != TLOAM_FR_NONE)
          fr_union_shared(s_lab, k, k - TLOAM_FR_TILE + 1);
      }
    }
    __syncthreads();
  }
  for (unsigned q = 0; q < kFrRows; ++q) {
    const unsigned ly = ty + 8 * q;
    const long long x = x0 + 1 + tx, y = y0 + 1 + ly;
    if (x >= (long long)a.width || y >= (long long)a.height) continue;
    unsigned lab = TLOAM_FR_NONE;
    if ((flags >> q) & 1u) {
      const unsigned r = fr_find_shared(s_lab, ly * TLOAM_FR_TILE + tx);
      lab = (unsigned)((unsigned long long)(y0 + 1 + r / TLOAM_FR_TILE) * a.width +
                       (unsigned long long)(x0 + 1 + r % TLOAM_FR_TILE));
    }
    a.labels[(unsigned long long)y * a.width + (unsigned long long)x] = lab;
  }
}

// one block per tile: the unions across the tile's top edge and its sides
__global__ void __launch_bounds__(kFrBorderT) k_fr_border(tloam_fr_args a) {
  if (!a.tile_any[blockIdx.x]) return;
  const unsigned t = threadIdx.x;
  if (t >= 3 * TLOAM_FR_TILE - 2) return;
  const unsigned lx = t < TLOAM_FR_TILE ? t : t < 2 * TLOAM_FR_TILE - 1 ? 0u : TLOAM_FR_TILE - 1;
  const unsigned ly = t < TLOAM_FR_TILE ? 0u : t < 2 * TLOAM_FR_TILE - 1 ? t - (TLOAM_FR_TILE - 1) : t - (2 * TLOAM_FR_TILE - 2);
  const unsigned ntx = (a.width + TLOAM_FR_TILE - 1) / TLOAM_FR_TILE;
  const unsigned ti = blockIdx.x % ntx, tj = blockIdx.x / ntx;
  const long long x = (long long)ti * TLOAM_FR_TILE + lx, y = (long long)tj * TLOAM_FR_TILE + ly;
  if (x >= (long long)a.width || y >= (long long)a.height) return;
  const unsigned c = (unsigned)((unsigned long long)y * a.width + (unsigned long long)x);
  if (a.labels[c] == TLOAM_FR_NONE) return;
  const int dx[4] = {-1, -1, 0, 1}, dy[4] = {0, -1, -1, -1};     // W, NW, N, NE
  for (int d = 0; d < 4; ++d) {
    const long long ux = x + dx[d], uy = y + dy[d];
    if (ux < 0 || uy < 0 || ux >= (long long)a.width) continue;
    if (ux / TLOAM_FR_TILE == (long long)ti && uy / TLOAM_FR_TILE == (long long)tj) continue;
    const unsigned u = (unsigned)((unsigned long long)uy * a.width + (unsigned long long)ux);
    if (a.labels[u] == TLOAM_FR_NONE) continue;
    fr_union_global(a.labels, c, u);
  }
}

// block b, cells [b chunk, (b + 1) chunk): each frontier cell's label becomes its root; the frontier cells counted
__global__ void __launch_bounds__(kGmmT) k_fr_flatten(tloam_fr_args a, unsigned long long n, unsigned long long chunk) {
  const unsigned long long lo = blockIdx.x * chunk, hi = lo + chunk < n ? lo + chunk : n;
  unsigned count = 0;
  for (unsigned long long p = lo + threadIdx.x; p < hi; p += kGmmT) {
    const unsigned l = a.labels[p];
    if (l == TLOAM_FR_NONE) continue;
    ++count;
    const unsigned r = fr_find_global(a.labels, l);
    if (r != l) a.labels[p] = r;
  }
  count = gmm_block_sum(count);
  if (threadIdx.x == 0) {
    a.block_counts[blockIdx.x] = count;
    if (count) atomicAdd(&a.state->cells, (unsigned long long)count);
  }
}

// block b: its base = the frontier cells of blocks 0 .. b - 1, then its chunk in order: (root, cell) at key[0] / row[0]
__global__ void __launch_bounds__(kGmmT) k_fr_compact(tloam_fr_args a, unsigned long long n, unsigned long long chunk) {
  __shared__ unsigned warp_n[kGmmT / 32];
  unsigned before = 0u;
  for (unsigned k = threadIdx.x; k < blockIdx.x; k += kGmmT) before += a.block_counts[k];
  unsigned base = gmm_block_sum(before);
  const unsigned long long lo = blockIdx.x * chunk, hi = lo + chunk < n ? lo + chunk : n;
  const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  for (unsigned long long t = lo; t < hi; t += kGmmT) {
    const unsigned long long p = t + threadIdx.x;
    const unsigned l = p < hi ? a.labels[p] : TLOAM_FR_NONE;
    const bool f = l != TLOAM_FR_NONE;
    const unsigned ballot = __ballot_sync(0xffffffffu, f);
    if (lane == 0) warp_n[warp] = __popc(ballot);
    __syncthreads();
    unsigned off = 0u, tile = 0u;
    for (unsigned w = 0; w < kGmmT / 32; ++w) {
      off += w < warp ? warp_n[w] : 0u;
      tile += warp_n[w];
    }
    if (f) {
      const unsigned pos = base + off + __popc(ballot & ((1u << lane) - 1u));
      a.key[0][pos] = l;
      a.row[0][pos] = (unsigned)p;
    }
    base += tile;
    __syncthreads();
  }
}

// one warp per component j over its cells start[j] .. start[j + 1] - 1 of `rows`
__global__ void __launch_bounds__(kFrT) k_fr_stats(tloam_fr_args a, const unsigned* rows) {
  const unsigned nf = (unsigned)a.state->gmm.n_vox;
  const unsigned lane = threadIdx.x & 31u;
  const unsigned nw = gridDim.x * (kFrT / 32);
  const unsigned W = a.width, H = a.height, fm = a.free_max;
  for (unsigned j = blockIdx.x * (kFrT / 32) + (threadIdx.x >> 5); j < nf; j += nw) {
    const unsigned lo = a.start[j], hi = a.start[j + 1];
    unsigned long long si = 0, sj = 0, bp = 0xFFFFFFFFFFFFFFFFull;
    unsigned mi = 0xFFFFFFFFu, mj = 0xFFFFFFFFu, Mi = 0, Mj = 0, bu = 0xFFFFFFFFu;
    for (unsigned k = lo + lane; k < hi; k += 32) {
      const unsigned c = rows[k];
      const unsigned i = c % W, jj = c / W;
      si += i; sj += jj;
      mi = min(mi, i); mj = min(mj, jj); Mi = max(Mi, i); Mj = max(Mj, jj);
      a.labels[c] = j;
      const bool ok[4] = {i + 1 < W, i > 0, jj + 1 < H, jj > 0};
      const unsigned u4[4] = {c + 1, c - 1, c + W, c - W};
      for (int d = 0; d < 4; ++d) {
        if (!ok[d]) continue;
        const unsigned u = u4[d];
        if (a.costs[u] > fm) continue;
        const unsigned long long p = a.P[u];
        if (p < bp || (p == bp && u < bu)) { bp = p; bu = u; }
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      si += __shfl_xor_sync(0xffffffffu, si, o);
      sj += __shfl_xor_sync(0xffffffffu, sj, o);
      mi = min(mi, __shfl_xor_sync(0xffffffffu, mi, o));
      mj = min(mj, __shfl_xor_sync(0xffffffffu, mj, o));
      Mi = max(Mi, __shfl_xor_sync(0xffffffffu, Mi, o));
      Mj = max(Mj, __shfl_xor_sync(0xffffffffu, Mj, o));
      const unsigned long long op = __shfl_xor_sync(0xffffffffu, bp, o);
      const unsigned ou = __shfl_xor_sync(0xffffffffu, bu, o);
      if (op < bp || (op == bp && ou < bu)) { bp = op; bu = ou; }
    }
    if (lane == 0) {
      tloam_fr_stat s;
      s.sum_i = si; s.sum_j = sj; s.approach_p = bp;
      s.n = hi - lo; s.approach = bu;
      s.min_i = mi; s.min_j = mj; s.max_i = Mi; s.max_j = Mj;
      s.first = lo; s.pad[0] = s.pad[1] = s.pad[2] = 0;
      a.stats[j] = s;
    }
  }
}

static int fr_sms(int device) {
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0) sms = 132;
  return sms;
}

}  // namespace tloam

using namespace tloam;

#define TLOAM_FR_API extern "C" __attribute__((visibility("default")))

// the chunks of the ordered compaction over n cells: at most TLOAM_FR_BLOCKS blocks
static void fr_chunks(unsigned long long n, unsigned long long* chunk, unsigned* blocks) {
  unsigned long long b = (n + kGmmT - 1) / kGmmT;
  if (b > TLOAM_FR_BLOCKS) b = TLOAM_FR_BLOCKS;
  *chunk = gmm_chunk(n, (unsigned)b);
  *blocks = (unsigned)((n + *chunk - 1) / *chunk);
}

TLOAM_FR_API int tloam_fr_label(const tloam_fr_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  const unsigned long long n = (unsigned long long)a->width * a->height;
  const unsigned ntiles = ((a->width + TLOAM_FR_TILE - 1) / TLOAM_FR_TILE) * ((a->height + TLOAM_FR_TILE - 1) / TLOAM_FR_TILE);
  if ((e = cudaMemsetAsync(&a->state->cells, 0, sizeof(a->state->cells), a->stream)) != cudaSuccess) return (int)e;
  k_fr_tile<<<ntiles, kFrT, 0, a->stream>>>(*a);
  k_fr_border<<<ntiles, kFrBorderT, 0, a->stream>>>(*a);
  unsigned long long chunk;
  unsigned blocks;
  fr_chunks(n, &chunk, &blocks);
  k_fr_flatten<<<blocks, kGmmT, 0, a->stream>>>(*a, n, chunk);
  *launches += 3;
  return (int)cudaGetLastError();
}

TLOAM_FR_API int tloam_fr_group(const tloam_fr_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  const unsigned long long m = a->cells;
  if (!m) return cudaSuccess;
  const unsigned long long n = (unsigned long long)a->width * a->height;
  unsigned long long chunk;
  unsigned blocks;
  fr_chunks(n, &chunk, &blocks);
  k_fr_compact<<<blocks, kGmmT, 0, a->stream>>>(*a, n, chunk);
  *launches += 1;
  const int passes = tloam_fr_passes(n);
  *launches += gmm_radix_sort(a->key, a->row, m, passes, a->hist, a->totals, a->stream);
  const int sorted = passes & 1;
  *launches += gmm_heads(a->key[sorted], m, a->block_counts, a->start, &a->state->gmm, a->stream);
  const unsigned long long want = (m + kFrT / 32 - 1) / (kFrT / 32), most = (unsigned long long)fr_sms(a->device) * 16u;
  k_fr_stats<<<(unsigned)(want < most ? want : most), kFrT, 0, a->stream>>>(*a, a->row[sorted]);
  *launches += 1;
  return (int)cudaGetLastError();
}

static unsigned long long fr_align(unsigned long long v) { return (v + 255ull) / 256ull * 256ull; }

TLOAM_FR_API size_t tloam_fr_sort_bytes(unsigned long long cells) {
  return (size_t)(fr_align(16ull * cells) + fr_align(8ull * cells) + fr_align(4ull * 256ull * gmm_tiles(cells)) +
                  fr_align(4ull * 256ull) + fr_align(4ull * (cells + 1)) + fr_align(sizeof(tloam_fr_stat) * cells));
}

TLOAM_FR_API void tloam_fr_sort_layout(void* scratch, unsigned long long cells, tloam_fr_args* a) {
  unsigned char* p = static_cast<unsigned char*>(scratch);
  a->key[0] = reinterpret_cast<unsigned long long*>(p);
  a->key[1] = a->key[0] + cells;
  p += fr_align(16ull * cells);
  a->row[0] = reinterpret_cast<unsigned*>(p);
  a->row[1] = a->row[0] + cells;
  p += fr_align(8ull * cells);
  a->hist = reinterpret_cast<unsigned*>(p);
  p += fr_align(4ull * 256ull * gmm_tiles(cells));
  a->totals = reinterpret_cast<unsigned*>(p);
  p += fr_align(4ull * 256ull);
  a->start = reinterpret_cast<unsigned*>(p);
  p += fr_align(4ull * (cells + 1));
  a->stats = reinterpret_cast<tloam_fr_stat*>(p);
}
