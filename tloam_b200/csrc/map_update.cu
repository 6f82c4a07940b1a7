// map_update.cu -- libtloam_b200_mapu.so: updating a prior map from localized frames on the device (hand-written CUDA for
// sm_90a).  The full definition is in include/tloam_b200.h ("Updating a prior map"); tests/map_update_oracle.py restates
// it in numpy bit for bit.
//
// Per add (the free-space votes are tloam_gmd_vote of libtloam_b200_gmd.so, called by the host between these):
//   k_mu_pose           T column-major from the localization's final state, and the prior map's row count, for the votes
//   k_mu_novel          one thread per query row: p = T q by loc_apply, then the cells and columns of the localization's
//                       grid search (loc_range / loc_column) until a prior row lies within novel_radius
//   k_mu_count \        an order-preserving compaction: per-block counts, then a ballot per warp and a scan over the
//   k_mu_scatter/       warps; the new rows go behind the additions in query order
// Per build (the prior rows' part is tloam_gmd_static):
//   k_mu_bounds         the kept additions' count and bounds (atomics on the ordered encodings: exact in any schedule)
//   k_mu_keys           the merge's voxel key per kept addition, a sentinel above every key for the others
//   k_gmm_*             the shared stable radix sort and head scan (radix_sort.cuh): a voxel's rows stay in row order
//   k_mu_average        one thread per voxel: the merge's sums in row order, the distinct frames (1 + the frame increases,
//                       since the frame numbers never decrease along the rows), the min_frames test
//   k_mu_count / k_mu_scatter of the supported voxels behind the kept prior rows
// Every product, sum, quotient and square root is a separately rounded intrinsic, so nothing is contracted into an FMA.
//
// A separate library so that the kernels of libtloam_b200.so keep their SASS.
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>

#include "localize_icp.cuh"
#include "map_grid.cuh"
#include "map_update.h"
#include "radix_sort.cuh"

namespace tloam {

static size_t mu_align(size_t v) { return (v + 255) & ~(size_t)255; }

// ---- compaction -----------------------------------------------------------------------------------------------------------
// block b: the flagged rows of its chunk [b chunk, (b + 1) chunk); block 0 also keeps *count as the base of the scatter
__global__ void __launch_bounds__(kGmmT) k_mu_count(const unsigned char* flag, unsigned long long n, unsigned long long chunk,
                                                    unsigned* block_counts, const unsigned long long* count,
                                                    unsigned long long* base) {
  const unsigned long long lo = blockIdx.x * chunk, hi = lo + chunk < n ? lo + chunk : n;
  unsigned c = 0u;
  for (unsigned long long i = lo + threadIdx.x; i < hi; i += kGmmT) c += flag[i] ? 1u : 0u;
  c = gmm_block_sum(c);
  if (threadIdx.x == 0) {
    block_counts[blockIdx.x] = c;
    if (blockIdx.x == 0) *base = *count;
  }
}

// block b: its first output = *base + the flagged rows of blocks 0 .. b - 1, then its chunk tile by tile; row i goes to
// that output + the flagged rows before it, with the frame number and counters (0, 0) when those outputs are given.  The
// last block writes *count = *base + every flagged row.
__global__ void __launch_bounds__(kGmmT) k_mu_scatter(const unsigned char* flag, const double* src, unsigned long long n,
                                                      unsigned long long chunk, const unsigned* block_counts,
                                                      const unsigned long long* base, double* dst, unsigned* frame_out,
                                                      unsigned frame, unsigned* through, unsigned* hits,
                                                      unsigned long long* count) {
  __shared__ unsigned warp_n[kGmmT / 32];
  unsigned before = 0u;
  for (unsigned k = threadIdx.x; k < blockIdx.x; k += kGmmT) before += block_counts[k];
  unsigned long long o0 = *base + gmm_block_sum(before);
  const unsigned long long lo = blockIdx.x * chunk, hi = lo + chunk < n ? lo + chunk : n;
  const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  for (unsigned long long t = lo; t < hi; t += kGmmT) {
    const unsigned long long i = t + threadIdx.x;
    const bool keep = i < hi && flag[i];
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_n[warp] = __popc(ballot);
    __syncthreads();
    unsigned off = 0u, tile = 0u;
    for (unsigned w = 0; w < kGmmT / 32; ++w) {
      off += w < warp ? warp_n[w] : 0u;
      tile += warp_n[w];
    }
    if (keep) {
      const unsigned long long o = o0 + off + __popc(ballot & ((1u << lane) - 1u));
      dst[3 * o] = src[3 * i];
      dst[3 * o + 1] = src[3 * i + 1];
      dst[3 * o + 2] = src[3 * i + 2];
      if (frame_out) { frame_out[o] = frame; through[o] = 0u; hits[o] = 0u; }
    }
    o0 += tile;
    __syncthreads();
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) *count = o0;
}

static unsigned long long mu_chunk(unsigned long long n, unsigned* blocks) {
  unsigned long long b = (n + kGmmT - 1) / kGmmT;
  if (b > TLOAM_MU_MAX_BLOCKS) b = TLOAM_MU_MAX_BLOCKS;
  const unsigned long long chunk = gmm_chunk(n, (unsigned)b);
  *blocks = (unsigned)((n + chunk - 1) / chunk);
  return chunk;
}

// ---- add ------------------------------------------------------------------------------------------------------------------
__global__ void k_mu_pose(tloam_mu_add_args a) {
  if (threadIdx.x != 0) return;
  const tloam_loc_state* s = a.state;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) a.pose[4 * c + r] = s->R[3 * r + c];
    a.pose[12 + r] = s->t[r];
    a.pose[4 * r + 3] = 0.0;
  }
  a.pose[15] = 1.0;
  *a.prior_count = a.n_prior;
}

// one thread per query row: p = T q, new iff no prior row has d2 <= radius^2.  The cells visited are the grid search's, so
// the answer is the exhaustive scan's; the first row within the radius ends the search.
__global__ void __launch_bounds__(kGmmT) k_mu_novel(tloam_mu_add_args a) {
  const unsigned long long i = blockIdx.x * (unsigned long long)kGmmT + threadIdx.x;
  if (i >= a.nq) return;
  double px, py, pz;
  loc_apply(a.state, a.query[3 * i], a.query[3 * i + 1], a.query[3 * i + 2], px, py, pz);
  a.p[3 * i] = px; a.p[3 * i + 1] = py; a.p[3 * i + 2] = pz;
  bool near = false;
  if (a.n_prior) {
    const tloam_loc_grid& g = a.grid;
    const unsigned n_cells = (unsigned)g.st->n_vox;
    const double r2 = __dmul_rn(a.radius, a.radius), rr = __dmul_ru(a.radius, kLocInflate);
    long long lx, hx, ly, hy, lz, hz;
    loc_range(g, 0, px, rr, lx, hx);
    loc_range(g, 1, py, rr, ly, hy);
    loc_range(g, 2, pz, rr, lz, hz);
    if (lz <= hz)
      for (long long ix = lx; ix <= hx && !near; ++ix)
        for (long long iy = ly; iy <= hy && !near; ++iy) {
          unsigned j0, j1;
          loc_column(g, n_cells, ix, iy, lz, hz, j0, j1);
          for (unsigned j = j0; j < j1; ++j)
            if (nf_d2(px, py, pz, g.sxyz[3ull * j], g.sxyz[3ull * j + 1], g.sxyz[3ull * j + 2]) <= r2) { near = true; break; }
        }
  }
  a.flag[i] = near ? 0 : 1;
}

// ---- build ----------------------------------------------------------------------------------------------------------------
struct MuScratch {
  unsigned long long* key[2];
  unsigned* row[2];
  unsigned* hist;
  unsigned* totals;
  unsigned* block_counts;
  double* vox;                                             // n_vox x 3: every voxel's average
  unsigned char* keep;                                     // n_vox: the voxel has min_frames distinct frames
  unsigned long long* base;
  tloam_gmm_state* state;
};
static MuScratch mu_carve(void* scratch, unsigned long long n) {
  char* p = static_cast<char*>(scratch);
  MuScratch s;
  for (int b = 0; b < 2; ++b) { s.key[b] = reinterpret_cast<unsigned long long*>(p); p += mu_align((size_t)n * 8); }
  for (int b = 0; b < 2; ++b) { s.row[b] = reinterpret_cast<unsigned*>(p); p += mu_align((size_t)n * 4); }
  s.hist = reinterpret_cast<unsigned*>(p); p += mu_align((size_t)gmm_tiles(n) * 256 * 4);
  s.totals = reinterpret_cast<unsigned*>(p); p += mu_align(256 * 4);
  s.block_counts = reinterpret_cast<unsigned*>(p); p += mu_align(kGmmMaxBlocks * 4);
  s.vox = reinterpret_cast<double*>(p); p += mu_align((size_t)n * 24);
  s.keep = reinterpret_cast<unsigned char*>(p); p += mu_align((size_t)n);
  s.base = reinterpret_cast<unsigned long long*>(p); p += mu_align(sizeof(unsigned long long));
  s.state = reinterpret_cast<tloam_gmm_state*>(p);
  return s;
}

// the addition is kept: not removed by the dynamic removal's rule
__device__ __forceinline__ bool mu_kept(const tloam_mu_build_args& a, unsigned long long i) {
  const unsigned t = a.add_through[i];
  return !(t >= a.min_through && t > a.add_hits[i]);
}

__global__ void __launch_bounds__(kGmmT) k_mu_bounds(tloam_mu_build_args a, tloam_gmm_state* st) {
  double mn[3] = {DBL_MAX, DBL_MAX, DBL_MAX}, mx[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX};
  unsigned long long sel = 0;
  unsigned bad = 0u, any = 0u;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n_add;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    if (!mu_kept(a, i)) continue;
    ++sel;
    const double p[3] = {a.add_xyz[3 * i], a.add_xyz[3 * i + 1], a.add_xyz[3 * i + 2]};
    if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]))) { bad = 1u; continue; }
    any = 1u;
#pragma unroll
    for (int d = 0; d < 3; ++d) { mn[d] = fmin(mn[d], p[d]); mx[d] = fmax(mx[d], p[d]); }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      mn[d] = fmin(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o));
      mx[d] = fmax(mx[d], __shfl_xor_sync(0xffffffffu, mx[d], o));
    }
    sel += __shfl_xor_sync(0xffffffffu, sel, o);
    bad |= __shfl_xor_sync(0xffffffffu, bad, o);
    any |= __shfl_xor_sync(0xffffffffu, any, o);
  }
  if ((threadIdx.x & 31u) != 0u) return;
  if (sel) atomicAdd(&st->n_sel, sel);
  if (bad) atomicOr(&st->nonfinite, 1u);
  if (any) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      atomicMax(&st->lo[d], ~enc_ordered(mn[d]));
      atomicMax(&st->hi[d], enc_ordered(mx[d]));
    }
  }
}

__global__ void __launch_bounds__(kGmmT) k_mu_keys(tloam_mu_build_args a, unsigned long long* key, unsigned* row) {
  const int sy = a.bits[2], sx = a.bits[1] + a.bits[2];
  const unsigned long long sentinel = 1ull << (a.bits[0] + a.bits[1] + a.bits[2]);
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n_add;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    unsigned long long k = sentinel;
    if (mu_kept(a, i)) {
      unsigned long long idx[3];
#pragma unroll
      for (int d = 0; d < 3; ++d)
        idx[d] = (unsigned long long)floor(__ddiv_rn(__dsub_rn(a.add_xyz[3 * i + d], a.mb[d]), a.voxel));
      k = (idx[0] << sx) | (idx[1] << sy) | idx[2];
    }
    key[i] = k;
    row[i] = (unsigned)i;
  }
}

// voxel j (one thread): its rows start[j] .. start[j + 1] - 1 of the sorted order, summed in row order from +0.0 and
// divided by the count; kept iff its rows come from at least min_frames distinct adds
__global__ void __launch_bounds__(kGmmT) k_mu_average(tloam_mu_build_args a, const unsigned* row, const unsigned* start,
                                                      double* vox, unsigned char* keep) {
  for (unsigned long long j = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; j < a.n_vox;
       j += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned lo = start[j], hi = start[j + 1];
    double sx = 0.0, sy = 0.0, sz = 0.0;
    unsigned frames = 0u, last = 0u;
    for (unsigned k = lo; k < hi; ++k) {
      const unsigned long long r = row[k];
      sx = __dadd_rn(sx, a.add_xyz[3 * r]);
      sy = __dadd_rn(sy, a.add_xyz[3 * r + 1]);
      sz = __dadd_rn(sz, a.add_xyz[3 * r + 2]);
      const unsigned f = a.add_frame[r];
      if (k == lo || f > last) ++frames;
      last = f;
    }
    const double c = (double)(hi - lo);
    vox[3 * j] = __ddiv_rn(sx, c);
    vox[3 * j + 1] = __ddiv_rn(sy, c);
    vox[3 * j + 2] = __ddiv_rn(sz, c);
    keep[j] = frames >= a.min_frames ? 1 : 0;
  }
}

static unsigned mu_grid(unsigned long long n, int device) {
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0) sms = 132;
  const unsigned long long need = (n + kGmmT - 1) / kGmmT, cap = (unsigned long long)sms * 8u;
  return (unsigned)(need < cap ? (need ? need : 1ull) : cap);
}

static int mu_passes(const tloam_mu_build_args& a) {       // 8-bit digits over the key bits and the sentinel's bit
  return (a.bits[0] + a.bits[1] + a.bits[2] + 1 + 7) / 8;
}

}  // namespace tloam

using namespace tloam;

#define TLOAM_MU_API extern "C" __attribute__((visibility("default")))

TLOAM_MU_API int tloam_mu_pose(const tloam_mu_add_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  k_mu_pose<<<1, 32, 0, a->stream>>>(*a);
  *launches = 1;
  return (int)cudaGetLastError();
}

TLOAM_MU_API int tloam_mu_novel(const tloam_mu_add_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  if (!a->nq) return (int)cudaSuccess;
  k_mu_novel<<<(unsigned)((a->nq + kGmmT - 1) / kGmmT), kGmmT, 0, a->stream>>>(*a);
  unsigned blocks;
  const unsigned long long chunk = mu_chunk(a->nq, &blocks);
  k_mu_count<<<blocks, kGmmT, 0, a->stream>>>(a->flag, a->nq, chunk, a->block_counts, a->count, a->base);
  k_mu_scatter<<<blocks, kGmmT, 0, a->stream>>>(a->flag, a->p, a->nq, chunk, a->block_counts, a->base, a->add_xyz, a->add_frame,
                                                a->frame, a->add_through, a->add_hits, a->count);
  *launches = 3;
  return (int)cudaGetLastError();
}

TLOAM_MU_API size_t tloam_mu_scratch_bytes(unsigned long long n) {
  return 2 * mu_align((size_t)n * 8) + 2 * mu_align((size_t)n * 4) + mu_align((size_t)gmm_tiles(n) * 256 * 4) +
         mu_align(256 * 4) + mu_align(kGmmMaxBlocks * 4) + mu_align((size_t)n * 24) + mu_align((size_t)n) +
         mu_align(sizeof(unsigned long long)) + mu_align(sizeof(tloam_gmm_state));
}

TLOAM_MU_API tloam_gmm_state* tloam_mu_state_of(void* scratch, unsigned long long n) { return mu_carve(scratch, n).state; }

TLOAM_MU_API int tloam_mu_bounds(const tloam_mu_build_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  const MuScratch s = mu_carve(a->scratch, a->n_add);
  if ((e = cudaMemsetAsync(s.state, 0, sizeof(tloam_gmm_state), a->stream)) != cudaSuccess) return (int)e;
  if (!a->n_add) return (int)cudaSuccess;
  k_mu_bounds<<<mu_grid(a->n_add, a->device), kGmmT, 0, a->stream>>>(*a, s.state);
  *launches = 1;
  return (int)cudaGetLastError();
}

TLOAM_MU_API int tloam_mu_sort(const tloam_mu_build_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  if (!a->n_sel) return (int)cudaSuccess;                    // n_vox stays 0 from the bounds' clear
  const MuScratch s = mu_carve(a->scratch, a->n_add);
  const unsigned long long n = a->n_add;
  k_mu_keys<<<mu_grid(n, a->device), kGmmT, 0, a->stream>>>(*a, s.key[0], s.row[0]);
  const int passes = mu_passes(*a), cur = passes & 1;
  const int nl = 1 + gmm_radix_sort(s.key, s.row, n, passes, s.hist, s.totals, a->stream);
  // the kept rows are positions [0, n_sel) of the sorted keys (the sentinel sorts last); the voxel starts go to the other
  // key buffer, free after the last pass
  gmm_heads(s.key[cur], a->n_sel, s.block_counts, reinterpret_cast<unsigned*>(s.key[cur ^ 1]), s.state, a->stream);
  *launches = nl + 2;
  return (int)cudaGetLastError();
}

TLOAM_MU_API int tloam_mu_average(const tloam_mu_build_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  if (!a->n_vox) return (int)cudaSuccess;
  const MuScratch s = mu_carve(a->scratch, a->n_add);
  const int cur = mu_passes(*a) & 1;
  k_mu_average<<<mu_grid(a->n_vox, a->device), kGmmT, 0, a->stream>>>(*a, s.row[cur],
                                                                      reinterpret_cast<const unsigned*>(s.key[cur ^ 1]), s.vox,
                                                                      s.keep);
  unsigned blocks;
  const unsigned long long chunk = mu_chunk(a->n_vox, &blocks);
  k_mu_count<<<blocks, kGmmT, 0, a->stream>>>(s.keep, a->n_vox, chunk, s.block_counts, a->count, s.base);
  k_mu_scatter<<<blocks, kGmmT, 0, a->stream>>>(s.keep, s.vox, a->n_vox, chunk, s.block_counts, s.base, a->out_xyz, nullptr, 0u,
                                                nullptr, nullptr, a->count);
  *launches = 3;
  return (int)cudaGetLastError();
}
