// map_merge.cu -- libtloam_b200_gmm.so: the global map merged into one voxel grid on the device (hand-written CUDA for
// sm_90a).  The full definition is in include/tloam_b200.h ("Merged global map"); tests/global_map_merge_oracle.py
// restates it in numpy bit for bit.
//
// The merge is VoxelDownSample (ref: src/open3d/PointCloud2.cpp:358-403) of the map, or of its static rows:
//   k_gmm_bounds        the selected rows' count and bounds (atomics on the ordered encodings: exact in any schedule);
//                       the host reads them, checks the key range and chooses the bits of ix, iy and iz
//   k_gmm_keys          key = ix << (by + bz) | iy << bz | iz per selected row, 1 << (bx + by + bz) for the others, with
//                       the row index as a u32 payload
//   k_gmm_hist     \
//   k_gmm_offsets   |   stable LSD radix sort on 8-bit digits: per-tile digit counts, per-digit offsets, a stable scatter;
//   k_gmm_scatter  /    a voxel's rows stay in row order
//   k_gmm_head_count \  the positions whose key differs from the previous one, numbered in order: voxel j's first
//   k_gmm_head_scatter/ position, and the voxel count
//   k_gmm_average       one thread per voxel: +0.0, then __dadd_rn over its rows in row order, then __ddiv_rn by the
//                       count (AccumulatedPoint, :246-294), for x, y, z and the intensity
// Every subtraction, quotient and sum is a separately rounded intrinsic, so nothing is contracted into an FMA.
//
// A separate library so that the kernels of libtloam_b200.so keep their SASS: this TU includes map_grid.cuh (no kernels)
// and nothing that defines one.
#include <cuda_runtime.h>
#include <float.h>
#include <string.h>

#include "map_grid.cuh"
#include "map_merge.h"
#include "radix_sort.cuh"

namespace tloam {

static size_t gmm_align(size_t v) { return (v + 255) & ~(size_t)255; }

struct GmmScratch {
  unsigned long long* key[2];
  unsigned* row[2];
  unsigned* hist;                                          // [256][tiles], digit-major
  unsigned* totals;                                        // [256]: rows per digit
  unsigned* block_counts;                                  // [kGmmMaxBlocks]: heads per block
  tloam_gmm_state* state;
};
static GmmScratch gmm_carve(void* base, unsigned long long n) {
  char* p = static_cast<char*>(base);
  GmmScratch s;
  for (int b = 0; b < 2; ++b) { s.key[b] = reinterpret_cast<unsigned long long*>(p); p += gmm_align((size_t)n * 8); }
  for (int b = 0; b < 2; ++b) { s.row[b] = reinterpret_cast<unsigned*>(p); p += gmm_align((size_t)n * 4); }
  s.hist = reinterpret_cast<unsigned*>(p); p += gmm_align((size_t)gmm_tiles(n) * 256 * 4);
  s.totals = reinterpret_cast<unsigned*>(p); p += gmm_align(256 * 4);
  s.block_counts = reinterpret_cast<unsigned*>(p); p += gmm_align(kGmmMaxBlocks * 4);
  s.state = reinterpret_cast<tloam_gmm_state*>(p);
  return s;
}

// the row is in the merge: every row, or (with the counters) a row that is not dynamic
__device__ __forceinline__ bool gmm_selected(const tloam_gmm_args& a, unsigned long long i) {
  if (!a.through) return true;
  const unsigned t = a.through[i];
  return !(t >= a.min_through && t > a.hits[i]);
}

__global__ void __launch_bounds__(kGmmT) k_gmm_bounds(tloam_gmm_args a, tloam_gmm_state* st) {
  double mn[3] = {DBL_MAX, DBL_MAX, DBL_MAX}, mx[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX};
  unsigned long long sel = 0;
  unsigned bad = 0u, any = 0u;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.count;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    if (!gmm_selected(a, i)) continue;
    ++sel;
    const double p[3] = {a.map[3 * i], a.map[3 * i + 1], a.map[3 * i + 2]};
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

__global__ void __launch_bounds__(kGmmT) k_gmm_keys(tloam_gmm_args a, unsigned long long* key, unsigned* row) {
  const int sy = a.bits[2], sx = a.bits[1] + a.bits[2];
  const unsigned long long sentinel = 1ull << (a.bits[0] + a.bits[1] + a.bits[2]);
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.count;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    unsigned long long k = sentinel;
    if (gmm_selected(a, i)) {
      unsigned long long idx[3];
#pragma unroll
      for (int d = 0; d < 3; ++d)
        idx[d] = (unsigned long long)floor(__ddiv_rn(__dsub_rn(a.map[3 * i + d], a.mb[d]), a.voxel));
      k = (idx[0] << sx) | (idx[1] << sy) | idx[2];
    }
    key[i] = k;
    row[i] = (unsigned)i;
  }
}

// voxel j (one thread): its rows start[j] .. start[j + 1] - 1 of the sorted order, summed in row order from +0.0
__global__ void __launch_bounds__(kGmmT) k_gmm_average(tloam_gmm_args a, const unsigned* row, const unsigned* start) {
  for (unsigned long long j = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; j < a.n_vox;
       j += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned lo = start[j], hi = start[j + 1];
    double sx = 0.0, sy = 0.0, sz = 0.0, si = 0.0;
    for (unsigned k = lo; k < hi; ++k) {
      const unsigned long long r = row[k];
      sx = __dadd_rn(sx, a.map[3 * r]);
      sy = __dadd_rn(sy, a.map[3 * r + 1]);
      sz = __dadd_rn(sz, a.map[3 * r + 2]);
      if (a.out_intensity) si = __dadd_rn(si, a.intensity[r]);
    }
    const double c = (double)(hi - lo);
    a.out_xyz[3 * j] = __ddiv_rn(sx, c);
    a.out_xyz[3 * j + 1] = __ddiv_rn(sy, c);
    a.out_xyz[3 * j + 2] = __ddiv_rn(sz, c);
    if (a.out_intensity) a.out_intensity[j] = __ddiv_rn(si, c);
  }
}

static unsigned gmm_grid(unsigned long long n, int device) {
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0) sms = 132;
  const unsigned long long need = (n + kGmmT - 1) / kGmmT, cap = (unsigned long long)sms * 8u;
  return (unsigned)(need < cap ? (need ? need : 1ull) : cap);
}

static int gmm_passes(const tloam_gmm_args& a) {          // 8-bit digits over the key bits (and the sentinel's bit)
  const int bits = a.bits[0] + a.bits[1] + a.bits[2] + (a.through ? 1 : 0);
  return (bits + 7) / 8;
}

}  // namespace tloam

using namespace tloam;

#define TLOAM_GMM_API extern "C" __attribute__((visibility("default")))

TLOAM_GMM_API size_t tloam_gmm_scratch_bytes(unsigned long long count) {
  return 2 * gmm_align((size_t)count * 8) + 2 * gmm_align((size_t)count * 4) + gmm_align((size_t)gmm_tiles(count) * 256 * 4) +
         gmm_align(256 * 4) + gmm_align(kGmmMaxBlocks * 4) + gmm_align(sizeof(tloam_gmm_state));
}

TLOAM_GMM_API tloam_gmm_state* tloam_gmm_state_of(void* scratch, unsigned long long count) {
  return gmm_carve(scratch, count).state;
}

TLOAM_GMM_API int tloam_gmm_bounds(const tloam_gmm_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  const GmmScratch s = gmm_carve(a->scratch, a->count);
  if ((e = cudaMemsetAsync(s.state, 0, sizeof(tloam_gmm_state), a->stream)) != cudaSuccess) return (int)e;
  if (!a->count) return (int)cudaSuccess;
  k_gmm_bounds<<<gmm_grid(a->count, a->device), kGmmT, 0, a->stream>>>(*a, s.state);
  *launches = 1;
  return (int)cudaGetLastError();
}

TLOAM_GMM_API int tloam_gmm_sort(const tloam_gmm_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  const GmmScratch s = gmm_carve(a->scratch, a->count);
  if (!a->n_sel) return (int)cudaSuccess;                    // n_vox stays 0 from the bounds' clear
  const unsigned long long n = a->count;
  k_gmm_keys<<<gmm_grid(n, a->device), kGmmT, 0, a->stream>>>(*a, s.key[0], s.row[0]);
  const int passes = gmm_passes(*a), cur = passes & 1;
  const int nl = 1 + gmm_radix_sort(s.key, s.row, n, passes, s.hist, s.totals, a->stream);
  // the selected rows are positions [0, n_sel) of the sorted keys (the sentinel sorts last); the voxel starts go to the
  // other key buffer, free after the last pass, and the average reads the rows of the buffer the last pass wrote
  unsigned* start = reinterpret_cast<unsigned*>(s.key[cur ^ 1]);
  gmm_heads(s.key[cur], a->n_sel, s.block_counts, start, s.state, a->stream);
  *launches = nl + 2;
  return (int)cudaGetLastError();
}

TLOAM_GMM_API int tloam_gmm_average(const tloam_gmm_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  if (!a->n_vox) return (int)cudaSuccess;
  const GmmScratch s = gmm_carve(a->scratch, a->count);
  const int cur = gmm_passes(*a) & 1;
  const unsigned* start = reinterpret_cast<const unsigned*>(s.key[cur ^ 1]);
  const unsigned long long need = (a->n_vox + kGmmT - 1) / kGmmT;
  k_gmm_average<<<(unsigned)(need < 65535ull * 16 ? need : 65535ull * 16), kGmmT, 0, a->stream>>>(*a, s.row[cur], start);
  *launches = 1;
  return (int)cudaGetLastError();
}
