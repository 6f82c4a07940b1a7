// scan_context.cu -- libtloam_b200_loop.so: Scan Context place recognition on the device (hand-written CUDA for sm_90a).
//
// A frame's descriptor (Kim & Kim, "Scan Context", IROS 2018) is an n_ring x n_sector polar grid of the scan around the
// sensor: each bin holds the largest z + lidar_height of its finite rows within max_radius (0 when empty).  Every earlier
// frame of the database is compared with the newest at every column shift, and the lexicographic minimum of (distance,
// candidate, shift) is kept: an exact search where the CPU implementation narrows the database with a ring-key KD-tree.
// The full definition is in include/tloam_b200.h ("Loop closure"); tests/scan_context_oracle.py restates it in numpy.
//
// Every value is bit-reproducible on the host: each operation is a separately rounded __d*_rn (no FMA contraction), every
// sum runs in a fixed order, the bin maximum is exact (atomicMax on an order-preserving encoding) and the sector of a row
// is found by comparing it with a table of boundary directions the host computed, not by atan2.
//
// A separate library so that the kernels of libtloam_b200.so keep their SASS.
#include <cuda_runtime.h>
#include <math.h>

#include "scan_context.cuh"
#include "scan_context.h"

namespace tloam {

constexpr unsigned kScThreads = 256;
constexpr size_t kScMaxSmem = 200 * 1024;             // the search's dynamic shared memory (two descriptors at most 128 KB)
constexpr long long kScNone = 0x7fffffffffffffffll;

// order-preserving map of a double onto an unsigned 64-bit integer (a > b <=> enc(a) > enc(b)); 0 is below every encoded
// finite value and stands for an empty bin
__device__ __forceinline__ unsigned long long sc_enc(double v) {
  const unsigned long long u = (unsigned long long)__double_as_longlong(v);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double sc_dec(unsigned long long e) {
  return __longlong_as_double((long long)((e >> 63) ? (e & 0x7fffffffffffffffull) : ~e));
}

// the sector of (x, y): the number of boundary directions k = 1 .. n_sector - 1 (angle 2 pi k / n_sector) the row lies
// strictly counter-clockwise of, the row's azimuth taken in [0, 2 pi).  A row in the upper half-plane [0, pi) (y > 0, or
// y == 0 and x >= 0) is compared with the boundaries below pi (2k < n_sector); a row in the lower one lies above all of
// those and is compared with the rest.  "Counter-clockwise of (c, s)" is c * y - s * x > 0, separately rounded.
__device__ __forceinline__ int sc_sector(const tloam_sc_args& a, double x, double y) {
  const int n_up = (a.n_sector - 1) / 2;
  const bool upper = y > 0.0 || (y == 0.0 && x >= 0.0);
  int sector = upper ? 0 : n_up;
  const int k0 = upper ? 1 : n_up + 1, k1 = upper ? n_up : a.n_sector - 1;
  for (int k = k0; k <= k1; ++k) {
    const double c = __ldg(a.dirs + 2 * (k - 1)), s = __ldg(a.dirs + 2 * (k - 1) + 1);
    if (__dsub_rn(__dmul_rn(c, y), __dmul_rn(s, x)) > 0.0) ++sector;
  }
  return sector;
}

// one thread per row: the bin's maximum of z + lidar_height
__global__ void __launch_bounds__(kScThreads) k_sc_bin(tloam_sc_args a) {
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const double x = a.xyz[3 * i], y = a.xyz[3 * i + 1], z = a.xyz[3 * i + 2];
  if (!isfinite(x) || !isfinite(y) || !isfinite(z)) return;
  const double r = __dsqrt_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)));
  if (!(r <= a.max_radius)) return;
  int ring = (int)ceil(__dmul_rn(__ddiv_rn(r, a.max_radius), (double)a.n_ring));
  ring = (ring < 1 ? 1 : ring > a.n_ring ? a.n_ring : ring) - 1;
  const int sector = sc_sector(a, x, y);
  unsigned long long* bins = reinterpret_cast<unsigned long long*>(a.db + a.frame * TLOAM_SC_SLOT_DOUBLES(a.n_ring, a.n_sector));
  atomicMax(bins + (size_t)ring * a.n_sector + sector, sc_enc(__dadd_rn(z, a.lidar_height)));
}

// one block: the bins decoded in place, then the ring key (row sums in sector order / n_sector) and the column norms
// (sqrt of the sum of squares in ring order), every sum from +0.0
__global__ void __launch_bounds__(kScThreads) k_sc_finish(tloam_sc_args a) {
  const int R = a.n_ring, S = a.n_sector;
  double* d = a.db + a.frame * TLOAM_SC_SLOT_DOUBLES(R, S);
  const unsigned long long* u = reinterpret_cast<const unsigned long long*>(d);
  for (int k = threadIdx.x; k < R * S; k += blockDim.x) {
    const unsigned long long e = u[k];
    d[k] = e ? sc_dec(e) : 0.0;
  }
  __syncthreads();
  for (int t = threadIdx.x; t < R + S; t += blockDim.x) {
    double acc = 0.0;
    if (t < R) {
      for (int s = 0; s < S; ++s) acc = __dadd_rn(acc, d[t * S + s]);
      d[R * S + t] = __ddiv_rn(acc, (double)S);
    } else {
      const int c = t - R;
      for (int r = 0; r < R; ++r) acc = __dadd_rn(acc, __dmul_rn(d[r * S + c], d[r * S + c]));
      d[R * S + R + c] = __dsqrt_rn(acc);
    }
  }
}

// the block's minimum of (d, j, s) into *out (thread 0)
__device__ void sc_block_min(double d, long long j, long long s, tloam_sc_best* out) {
  __shared__ tloam_sc_best wb[kScThreads / 32];
  for (int o = 16; o > 0; o >>= 1) {
    const double od = __shfl_down_sync(0xffffffffu, d, o);
    const long long oj = __shfl_down_sync(0xffffffffu, j, o), os = __shfl_down_sync(0xffffffffu, s, o);
    if (sc_less(od, oj, os, d, j, s)) { d = od; j = oj; s = os; }
  }
  if ((threadIdx.x & 31) == 0) wb[threadIdx.x >> 5] = tloam_sc_best{d, j, s};
  __syncthreads();
  if (threadIdx.x == 0) {
    tloam_sc_best b = wb[0];
    for (unsigned w = 1; w < blockDim.x / 32; ++w)
      if (sc_less(wb[w].distance, wb[w].candidate, wb[w].shift, b.distance, b.candidate, b.shift)) b = wb[w];
    *out = b;
  }
}

// Each block holds the query in shared memory and streams groups of `per_block` candidates through it; thread p of a group
// takes candidate p / S at shift s = p % S, at sc_distance (scan_context.cuh).  Each block's minimum goes to a.partial.
__global__ void __launch_bounds__(kScThreads) k_sc_search(tloam_sc_args a, int per_block) {
  extern __shared__ double sm[];
  const int R = a.n_ring, S = a.n_sector;
  const int bins = R * S, desc = bins + S;
  const unsigned long long slot = TLOAM_SC_SLOT_DOUBLES(R, S);
  const double* q = a.db + a.frame * slot;
  double* qb = sm;                                         // query bins, then its norms
  for (int k = threadIdx.x; k < desc; k += blockDim.x) qb[k] = k < bins ? q[k] : q[bins + R + (k - bins)];
  const double* qn = qb + bins;
  double bd = INFINITY;
  long long bj = kScNone, bs = kScNone;
  const unsigned long long M = a.n_candidates;
  for (unsigned long long g = blockIdx.x; g * per_block < M; g += gridDim.x) {
    __syncthreads();                                       // the previous group is no longer read
    for (int k = threadIdx.x; k < per_block * desc; k += blockDim.x) {
      const int m = k / desc, o = k - m * desc;
      const unsigned long long j = g * per_block + m;
      if (j < M) sm[desc + k] = a.db[j * slot + (o < bins ? o : bins + R + (o - bins))];
    }
    __syncthreads();
    for (int p = threadIdx.x; p < per_block * S; p += blockDim.x) {
      const int m = p / S, s = p - m * S;
      const unsigned long long j = g * per_block + m;
      if (j >= M) continue;
      const double* cb = sm + desc + (size_t)m * desc;
      const double dist = sc_distance(qb, qn, cb, cb + bins, R, S, s);
      if (sc_less(dist, (long long)j, s, bd, bj, bs)) { bd = dist; bj = (long long)j; bs = s; }
    }
  }
  sc_block_min(bd, bj, bs, a.partial + blockIdx.x);
}

// one block: the minimum of the n_part block minima; candidate -1 (distance +inf, shift 0) when there was none
__global__ void __launch_bounds__(kScThreads) k_sc_reduce(tloam_sc_args a, unsigned n_part) {
  double bd = INFINITY;
  long long bj = kScNone, bs = kScNone;
  for (unsigned k = threadIdx.x; k < n_part; k += blockDim.x) {
    const tloam_sc_best p = a.partial[k];
    if (sc_less(p.distance, p.candidate, p.shift, bd, bj, bs)) { bd = p.distance; bj = p.candidate; bs = p.shift; }
  }
  __shared__ tloam_sc_best b;
  sc_block_min(bd, bj, bs, &b);
  if (threadIdx.x == 0) *a.best = b.candidate == kScNone ? tloam_sc_best{INFINITY, -1, 0} : b;
}

}  // namespace tloam

using namespace tloam;

#define TLOAM_SC_API extern "C" __attribute__((visibility("default")))

TLOAM_SC_API int tloam_sc_bin(const tloam_sc_args* a) {
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  double* slot = a->db + a->frame * TLOAM_SC_SLOT_DOUBLES(a->n_ring, a->n_sector);
  e = cudaMemsetAsync(slot, 0, (size_t)a->n_ring * a->n_sector * sizeof(double), a->stream);
  if (e != cudaSuccess || a->n == 0) return (int)e;
  k_sc_bin<<<(unsigned)((a->n + kScThreads - 1) / kScThreads), kScThreads, 0, a->stream>>>(*a);
  return (int)cudaGetLastError();
}

TLOAM_SC_API int tloam_sc_finish(const tloam_sc_args* a) {
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  k_sc_finish<<<1, kScThreads, 0, a->stream>>>(*a);
  return (int)cudaGetLastError();
}

TLOAM_SC_API int tloam_sc_search(const tloam_sc_args* a) {
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  const size_t desc = (size_t)a->n_ring * a->n_sector + a->n_sector;
  int per_block = a->n_sector >= (int)kScThreads ? 1 : (int)kScThreads / a->n_sector;
  while (per_block > 1 && (1 + per_block) * desc * sizeof(double) > kScMaxSmem) --per_block;
  const size_t smem = (1 + per_block) * desc * sizeof(double);
  const unsigned long long groups = (a->n_candidates + per_block - 1) / per_block;
  const unsigned grid = (unsigned)(groups < TLOAM_SC_MAX_BLOCKS ? groups : TLOAM_SC_MAX_BLOCKS);
  if (grid) {
    if (smem > 48 * 1024 &&
        (e = cudaFuncSetAttribute(k_sc_search, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess)
      return (int)e;
    k_sc_search<<<grid, kScThreads, smem, a->stream>>>(*a, per_block);
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  }
  k_sc_reduce<<<1, kScThreads, 0, a->stream>>>(*a, grid);
  return (int)cudaGetLastError();
}
