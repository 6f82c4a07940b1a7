// occupancy.cu -- libtloam_b200_occ.so: the 2D occupancy grid of the global map on the device (hand-written CUDA for
// sm_90a).  The full definition is in include/tloam_b200.h ("Occupancy grid"); tests/occupancy_oracle.py restates it in
// numpy bit for bit.
//
// Per append: the scan's 2D scan, one 32 B record per sector (the nearest row in the obstacle band, by atomicMin on the
// ordered bits of its range and then on its row index, and the farthest floor row, by atomicMax), into the slot the append
// takes.  Per build: one thread per (frame, window cell) counts free cells, one per (frame, sector) counts hits, one per
// cell turns the counts into a value.  Every count is an integer atomicAdd, so the result does not depend on the order.
// Every product, sum, quotient and square root is a separately rounded __dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn /
// __dsqrt_rn in the order written, so that nothing is contracted into an FMA and a numpy restatement reproduces every count.
//
// A separate library so that the kernels of libtloam_b200.so and of the other side libraries keep their SASS.
#include <cuda_runtime.h>

#include "occupancy.h"

namespace tloam {

constexpr unsigned kOccT = 256;
constexpr unsigned kOccCellsPerThread = 16;
constexpr unsigned long long kOccInf = 0x7FF0000000000000ull;   // the bits of +inf: no obstacle yet
constexpr unsigned long long kOccNoRow = ~0ull;

// Scan Context's sector of (x, y).  The same rule as gmd_column in map_dynamic.cu (the half-plane split, then a binary
// search of the boundaries k of that half with c_k y - s_k x > 0); a copy, so that libtloam_b200_gmd.so keeps its SASS.
__device__ __forceinline__ int occ_sector(double x, double y, const double* D, int n_cols) {
  const int n_up = (n_cols - 1) / 2;
  const bool upper = y > 0.0 || (y == 0.0 && x >= 0.0);
  const int base = upper ? 0 : n_up;
  int lo = 0, hi = upper ? n_up : n_cols - 1 - n_up;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    const int k = base + mid - 1;
    if (__dsub_rn(__dmul_rn(D[2 * k], y), __dmul_rn(D[2 * k + 1], x)) > 0.0) lo = mid;
    else hi = mid - 1;
  }
  return base + lo;
}

__device__ __forceinline__ double occ_rho(double x, double y) {
  return __dsqrt_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)));
}

// a used row: finite, min_range <= rho <= max_range; its sector and rho
__device__ __forceinline__ bool occ_used(double x, double y, double z, const tloam_occ_params& p, int* j, double* rho) {
  if (!isfinite(x) || !isfinite(y) || !isfinite(z)) return false;
  const double r = occ_rho(x, y);
  if (!(r >= p.min_range && r <= p.max_range)) return false;
  *rho = r;
  *j = occ_sector(x, y, p.dirs, p.n_cols);
  return true;
}

__global__ void __launch_bounds__(kOccT) k_occ_clear(tloam_occ_capture_args a) {
  const unsigned long long slot = *a.frames;
  if (slot >= a.cap) return;                       // k_gmap_commit flags the overflow
  unsigned long long* s = reinterpret_cast<unsigned long long*>(a.scans + slot * (unsigned long long)a.p.n_cols * TLOAM_OCC_SLOT);
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < a.p.n_cols; j += gridDim.x * blockDim.x) {
    s[TLOAM_OCC_SLOT * j] = kOccInf;               // the obstacle's range bits (atomicMin)
    s[TLOAM_OCC_SLOT * j + 1] = kOccNoRow;         // its row (atomicMin)
    s[TLOAM_OCC_SLOT * j + 2] = 0ull;
    s[TLOAM_OCC_SLOT * j + 3] = 0ull;              // the floor's range bits (atomicMax; 0: none, every rho is > 0)
  }
  if (blockIdx.x == 0 && threadIdx.x < 16) a.poses[slot * 16 + threadIdx.x] = a.pose[threadIdx.x];
}

__global__ void __launch_bounds__(kOccT) k_occ_bin(tloam_occ_capture_args a) {
  const unsigned long long slot = *a.frames;
  if (slot >= a.cap) return;
  unsigned long long* s = reinterpret_cast<unsigned long long*>(a.scans + slot * (unsigned long long)a.p.n_cols * TLOAM_OCC_SLOT);
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
    const double x = a.scan[3ull * i], y = a.scan[3ull * i + 1], z = a.scan[3ull * i + 2];
    int j;
    double r;
    if (!occ_used(x, y, z, a.p, &j, &r)) continue;
    const unsigned long long bits = (unsigned long long)__double_as_longlong(r);   // r > 0: the bits order as the values
    if (z >= a.p.z_lo && z <= a.p.z_hi) atomicMin(s + TLOAM_OCC_SLOT * j, bits);
    else if (z < a.p.z_lo) atomicMax(s + TLOAM_OCC_SLOT * j + 3, bits);
  }
}

// the lowest row index among the band rows at the sector's least range
__global__ void __launch_bounds__(kOccT) k_occ_pick(tloam_occ_capture_args a) {
  const unsigned long long slot = *a.frames;
  if (slot >= a.cap) return;
  unsigned long long* s = reinterpret_cast<unsigned long long*>(a.scans + slot * (unsigned long long)a.p.n_cols * TLOAM_OCC_SLOT);
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
    const double x = a.scan[3ull * i], y = a.scan[3ull * i + 1], z = a.scan[3ull * i + 2];
    int j;
    double r;
    if (!(z >= a.p.z_lo && z <= a.p.z_hi) || !occ_used(x, y, z, a.p, &j, &r)) continue;
    if ((unsigned long long)__double_as_longlong(r) == s[TLOAM_OCC_SLOT * j]) atomicMin(s + TLOAM_OCC_SLOT * j + 1, (unsigned long long)i);
  }
}

// the record: the obstacle's sensor-frame row (NaN x 3 without one), the floor's range (NaN without one)
__global__ void __launch_bounds__(kOccT) k_occ_final(tloam_occ_capture_args a) {
  const unsigned long long slot = *a.frames;
  if (slot >= a.cap) return;
  double* s = a.scans + slot * (unsigned long long)a.p.n_cols * TLOAM_OCC_SLOT;
  const double nan = __longlong_as_double(0x7FF8000000000000ll);
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < a.p.n_cols; j += gridDim.x * blockDim.x) {
    double* r = s + TLOAM_OCC_SLOT * j;
    const unsigned long long row = (unsigned long long)__double_as_longlong(r[1]);
    if (row != kOccNoRow) {
      r[0] = a.scan[3ull * row]; r[1] = a.scan[3ull * row + 1]; r[2] = a.scan[3ull * row + 2];
    } else {
      r[0] = nan; r[1] = nan; r[2] = nan;
    }
    if (__double_as_longlong(r[3]) == 0) r[3] = nan;
  }
}

// one block: min and max of the poses' t_x, t_y
__global__ void __launch_bounds__(kOccT) k_occ_extent(const double* poses, unsigned long long n, double* extent) {
  __shared__ double part[4][kOccT];
  double v[4] = {__longlong_as_double((long long)kOccInf), __longlong_as_double((long long)kOccInf),
                 -__longlong_as_double((long long)kOccInf), -__longlong_as_double((long long)kOccInf)};
  for (unsigned long long f = threadIdx.x; f < n; f += kOccT) {
    const double tx = poses[16 * f + 12], ty = poses[16 * f + 13];
    v[0] = fmin(v[0], tx); v[1] = fmin(v[1], ty); v[2] = fmax(v[2], tx); v[3] = fmax(v[3], ty);
  }
  for (int k = 0; k < 4; ++k) part[k][threadIdx.x] = v[k];
  __syncthreads();
  for (unsigned o = kOccT / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      part[0][threadIdx.x] = fmin(part[0][threadIdx.x], part[0][threadIdx.x + o]);
      part[1][threadIdx.x] = fmin(part[1][threadIdx.x], part[1][threadIdx.x + o]);
      part[2][threadIdx.x] = fmax(part[2][threadIdx.x], part[2][threadIdx.x + o]);
      part[3][threadIdx.x] = fmax(part[3][threadIdx.x], part[3][threadIdx.x + o]);
    }
    __syncthreads();
  }
  if (threadIdx.x < 4) extent[threadIdx.x] = part[threadIdx.x][0];
}

// block (tile, frame): the frame's sector extents in shared memory, then kOccCellsPerThread window cells per thread.
// The tiles are on x, which the blocks are dispatched along first, so a frame's tiles run together and its 2D scan is
// read from HBM once and from L2 by the other tiles; frames past gridDim.y are taken by a stride over y.
__global__ void __launch_bounds__(kOccT) k_occ_free(tloam_occ_build_args a) {
  extern __shared__ double ext[];                  // n_cols: the obstacle's rho, else the floor's rho, else NaN
  __shared__ double T[16];
  const unsigned long long nw = (unsigned long long)a.nwin * (unsigned long long)a.nwin;
  const unsigned long long base = (unsigned long long)blockIdx.x * kOccT * kOccCellsPerThread;
  for (unsigned long long f = blockIdx.y; f < a.n_frames; f += gridDim.y) {
    __syncthreads();                               // the previous frame's extents are no longer read
    const double* s = a.scans + f * (unsigned long long)a.p.n_cols * TLOAM_OCC_SLOT;
    if (threadIdx.x < 16) T[threadIdx.x] = a.poses[16 * f + threadIdx.x];
    for (int j = threadIdx.x; j < a.p.n_cols; j += kOccT) {
      const double* r = s + TLOAM_OCC_SLOT * j;
      ext[j] = isnan(r[0]) ? r[3] : occ_rho(r[0], r[1]);
    }
    __syncthreads();
    const double tx = T[12], ty = T[13];
    const long long i0 = (long long)floor(__ddiv_rn(__dsub_rn(__dsub_rn(tx, a.W), a.origin_x), a.resolution)) - 1;
    const long long j0 = (long long)floor(__ddiv_rn(__dsub_rn(__dsub_rn(ty, a.W), a.origin_y), a.resolution)) - 1;
#pragma unroll 2
    for (unsigned k = 0; k < kOccCellsPerThread; ++k) {
      const unsigned long long w = base + k * kOccT + threadIdx.x;
      if (w >= nw) break;
      const long long i = i0 + (long long)(w % (unsigned long long)a.nwin), jy = j0 + (long long)(w / (unsigned long long)a.nwin);
      if (i < 0 || jy < 0 || i >= (long long)a.width || jy >= (long long)a.height) continue;
      const double cx = __dadd_rn(a.origin_x, __dmul_rn(__dadd_rn((double)i, 0.5), a.resolution));
      const double cy = __dadd_rn(a.origin_y, __dmul_rn(__dadd_rn((double)jy, 0.5), a.resolution));
      const double d0 = __dsub_rn(cx, tx), d1 = __dsub_rn(cy, ty);
      if (!(fabs(d0) <= a.W && fabs(d1) <= a.W)) continue;
      const double q0 = __dadd_rn(__dmul_rn(T[0], d0), __dmul_rn(T[1], d1));   // q_r = R(0, r) d0 + R(1, r) d1
      const double q1 = __dadd_rn(__dmul_rn(T[4], d0), __dmul_rn(T[5], d1));
      const double rho = occ_rho(q0, q1);
      if (!(rho >= a.p.min_range)) continue;
      const double e = ext[occ_sector(q0, q1, a.p.dirs, a.p.n_cols)];
      if (__dadd_rn(rho, a.free_margin) <= e) atomicAdd(a.free_count + (unsigned long long)jy * a.width + (unsigned long long)i, 1u);
    }
  }
}

// one thread per (frame, sector): the obstacle into the world, w = P o, and its cell
__global__ void __launch_bounds__(kOccT) k_occ_hits(tloam_occ_build_args a) {
  const unsigned long long n = a.n_frames * (unsigned long long)a.p.n_cols;
  for (unsigned long long g = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; g < n;
       g += (unsigned long long)gridDim.x * blockDim.x) {
    const double* r = a.scans + g * TLOAM_OCC_SLOT;
    const double x = r[0], y = r[1], z = r[2];
    if (isnan(x)) continue;
    const double* T = a.poses + 16 * (g / (unsigned long long)a.p.n_cols);
    const double wx = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[0], x), __dmul_rn(T[4], y)), __dmul_rn(T[8], z)), T[12]);
    const double wy = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[1], x), __dmul_rn(T[5], y)), __dmul_rn(T[9], z)), T[13]);
    const double fx = floor(__ddiv_rn(__dsub_rn(wx, a.origin_x), a.resolution));
    const double fy = floor(__ddiv_rn(__dsub_rn(wy, a.origin_y), a.resolution));
    if (fx >= 0.0 && fy >= 0.0 && fx < (double)a.width && fy < (double)a.height)
      atomicAdd(a.occupied + (unsigned long long)fy * a.width + (unsigned long long)fx, 1u);
    else
      atomicAdd(a.dropped, 1ull);
  }
}

// -1 without a count, else (100 occ + n / 2) / n
__global__ void __launch_bounds__(kOccT) k_occ_value(tloam_occ_build_args a) {
  const unsigned long long n = (unsigned long long)a.width * a.height;
  for (unsigned long long c = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; c < n;
       c += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long o = a.occupied[c], t = o + a.free_count[c];
    a.cells[c] = t == 0 ? (signed char)-1 : (signed char)((100ull * o + t / 2) / t);
  }
}

static int occ_sms(int device) {
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0) sms = 132;
  return sms;
}

}  // namespace tloam

using namespace tloam;

#define TLOAM_OCC_API extern "C" __attribute__((visibility("default")))

TLOAM_OCC_API int tloam_occ_capture(const tloam_occ_capture_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  const tloam_occ_capture_args args = *a;
  const unsigned gs = (unsigned)((a->p.n_cols + kOccT - 1) / kOccT);
  k_occ_clear<<<gs, kOccT, 0, a->stream>>>(args);
  *launches += 1;
  if (a->n) {
    const unsigned gr = (a->n + kOccT - 1) / kOccT;
    k_occ_bin<<<gr, kOccT, 0, a->stream>>>(args);
    k_occ_pick<<<gr, kOccT, 0, a->stream>>>(args);
    *launches += 2;
  }
  k_occ_final<<<gs, kOccT, 0, a->stream>>>(args);
  *launches += 1;
  return (int)cudaGetLastError();
}

TLOAM_OCC_API int tloam_occ_extent(const tloam_occ_build_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  k_occ_extent<<<1, kOccT, 0, a->stream>>>(a->poses, a->n_frames, a->extent);
  *launches += 1;
  return (int)cudaGetLastError();
}

TLOAM_OCC_API int tloam_occ_rasterise(const tloam_occ_build_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  const size_t cells = (size_t)a->width * a->height;
  if ((e = cudaMemsetAsync(a->occupied, 0, cells * sizeof(unsigned), a->stream)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(a->free_count, 0, cells * sizeof(unsigned), a->stream)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(a->dropped, 0, sizeof(unsigned long long), a->stream)) != cudaSuccess) return (int)e;
  const tloam_occ_build_args args = *a;
  const unsigned long long nw = (unsigned long long)a->nwin * (unsigned long long)a->nwin;
  const unsigned long long tiles = (nw + kOccT * kOccCellsPerThread - 1) / (kOccT * kOccCellsPerThread);
  const dim3 grid((unsigned)tiles, (unsigned)(a->n_frames < 65535ull ? a->n_frames : 65535ull));
  k_occ_free<<<grid, kOccT, a->p.n_cols * sizeof(double), a->stream>>>(args);
  *launches += 1;
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  const unsigned blocks = (unsigned)occ_sms(a->device) * 8u;   // grid-stride over the records and the cells
  k_occ_hits<<<blocks, kOccT, 0, a->stream>>>(args);
  k_occ_value<<<blocks, kOccT, 0, a->stream>>>(args);
  *launches += 2;
  return (int)cudaGetLastError();
}
