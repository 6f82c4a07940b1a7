// terrain.cu -- libtloam_b200_terrain.so: the terrain map of a cloud on the device, per cell the ground reference,
// elevation, step, slope, roughness and traversability value (hand-written CUDA for sm_90a).  The full definition is in
// include/tloam_b200.h ("Terrain"); tests/terrain_oracle.py restates it in numpy bit for bit.
//
// Every extremum is an atomic or a comparison on the ordered 64-bit encoding of a double (map_grid.cuh's enc_ordered:
// -0.0 orders below +0.0), so it does not depend on the order of the rows; every sum runs over a window in a fixed order.
//   - k_ter_bounds  one thread per row: the selected finite rows' x / y extent (atomics on the encodings)
//   - k_ter_low     one thread per row: its cell, atomicMax of the complemented encoding of z (the least z) and the count
//   - k_ter_ground  one thread per cell, launched twice: the max of the complemented encodings over the clipped window
//                   along x, then along y; a window max is separable, so the two passes give G over the (2 rg + 1)^2 window
//   - k_ter_high    one thread per row: rows at or below G + clearance give the elevation by atomicMax, the others are
//                   overhangs
//   - k_ter_layers  one block per 32 x 32 tile: the known cells' encodings with a halo of max(rs, rp) in shared memory,
//                   then per cell the step, the plane fit (integer moments exact, FP64 sums in window order), the
//                   roughness, the class and the value, combined with the occupancy value when asked
// Every subtraction, product, sum, quotient and square root is a separately rounded intrinsic, so nothing is contracted
// into an FMA.
//
// A separate library so that the kernels of libtloam_b200.so and of the other side libraries keep their SASS: this TU
// includes map_grid.cuh (no kernels) and nothing that defines one.
#include <cuda_runtime.h>
#include <math.h>
#include <math_constants.h>

#include "map_grid.cuh"
#include "terrain.h"

namespace tloam {

constexpr unsigned kTerT = 256;                            // threads per block of every kernel
constexpr unsigned kTerRows = TLOAM_TER_TILE * TLOAM_TER_TILE / kTerT;
static_assert(kTerRows * 8 == TLOAM_TER_TILE, "a layers block is 32 x 8 threads, 4 rows each");

// the row is in the terrain: every row, or (with the counters) a row that is not dynamic (the merge's rule)
__device__ __forceinline__ bool ter_selected(const tloam_ter_args& a, unsigned long long i) {
  if (!a.through) return true;
  const unsigned t = a.through[i];
  return !(t >= a.min_through && t > a.hits[i]);
}

// the cell of a finite row, false outside the grid
__device__ __forceinline__ bool ter_cell(const tloam_ter_args& a, double x, double y, unsigned long long* c) {
  const double fi = floor(__ddiv_rn(__dsub_rn(x, a.origin_x), a.resolution));
  const double fj = floor(__ddiv_rn(__dsub_rn(y, a.origin_y), a.resolution));
  if (!(fi >= 0.0 && fi < (double)a.width && fj >= 0.0 && fj < (double)a.height)) return false;
  *c = (unsigned long long)fj * a.width + (unsigned long long)fi;
  return true;
}

__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(kTerT) k_ter_bounds(tloam_ter_args a) {
  unsigned long long lo[2] = {0, 0}, hi[2] = {0, 0};       // on the encodings, so that -0.0 orders below +0.0
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.count;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    if (!ter_selected(a, i)) continue;
    const double p[3] = {a.rows[3 * i], a.rows[3 * i + 1], a.rows[3 * i + 2]};
    if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]))) continue;
#pragma unroll
    for (int d = 0; d < 2; ++d) { lo[d] = max(lo[d], ~enc_ordered(p[d])); hi[d] = max(hi[d], enc_ordered(p[d])); }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int d = 0; d < 2; ++d) {
      lo[d] = max(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
      hi[d] = max(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
    }
  }
  if ((threadIdx.x & 31u) != 0u || !hi[0]) return;
#pragma unroll
  for (int d = 0; d < 2; ++d) {
    atomicMax(&a.state->lo[d], lo[d]);
    atomicMax(&a.state->hi[d], hi[d]);
  }
}

__global__ void __launch_bounds__(kTerT) k_ter_low(tloam_ter_args a) {
  unsigned long long used = 0, skipped = 0, dropped = 0;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.count;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    if (!ter_selected(a, i)) continue;
    const double x = a.rows[3 * i], y = a.rows[3 * i + 1], z = a.rows[3 * i + 2];
    if (!(isfinite(x) && isfinite(y) && isfinite(z))) { ++skipped; continue; }
    unsigned long long c;
    if (!ter_cell(a, x, y, &c)) { ++dropped; continue; }
    ++used;
    atomicMax(a.lo + c, ~enc_ordered(z));
    atomicAdd(a.n + c, 1u);
  }
  used = warp_sum(used); skipped = warp_sum(skipped); dropped = warp_sum(dropped);
  if ((threadIdx.x & 31u) != 0u) return;
  if (used) atomicAdd(&a.state->used, used);
  if (skipped) atomicAdd(&a.state->skipped, skipped);
  if (dropped) atomicAdd(&a.state->dropped, dropped);
}

// dst = the max of src over the cell's clipped window of radius r along x (along_y 0) or y (along_y 1)
__global__ void __launch_bounds__(kTerT) k_ter_ground(const unsigned long long* __restrict__ src,
                                                     unsigned long long* __restrict__ dst, unsigned width, unsigned height,
                                                     unsigned r, int along_y) {
  const unsigned long long n = (unsigned long long)width * height;
  for (unsigned long long c = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; c < n;
       c += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned i = (unsigned)(c % width), j = (unsigned)(c / width);
    const unsigned at = along_y ? j : i, size = along_y ? height : width;
    const unsigned lo = at > r ? at - r : 0u, hi = size - 1u - at > r ? at + r : size - 1u;
    const unsigned long long stride = along_y ? width : 1u;
    const unsigned long long* p = src + (c - (unsigned long long)(at - lo) * stride);
    unsigned long long m = 0;
    for (unsigned k = lo; k <= hi; ++k, p += stride) m = max(m, *p);
    dst[c] = m;
  }
}

__global__ void __launch_bounds__(kTerT) k_ter_high(tloam_ter_args a) {
  unsigned long long overhang = 0;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.count;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    if (!ter_selected(a, i)) continue;
    const double x = a.rows[3 * i], y = a.rows[3 * i + 1], z = a.rows[3 * i + 2];
    if (!(isfinite(x) && isfinite(y) && isfinite(z))) continue;
    unsigned long long c;
    if (!ter_cell(a, x, y, &c)) continue;
    const unsigned long long g = a.g[c];                     // never 0: the row's own cell is in its window
    if (z <= __dadd_rn(dec_ordered(~g), a.clearance)) {
      atomicMax(a.e + c, enc_ordered(z));
      atomicAdd(a.m + c, 1u);
    } else {
      ++overhang;
    }
  }
  overhang = warp_sum(overhang);
  if ((threadIdx.x & 31u) == 0u && overhang) atomicAdd(&a.state->overhang, overhang);
}

// one block per tile; the staged keys are the known cells' elevation encodings, 0 elsewhere (no finite double encodes
// to 0), over the tile and a halo of H = max(rs, rp) cells, cells outside the grid staged as 0 (the windows' clipping)
__global__ void __launch_bounds__(kTerT) k_ter_layers(tloam_ter_args a) {
  extern __shared__ unsigned long long s_key[];
  const unsigned H = a.rs > a.rp ? a.rs : a.rp, S = TLOAM_TER_TILE + 2 * H;
  const unsigned ntx = (a.width + TLOAM_TER_TILE - 1) / TLOAM_TER_TILE;
  const long long x0 = (long long)(blockIdx.x % ntx) * TLOAM_TER_TILE, y0 = (long long)(blockIdx.x / ntx) * TLOAM_TER_TILE;
  for (unsigned k = threadIdx.x; k < S * S; k += kTerT) {
    const long long x = x0 - H + (long long)(k % S), y = y0 - H + (long long)(k / S);
    unsigned long long v = 0;
    if (x >= 0 && y >= 0 && x < (long long)a.width && y < (long long)a.height) {
      const unsigned long long c = (unsigned long long)y * a.width + (unsigned long long)x;
      if (a.m[c] >= a.min_points) v = a.e[c];
    }
    s_key[k] = v;
  }
  __syncthreads();
  const unsigned tx = threadIdx.x % TLOAM_TER_TILE, ty = threadIdx.x / TLOAM_TER_TILE;
  unsigned known = 0, lethal = 0;
  for (unsigned q = 0; q < kTerRows; ++q) {
    const unsigned ly = ty + 8 * q;
    const long long x = x0 + tx, y = y0 + ly;
    if (x >= (long long)a.width || y >= (long long)a.height) continue;
    const unsigned long long c = (unsigned long long)y * a.width + (unsigned long long)x;
    const unsigned s = (ly + H) * S + tx + H;
    const unsigned long long kc = s_key[s];
    double step = CUDART_NAN, slope = CUDART_NAN, rough = CUDART_NAN;
    int tv = -1;
    if (kc) {
      // the step: the largest minus the least known elevation of the step window
      unsigned long long kmax = 0, kmin = ~0ull;
      const int rs = (int)a.rs, rp = (int)a.rp;
      for (int dj = -rs; dj <= rs; ++dj)
        for (int di = -rs; di <= rs; ++di) {
          const unsigned long long k = s_key[(int)s + dj * (int)S + di];
          if (k) { kmax = max(kmax, k); kmin = min(kmin, k); }
        }
      step = __dsub_rn(dec_ordered(kmax), dec_ordered(kmin));
      // the plane fit over the slope window, dj outer and di inner, ascending
      const double ec = dec_ordered(kc);
      int N = 0, Su = 0, Sv = 0, Suu = 0, Suv = 0, Svv = 0;
      double Sw = 0.0, Suw = 0.0, Svw = 0.0;
      for (int dj = -rp; dj <= rp; ++dj)
        for (int di = -rp; di <= rp; ++di) {
          const unsigned long long k = s_key[(int)s + dj * (int)S + di];
          if (!k) continue;
          const double w = __dsub_rn(dec_ordered(k), ec);
          ++N; Su += di; Sv += dj; Suu += di * di; Suv += di * dj; Svv += dj * dj;
          Sw = __dadd_rn(Sw, w);
          Suw = __dadd_rn(Suw, __dmul_rn((double)di, w));
          Svw = __dadd_rn(Svw, __dmul_rn((double)dj, w));
        }
      const long long n = N, su = Su, sv = Sv, suu = Suu, suv = Suv, svv = Svv;
      const long long c11 = svv * n - sv * sv, c12 = sv * su - suv * n, c13 = suv * sv - svv * su;
      const long long c22 = suu * n - su * su, c23 = suv * su - suu * sv, c33 = suu * svv - suv * suv;
      const long long det = suu * c11 + suv * c12 + su * c13;
      if ((unsigned)N >= a.min_fit && det != 0) {
        const double D = (double)det, C11 = (double)c11, C12 = (double)c12, C13 = (double)c13;
        const double C22 = (double)c22, C23 = (double)c23, C33 = (double)c33;
        const double pa = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(C11, Suw), __dmul_rn(C12, Svw)), __dmul_rn(C13, Sw)), D);
        const double pb = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(C12, Suw), __dmul_rn(C22, Svw)), __dmul_rn(C23, Sw)), D);
        const double pd = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(C13, Suw), __dmul_rn(C23, Svw)), __dmul_rn(C33, Sw)), D);
        slope = __ddiv_rn(__dsqrt_rn(__dadd_rn(__dmul_rn(pa, pa), __dmul_rn(pb, pb))), a.resolution);
        rough = 0.0;
        for (int dj = -rp; dj <= rp; ++dj)
          for (int di = -rp; di <= rp; ++di) {
            const unsigned long long k = s_key[(int)s + dj * (int)S + di];
            if (!k) continue;
            const double w = __dsub_rn(dec_ordered(k), ec);
            const double p = __dadd_rn(__dadd_rn(__dmul_rn(pa, (double)di), __dmul_rn(pb, (double)dj)), pd);
            rough = fmax(rough, fabs(__dsub_rn(w, p)));
          }
      }
      const bool bad = step > a.max_step || slope > a.tan_max_slope || rough > a.max_roughness;
      tv = bad ? 100 : 0;
      ++known;
      lethal += bad ? 1u : 0u;
    }
    int v = tv;
    if (a.occupancy) {
      const int o = a.occupancy[c];
      v = (tv == 100 || o >= 65) ? 100 : ((tv == 0 || (o >= 0 && o <= 25)) ? 0 : -1);
    }
    a.step[c] = step; a.slope[c] = slope; a.roughness[c] = rough;
    a.values[c] = (signed char)v;
  }
  known = __reduce_add_sync(0xffffffffu, known);
  lethal = __reduce_add_sync(0xffffffffu, lethal);
  if ((threadIdx.x & 31u) != 0u) return;
  if (known) atomicAdd(&a.state->known, (unsigned long long)known);
  if (lethal) atomicAdd(&a.state->lethal, (unsigned long long)lethal);
}

static unsigned ter_grid(unsigned long long n, int device) {
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0) sms = 132;
  const unsigned long long need = (n + kTerT - 1) / kTerT, cap = (unsigned long long)sms * 8u;
  return (unsigned)(need < cap ? (need ? need : 1ull) : cap);
}

}  // namespace tloam

using namespace tloam;

#define TLOAM_TER_API extern "C" __attribute__((visibility("default")))

TLOAM_TER_API int tloam_ter_bounds(const tloam_ter_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(a->state, 0, sizeof(tloam_ter_state), a->stream)) != cudaSuccess) return (int)e;
  if (!a->count) return (int)cudaSuccess;
  k_ter_bounds<<<ter_grid(a->count, a->device), kTerT, 0, a->stream>>>(*a);
  *launches = 1;
  return (int)cudaGetLastError();
}

TLOAM_TER_API int tloam_ter_build(const tloam_ter_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(a->state, 0, sizeof(tloam_ter_state), a->stream)) != cudaSuccess) return (int)e;
  const unsigned long long n = (unsigned long long)a->width * a->height;
  const unsigned rows = ter_grid(a->count, a->device), cells = ter_grid(n, a->device);
  if (!n) {                                                // no cell: k_ter_low only counts the rows
    if (!a->count) return (int)cudaSuccess;
    k_ter_low<<<rows, kTerT, 0, a->stream>>>(*a);
    *launches = 1;
    return (int)cudaGetLastError();
  }
  if ((e = cudaMemsetAsync(a->lo, 0, n * sizeof(unsigned long long), a->stream)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(a->e, 0, n * sizeof(unsigned long long), a->stream)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(a->n, 0, n * sizeof(unsigned), a->stream)) != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(a->m, 0, n * sizeof(unsigned), a->stream)) != cudaSuccess) return (int)e;
  int nl = 0;
  if (a->count) { k_ter_low<<<rows, kTerT, 0, a->stream>>>(*a); ++nl; }
  k_ter_ground<<<cells, kTerT, 0, a->stream>>>(a->lo, a->gx, a->width, a->height, a->rg, 0);
  k_ter_ground<<<cells, kTerT, 0, a->stream>>>(a->gx, a->g, a->width, a->height, a->rg, 1);
  nl += 2;
  if (a->count) { k_ter_high<<<rows, kTerT, 0, a->stream>>>(*a); ++nl; }
  const unsigned H = a->rs > a->rp ? a->rs : a->rp, S = TLOAM_TER_TILE + 2 * H;
  const unsigned tiles = ((a->width + TLOAM_TER_TILE - 1) / TLOAM_TER_TILE) * ((a->height + TLOAM_TER_TILE - 1) / TLOAM_TER_TILE);
  k_ter_layers<<<tiles, kTerT, (size_t)S * S * sizeof(unsigned long long), a->stream>>>(*a);
  *launches = nl + 1;
  return (int)cudaGetLastError();
}
