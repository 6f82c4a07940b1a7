// distance.cu -- libtloam_b200_dist.so: the distance field and the inflated costmap of an occupancy grid on the device
// (hand-written CUDA for sm_90a).  The full definition is in include/tloam_b200.h ("Distance field and costmap");
// tests/distance_oracle.py restates it in numpy bit for bit.
//
// The transform is the separable exact EDT (Meijster et al. 2000; Felzenszwalb and Huttenlocher 2012), done for both
// source classes at once.  A cell needs the distance to the nearest cell of the other class, so one column distance per
// cell is enough: g_obs is 0 at an obstacle and g at the others, g_other the reverse.
//   - Column pass, in bands of TLOAM_DIST_BAND rows so that it has width x bands threads: k_dist_bands records each band's
//     first and last row of either class, k_dist_cols finds the nearest such rows in the bands above and below and sweeps
//     its band down and up.  Neighbouring threads take neighbouring columns, so every row access is coalesced.
//   - Row pass, one thread per (row, source class): the lower envelope of the parabolas g_k^2 + (i - k)^2 over the
//     columns k with a finite g, kept as a stack of column indices in the row's own scratch, then one walk along it.
//     Every envelope test is the three-site test in 64-bit integers, cross-multiplied, so no intersection is rounded.
//     The thread writes sq at the cells of the other class.
//   - k_dist_cost: sd, the cost through the host's table, the published value, and the obstacle count.
// The query is one thread per point, each product, sum and quotient a separately rounded __dmul_rn / __dadd_rn /
// __dsub_rn / __ddiv_rn, so nothing is contracted into an FMA.
//
// A separate library so that the kernels of libtloam_b200.so and of the other side libraries keep their SASS.
#include <cuda_runtime.h>

#include "distance.h"

namespace tloam {

constexpr unsigned kDistT = 256;
constexpr unsigned kDistRowT = 32;                 // the row pass has 2 x height threads: small blocks spread them
constexpr int kDistObstacle = 65;                  // map_saver's classes: >= 65 obstacle, 0 .. 25 free, else unknown
constexpr int kDistFree = 25;

__device__ __forceinline__ bool dist_obstacle(signed char v) { return v >= kDistObstacle; }

// thread (column i, band b): the band's first and last obstacle row and first and last other row
__global__ void __launch_bounds__(kDistT) k_dist_bands(tloam_dist_build_args a, unsigned nb) {
  const unsigned long long n = (unsigned long long)a.width * nb;
  for (unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; t < n;
       t += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned i = (unsigned)(t % a.width), b = (unsigned)(t / a.width);
    const unsigned j0 = b * TLOAM_DIST_BAND, j1 = min(j0 + TLOAM_DIST_BAND, a.height);
    uint4 r = make_uint4(TLOAM_DIST_INF, TLOAM_DIST_INF, TLOAM_DIST_INF, TLOAM_DIST_INF);
    for (unsigned j = j0; j < j1; ++j) {
      if (dist_obstacle(a.cells[(unsigned long long)j * a.width + i])) {
        if (r.x == TLOAM_DIST_INF) r.x = j;
        r.y = j;
      } else {
        if (r.z == TLOAM_DIST_INF) r.z = j;
        r.w = j;
      }
    }
    reinterpret_cast<uint4*>(a.bands)[t] = r;
  }
}

// thread (column i, band b): the nearest rows of either class above and below the band from the band records, then a
// down sweep and an up sweep over the band; g = the row distance to the nearest cell of the other class in the column
__global__ void __launch_bounds__(kDistT) k_dist_cols(tloam_dist_build_args a, unsigned nb) {
  const unsigned long long n = (unsigned long long)a.width * nb;
  const uint4* B = reinterpret_cast<const uint4*>(a.bands);
  for (unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; t < n;
       t += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned i = (unsigned)(t % a.width), b = (unsigned)(t / a.width);
    const unsigned j0 = b * TLOAM_DIST_BAND, j1 = min(j0 + TLOAM_DIST_BAND, a.height);
    long long up_o = -1, up_f = -1;                // the last row above of either class (-1: none)
    for (unsigned c = b; c-- > 0 && (up_o < 0 || up_f < 0);) {
      const uint4 r = B[(unsigned long long)c * a.width + i];
      if (up_o < 0 && r.y != TLOAM_DIST_INF) up_o = r.y;
      if (up_f < 0 && r.w != TLOAM_DIST_INF) up_f = r.w;
    }
    long long dn_o = -1, dn_f = -1;                // the first row below of either class
    for (unsigned c = b + 1; c < nb && (dn_o < 0 || dn_f < 0); ++c) {
      const uint4 r = B[(unsigned long long)c * a.width + i];
      if (dn_o < 0 && r.x != TLOAM_DIST_INF) dn_o = r.x;
      if (dn_f < 0 && r.z != TLOAM_DIST_INF) dn_f = r.z;
    }
    for (unsigned j = j0; j < j1; ++j) {
      const unsigned long long c = (unsigned long long)j * a.width + i;
      const bool ob = dist_obstacle(a.cells[c]);
      if (ob) up_o = j;
      else up_f = j;
      const long long other = ob ? up_f : up_o;
      a.g[c] = other < 0 ? TLOAM_DIST_INF : (unsigned)((long long)j - other);
    }
    for (unsigned j = j1; j-- > j0;) {
      const unsigned long long c = (unsigned long long)j * a.width + i;
      const bool ob = dist_obstacle(a.cells[c]);
      if (ob) dn_o = j;
      else dn_f = j;
      const long long other = ob ? dn_f : dn_o;
      if (other >= 0) a.g[c] = min(a.g[c], (unsigned)(other - (long long)j));
    }
  }
}

// thread (row j, source class e): e = 0 takes the obstacles as sources (g_k at the other cells, 0 at obstacles), e = 1
// the other cells.  The envelope of g_k^2 + (i - k)^2, then sq at the cells of the other class.
__global__ void __launch_bounds__(kDistRowT) k_dist_rows(tloam_dist_build_args a) {
  const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned j = t >> 1, e = t & 1;
  if (j >= a.height) return;
  const unsigned long long row = (unsigned long long)j * a.width;
  const unsigned W = a.width;
  unsigned short* S = a.stack + 2 * row + e;      // S[2 p]: the envelope's p-th column
  // G of column k for this class: 0 at a source cell, g^2 at the others (g finite), or none
  auto G = [&](unsigned k, long long* out) -> bool {
    const bool src = dist_obstacle(a.cells[row + k]) == (e == 0);
    if (src) { *out = 0; return true; }
    const unsigned g = a.g[row + k];
    if (g == TLOAM_DIST_INF) return false;
    *out = (long long)g * (long long)g;
    return true;
  };
  int top = -1;                                   // the envelope's last entry; its column kb and F_b = G + kb^2
  long long kb = 0, Fb = 0;
  for (unsigned k = 0; k < W; ++k) {
    long long Gc;
    if (!G(k, &Gc)) continue;
    const long long kc = k, Fc = Gc + kc * kc;
    while (top >= 1) {                             // b is hidden when the (a, b) boundary is not left of the (b, c) one
      const long long ka = S[2 * (top - 1)];
      long long Ga;
      G((unsigned)ka, &Ga);
      const long long Fa = Ga + ka * ka;
      if ((Fb - Fa) * (kc - kb) < (Fc - Fb) * (kb - ka)) break;
      --top;
      kb = ka; Fb = Fa;
    }
    ++top;
    S[2 * top] = (unsigned short)k;
    kb = kc; Fb = Fc;
  }
  const int count = top + 1;
  int p = 0;
  long long k0 = 0, G0 = 0;
  if (count > 0) { k0 = S[0]; G(S[0], &G0); }
  for (unsigned x = 0; x < W; ++x) {
    if (dist_obstacle(a.cells[row + x]) != (e == 1)) continue;   // this thread writes the cells of the other class
    if (count == 0) { a.sq[row + x] = TLOAM_DIST_INF; continue; }
    long long d = (long long)x - k0, f = G0 + d * d;
    while (p + 1 < count) {
      const long long k1 = S[2 * (p + 1)];
      long long G1;
      G((unsigned)k1, &G1);
      const long long d1 = (long long)x - k1, f1 = G1 + d1 * d1;
      if (f1 > f) break;
      ++p; k0 = k1; G0 = G1; f = f1;
    }
    a.sq[row + x] = (unsigned)f;
  }
}

// one thread per cell: sd, the cost (254 at an obstacle, the table's c else, 255 for an unknown cell with c < 253), the
// published value, and the obstacles counted by warp
__global__ void __launch_bounds__(kDistT) k_dist_cost(tloam_dist_build_args a) {
  const unsigned long long n = (unsigned long long)a.width * a.height;
  const float inf = __int_as_float(0x7F800000);
  for (unsigned long long base = (unsigned long long)blockIdx.x * blockDim.x; base < n;
       base += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long c = base + threadIdx.x;
    bool ob = false;
    if (c < n) {
      const int v = a.cells[c];
      ob = v >= kDistObstacle;
      const unsigned s = a.sq[c];
      float d = inf;
      if (s != TLOAM_DIST_INF) d = (float)__dmul_rn(__dsqrt_rn((double)s), a.resolution);
      a.sd[c] = ob ? -d : d;
      unsigned cost = 254;
      if (!ob) {
        const unsigned cc = s <= a.r2 ? a.table[s] : 0u;
        cost = (v >= 0 && v <= kDistFree) ? cc : (cc == 253 ? 253u : 255u);
      }
      a.costs[c] = (unsigned char)cost;
      a.values[c] = cost == 0 ? 0 : cost <= 252 ? (signed char)(1 + (97 * (cost - 1)) / 251)
                  : cost == 253 ? 99 : cost == 254 ? 100 : -1;
    }
    const unsigned m = __ballot_sync(0xFFFFFFFFu, ob);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(a.obstacles, (unsigned long long)__popc(m));
  }
}

// one thread per point: the bilinear interpolation of sd at the cell centres and its gradient
__global__ void __launch_bounds__(kDistT) k_dist_query(tloam_dist_query_args a) {
  const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.n) return;
  const double nan = __longlong_as_double(0x7FF8000000000000ll);
  const double x = a.xy[2 * t], y = a.xy[2 * t + 1];
  const double u = __dsub_rn(__ddiv_rn(__dsub_rn(x, a.origin_x), a.resolution), 0.5);
  const double v = __dsub_rn(__ddiv_rn(__dsub_rn(y, a.origin_y), a.resolution), 0.5);
  const double wm = (double)a.width - 1.0, hm = (double)a.height - 1.0;
  if (!a.finite || a.width < 2 || a.height < 2 || !(u >= 0.0 && u <= wm && v >= 0.0 && v <= hm)) {
    a.distance[t] = nan; a.gradient[2 * t] = nan; a.gradient[2 * t + 1] = nan;
    return;
  }
  const unsigned i = min((unsigned)floor(u), a.width - 2), j = min((unsigned)floor(v), a.height - 2);
  const double fa = __dsub_rn(u, (double)i), fb = __dsub_rn(v, (double)j);
  const float* r0 = a.sd + (unsigned long long)j * a.width + i;
  const float* r1 = r0 + a.width;
  const double s00 = r0[0], s10 = r0[1], s01 = r1[0], s11 = r1[1];
  const double ia = __dsub_rn(1.0, fa), ib = __dsub_rn(1.0, fb);
  const double lo = __dadd_rn(__dmul_rn(ia, s00), __dmul_rn(fa, s10));
  const double hi = __dadd_rn(__dmul_rn(ia, s01), __dmul_rn(fa, s11));
  a.distance[t] = __dadd_rn(__dmul_rn(ib, lo), __dmul_rn(fb, hi));
  a.gradient[2 * t] = __ddiv_rn(__dadd_rn(__dmul_rn(ib, __dsub_rn(s10, s00)), __dmul_rn(fb, __dsub_rn(s11, s01))), a.resolution);
  a.gradient[2 * t + 1] = __ddiv_rn(__dadd_rn(__dmul_rn(ia, __dsub_rn(s01, s00)), __dmul_rn(fa, __dsub_rn(s11, s10))), a.resolution);
}

static int dist_sms(int device) {
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0) sms = 132;
  return sms;
}

}  // namespace tloam

using namespace tloam;

#define TLOAM_DIST_API extern "C" __attribute__((visibility("default")))

TLOAM_DIST_API int tloam_dist_build(const tloam_dist_build_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(a->obstacles, 0, sizeof(unsigned long long), a->stream)) != cudaSuccess) return (int)e;
  const tloam_dist_build_args args = *a;
  const unsigned nb = (a->height + TLOAM_DIST_BAND - 1) / TLOAM_DIST_BAND;
  const unsigned long long cb = (unsigned long long)a->width * nb;
  const unsigned blocks = (unsigned)dist_sms(a->device) * 16u;   // grid-stride beyond this
  const unsigned gc = (unsigned)((cb + kDistT - 1) / kDistT < blocks ? (cb + kDistT - 1) / kDistT : blocks);
  k_dist_bands<<<gc, kDistT, 0, a->stream>>>(args, nb);
  k_dist_cols<<<gc, kDistT, 0, a->stream>>>(args, nb);
  k_dist_rows<<<(2u * a->height + kDistRowT - 1) / kDistRowT, kDistRowT, 0, a->stream>>>(args);
  const unsigned long long cells = (unsigned long long)a->width * a->height;
  const unsigned gk = (unsigned)((cells + kDistT - 1) / kDistT < blocks ? (cells + kDistT - 1) / kDistT : blocks);
  k_dist_cost<<<gk, kDistT, 0, a->stream>>>(args);
  *launches += 4;
  return (int)cudaGetLastError();
}

TLOAM_DIST_API int tloam_dist_query(const tloam_dist_query_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  if (!a->n) return cudaSuccess;
  k_dist_query<<<(unsigned)((a->n + kDistT - 1) / kDistT), kDistT, 0, a->stream>>>(*a);
  *launches += 1;
  return (int)cudaGetLastError();
}
