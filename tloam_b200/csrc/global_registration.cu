// global_registration.cu -- libtloam_b200_greg.so: registration of two clouds with no initial guess (hand-written CUDA for
// sm_90a).  Each side's keypoints are indexed and given normals by tloam_loc_index (libtloam_b200_loc.so); here the
// normals are oriented to the sensor, each keypoint gets an FPFH feature (Rusu 2009), the features are matched both ways
// and the mutual pairs kept, a fixed number of three-pair hypotheses is scored in parallel, and the best one is refined by
// alternating a least-squares rigid fit (Horn's quaternion method) with the truncated inlier set.  The full definition is
// in include/tloam_b200.h ("Global registration"); tests/global_registration_oracle.py restates it in numpy.
//
// Every floating-point operation is a separately rounded FP64 intrinsic and no transcendental function runs on the
// device (theta is binned by sign tests against a host table), so each result is a fixed function of the inputs.
//
// A separate library so that the kernels of libtloam_b200.so keep their SASS.
#include <cuda_runtime.h>
#include <math.h>

#include "global_registration.h"
#include "localize_icp.cuh"
#include "normal_fit.cuh"

namespace tloam {

constexpr unsigned kGrT = TLOAM_GR_THREADS;
constexpr int kGrB = TLOAM_GR_BINS;
constexpr unsigned kGrRows = 64;                 // rows per block of the per-row kernels: about 5k keypoints fill ~80 SMs
constexpr unsigned kGrTile = 32;                 // target features per shared-memory tile of k_gr_match
constexpr unsigned kGrOneBlock = 1024;           // threads of the single-block k_gr_mutual
enum { kGrConverged = 0, kGrIterationLimit = 1, kGrFewInliers = 2, kGrFewCorrespondences = 3, kGrNoHypothesis = 4 };

// every sorted position of side g in the cells that can hold a row within rr of p, in ascending sorted position (the
// columns in (ix, iy) order, each a run of ascending cell key): f(j)
template <class F>
__device__ __forceinline__ void gr_walk(const tloam_loc_grid& g, double px, double py, double pz, double rr, F f) {
  const unsigned n_cells = (unsigned)g.st->n_vox;
  long long lx, hx, ly, hy, lz, hz;
  loc_range(g, 0, px, rr, lx, hx);
  loc_range(g, 1, py, rr, ly, hy);
  loc_range(g, 2, pz, rr, lz, hz);
  if (lz > hz) return;
  for (long long ix = lx; ix <= hx; ++ix)
    for (long long iy = ly; iy <= hy; ++iy) {
      unsigned j0, j1;
      loc_column(g, n_cells, ix, iy, lz, hz, j0, j1);
      for (unsigned j = j0; j < j1; ++j) f(j);
    }
}

__device__ __forceinline__ void gr_cross(const double a[3], const double b[3], double c[3]) {
  c[0] = __dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1]));
  c[1] = __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2]));
  c[2] = __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]));
}

__device__ __forceinline__ double gr_dot(const double a[3], const double b[3]) { return nf_dot3(a[0], b[0], a[1], b[1], a[2], b[2]); }

// floor(11 ((f + 1) / 2)), clamped to [0, 10]
__device__ __forceinline__ int gr_lin_bin(double f) {
  const double b = floor(__dmul_rn(11.0, __dmul_rn(__dadd_rn(f, 1.0), 0.5)));
  return b < 0.0 ? 0 : b > 10.0 ? 10 : (int)b;
}

// the bin of theta = atan2(y, x) among 11 equal bins of [-pi, pi]: the boundaries beta_k (k = 1 .. 10) with theta >=
// beta_k, each decided by the sign of c_k y - s_k x within the half plane where that sign is the order
__device__ __forceinline__ int gr_theta_bin(const double* cs, double x, double y) {
  const bool upper = y > 0.0 || (y == 0.0 && x < 0.0);
  int b = 0;
#pragma unroll
  for (int k = 0; k < 10; ++k) {
    const bool s = __dsub_rn(__dmul_rn(cs[2 * k], y), __dmul_rn(cs[2 * k + 1], x)) >= 0.0;
    b += (k < 5 ? (y >= 0.0 || s) : (upper && s)) ? 1 : 0;
  }
  return b;
}

// the pair (p1, n1) -> (p2, n2) at squared distance d2 > 0: the roles swapped when |n1 . d| < |n2 . d| (d = p2 - p1),
// then the Darboux frame u = n1, v = (d x u) / |d x u|, w = u x v and the bins of theta = atan2(w . n2, u . n2),
// alpha = v . n2 and phi = (u . d) / |d| at 0, 11 and 22; false when d x u = 0
__device__ __forceinline__ bool gr_pair(const double* cs, const double p1[3], const double n1[3], const double p2[3],
                                        const double n2[3], double d2, int bins[3]) {
  double d[3] = {__dsub_rn(p2[0], p1[0]), __dsub_rn(p2[1], p1[1]), __dsub_rn(p2[2], p1[2])};
  const double a1 = gr_dot(n1, d), a2 = gr_dot(n2, d);
  const bool swap = fabs(a1) < fabs(a2);
  const double u[3] = {swap ? n2[0] : n1[0], swap ? n2[1] : n1[1], swap ? n2[2] : n1[2]};
  const double m[3] = {swap ? n1[0] : n2[0], swap ? n1[1] : n2[1], swap ? n1[2] : n2[2]};
  if (swap) { d[0] = -d[0]; d[1] = -d[1]; d[2] = -d[2]; }
  const double phi = __ddiv_rn(swap ? -a2 : a1, __dsqrt_rn(d2));
  double v[3], w[3];
  gr_cross(d, u, v);
  const double vn = __dsqrt_rn(gr_dot(v, v));
  if (vn == 0.0) return false;
  v[0] = __ddiv_rn(v[0], vn); v[1] = __ddiv_rn(v[1], vn); v[2] = __ddiv_rn(v[2], vn);
  gr_cross(u, v, w);
  bins[0] = gr_theta_bin(cs, gr_dot(u, m), gr_dot(w, m));
  bins[1] = 11 + gr_lin_bin(gr_dot(v, m));
  bins[2] = 22 + gr_lin_bin(phi);
  return true;
}

// ---- features -----------------------------------------------------------------------------------------------------------
// one thread per row: n <- -n when n . p > 0 (the viewpoint is the origin)
__global__ void __launch_bounds__(kGrRows) k_gr_orient(tloam_gr_side s) {
  const unsigned long long i = (unsigned long long)blockIdx.x * kGrRows + threadIdx.x;
  if (i >= s.n) return;
  double* n = s.normal + 3 * i;
  const double* p = s.xyz + 3 * i;
  if (nf_dot3(n[0], p[0], n[1], p[1], n[2], p[2]) > 0.0) { n[0] = -n[0]; n[1] = -n[1]; n[2] = -n[2]; }
}

// one thread per row with a valid normal: the integer SPFH counts over its neighbours (valid normals, 0 < d2 <= r^2, not
// itself) and the number of pairs; spfh is zero on entry
__global__ void __launch_bounds__(kGrRows) k_gr_spfh(tloam_gr_side s, double radius, tloam_gr_args a) {
  const unsigned long long i = (unsigned long long)blockIdx.x * kGrRows + threadIdx.x;
  if (i >= s.n) return;
  int np = 0;
  if (s.valid[i]) {
    const double p[3] = {s.xyz[3 * i], s.xyz[3 * i + 1], s.xyz[3 * i + 2]};
    const double n[3] = {s.normal[3 * i], s.normal[3 * i + 1], s.normal[3 * i + 2]};
    const double r2 = __dmul_rn(radius, radius), rr = __dmul_ru(radius, kLocInflate);
    int* cnt = s.spfh + (size_t)kGrB * i;
    gr_walk(s.grid, p[0], p[1], p[2], rr, [&](unsigned j) {
      const unsigned v = s.grid.srow[j];
      if (v == i || !s.valid[v]) return;
      const double q[3] = {s.grid.sxyz[3ull * j], s.grid.sxyz[3ull * j + 1], s.grid.sxyz[3ull * j + 2]};
      const double d2 = nf_d2(p[0], p[1], p[2], q[0], q[1], q[2]);
      if (!(d2 <= r2) || d2 == 0.0) return;
      const double m[3] = {s.normal[3ull * v], s.normal[3ull * v + 1], s.normal[3ull * v + 2]};
      int b[3];
      if (!gr_pair(a.theta_cs, p, n, q, m, d2, b)) return;
      cnt[b[0]] += 1; cnt[b[1]] += 1; cnt[b[2]] += 1;
      ++np;
    });
  }
  s.pairs[i] = np;
}

// one thread per row: a row with pairs gets FPFH = SPFH(p) + per block of 11 bins 100 acc / sum, acc = the neighbours'
// SPFH(k) / d2_k summed in walk order over the neighbours with pairs (SPFH(k) = 100 count / pairs)
__global__ void __launch_bounds__(kGrRows) k_gr_fpfh(tloam_gr_side s, double radius) {
  const unsigned long long i = (unsigned long long)blockIdx.x * kGrRows + threadIdx.x;
  if (i >= s.n) return;
  double* F = s.feature + (size_t)kGrB * i;
  const int np = s.pairs[i];
  if (np == 0) {
#pragma unroll
    for (int j = 0; j < kGrB; ++j) F[j] = 0.0;
    s.has_feature[i] = 0;
    return;
  }
  const double p[3] = {s.xyz[3 * i], s.xyz[3 * i + 1], s.xyz[3 * i + 2]};
  const double r2 = __dmul_rn(radius, radius), rr = __dmul_ru(radius, kLocInflate);
  double acc[kGrB], sum[3] = {0.0, 0.0, 0.0};
#pragma unroll
  for (int j = 0; j < kGrB; ++j) acc[j] = 0.0;
  gr_walk(s.grid, p[0], p[1], p[2], rr, [&](unsigned j) {
    const unsigned v = s.grid.srow[j];
    if (v == i || !s.valid[v]) return;
    const double d2 = nf_d2(p[0], p[1], p[2], s.grid.sxyz[3ull * j], s.grid.sxyz[3ull * j + 1], s.grid.sxyz[3ull * j + 2]);
    if (!(d2 <= r2) || d2 == 0.0) return;
    const int pv = s.pairs[v];
    if (pv == 0) return;
    const int* c = s.spfh + (size_t)kGrB * v;
    const double npv = (double)pv;
#pragma unroll
    for (int k = 0; k < kGrB; ++k) {
      const double val = __ddiv_rn(__ddiv_rn(__dmul_rn((double)c[k], 100.0), npv), d2);
      acc[k] = __dadd_rn(acc[k], val);
      sum[k / 11] = __dadd_rn(sum[k / 11], val);
    }
  });
  const int* c = s.spfh + (size_t)kGrB * i;
  const double npi = (double)np;
#pragma unroll
  for (int k = 0; k < kGrB; ++k) {
    const double sc = sum[k / 11] != 0.0 ? __ddiv_rn(__dmul_rn(acc[k], 100.0), sum[k / 11]) : acc[k];
    F[k] = __dadd_rn(sc, __ddiv_rn(__dmul_rn((double)c[k], 100.0), npi));
  }
  s.has_feature[i] = 1;
  atomicAdd(s.n_features, 1ull);
}

// ---- matches ------------------------------------------------------------------------------------------------------------
// one thread per row of a: the row of b whose feature is nearest by the squared L2 distance summed in bin order (the
// lower row on a tie), over tiles of kGrTile features of b staged in shared memory; -1 for a row without a feature or
// when b has none
__global__ void __launch_bounds__(kGrRows) k_gr_match(tloam_gr_side a, tloam_gr_side b, int* nn) {
  __shared__ double tile[kGrTile * kGrB];
  __shared__ unsigned char ok[kGrTile];
  const unsigned long long i = (unsigned long long)blockIdx.x * kGrRows + threadIdx.x;
  const bool mine = i < a.n && a.has_feature[i];
  double f[kGrB];
#pragma unroll
  for (int k = 0; k < kGrB; ++k) f[k] = mine ? a.feature[(size_t)kGrB * i + k] : 0.0;
  double best = INFINITY;
  int bi = -1;
  for (unsigned long long base = 0; base < b.n; base += kGrTile) {
    __syncthreads();
    const unsigned long long lim = (b.n - base) * kGrB;
    for (unsigned e = threadIdx.x; e < kGrTile * kGrB; e += kGrRows) tile[e] = e < lim ? b.feature[(size_t)kGrB * base + e] : 0.0;
    for (unsigned e = threadIdx.x; e < kGrTile; e += kGrRows) ok[e] = base + e < b.n ? b.has_feature[base + e] : 0;
    __syncthreads();
    if (!mine) continue;
    for (unsigned k = 0; k < kGrTile; ++k) {
      if (!ok[k]) continue;
      double d = 0.0;
#pragma unroll
      for (int j = 0; j < kGrB; ++j) {
        const double t = __dsub_rn(f[j], tile[k * kGrB + j]);
        d = __dadd_rn(d, __dmul_rn(t, t));
      }
      if (d < best) { best = d; bi = (int)(base + k); }
    }
  }
  if (i < a.n) nn[i] = bi;
}

// one block: the pairs (i, j = nn_src[i]) with nn_tgt[j] = i, written in source order
__global__ void __launch_bounds__(kGrOneBlock) k_gr_mutual(tloam_gr_args a) {
  __shared__ unsigned wcount[kGrOneBlock / 32], woff[kGrOneBlock / 32];
  __shared__ unsigned long long base;
  const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  if (threadIdx.x == 0) base = 0;
  unsigned total = 0;                            // thread 0: this chunk's pairs, kept out of shared memory, which the next
                                                 // chunk's counts overwrite as soon as the last barrier releases the warps
  for (unsigned long long start = 0; start < a.src.n; start += kGrOneBlock) {
    const unsigned long long i = start + threadIdx.x;
    const int j = i < a.src.n ? a.src.nn[i] : -1;
    const bool ok = j >= 0 && a.tgt.nn[j] == (int)i;
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) wcount[warp] = __popc(bal);
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned o = 0;
      for (unsigned w = 0; w < kGrOneBlock / 32; ++w) { woff[w] = o; o += wcount[w]; }
      total = o;
    }
    __syncthreads();
    if (ok) {
      const unsigned long long pos = base + woff[warp] + __popc(bal & ((1u << lane) - 1u));
      a.corr[2 * pos] = (int)i;
      a.corr[2 * pos + 1] = j;
    }
    __syncthreads();
    if (threadIdx.x == 0) base += total;
  }
  __syncthreads();
  if (threadIdx.x == 0) a.state->n_corr = base;
}

// ---- hypotheses ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long gr_splitmix64(unsigned long long x) {
  unsigned long long z = x + 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

// draw d of hypothesis h
__device__ __forceinline__ unsigned long long gr_draw(unsigned long long seed, unsigned h, unsigned d) {
  return gr_splitmix64(seed ^ gr_splitmix64(((unsigned long long)h << 2) | d));
}

// the triangle (x0, x1, x2): its cross-product norm and its Gram-Schmidt frame e1 = a / |a|, e2 = b / |b| with
// b = u - (u . e1) e1, e3 = e1 x e2 (a = x1 - x0, u = x2 - x0)
__device__ __forceinline__ double gr_frame(const double x[3][3], double e[3][3]) {
  const double a[3] = {__dsub_rn(x[1][0], x[0][0]), __dsub_rn(x[1][1], x[0][1]), __dsub_rn(x[1][2], x[0][2])};
  const double u[3] = {__dsub_rn(x[2][0], x[0][0]), __dsub_rn(x[2][1], x[0][1]), __dsub_rn(x[2][2], x[0][2])};
  double c[3];
  gr_cross(a, u, c);
  const double area = __dsqrt_rn(gr_dot(c, c));
  const double la = __dsqrt_rn(gr_dot(a, a));
#pragma unroll
  for (int k = 0; k < 3; ++k) e[0][k] = __ddiv_rn(a[k], la);
  const double pr = gr_dot(u, e[0]);
  double b[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) b[k] = __dsub_rn(u[k], __dmul_rn(pr, e[0][k]));
  const double lb = __dsqrt_rn(gr_dot(b, b));
#pragma unroll
  for (int k = 0; k < 3; ++k) e[1][k] = __ddiv_rn(b[k], lb);
  gr_cross(e[0], e[1], e[2]);
  return area;
}

// hypothesis h over nc >= 3 pairs: its three distinct pairs, the edge-length and area checks, and T = (R, t) with
// R = F E^T and t = c_q - R c_p; false when rejected
__device__ __forceinline__ bool gr_hypothesis(const tloam_gr_args& a, unsigned h, unsigned long long nc, double R[9], double t[3]) {
  unsigned long long i0 = gr_draw(a.seed, h, 0) % nc, i1 = gr_draw(a.seed, h, 1) % (nc - 1), i2 = gr_draw(a.seed, h, 2) % (nc - 2);
  if (i1 >= i0) ++i1;
  const unsigned long long lo = i0 < i1 ? i0 : i1, hi = i0 < i1 ? i1 : i0;
  if (i2 >= lo) ++i2;
  if (i2 >= hi) ++i2;
  const unsigned long long id[3] = {i0, i1, i2};
  double p[3][3], q[3][3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const unsigned long long si = (unsigned long long)a.corr[2 * id[k]], ti = (unsigned long long)a.corr[2 * id[k] + 1];
#pragma unroll
    for (int c = 0; c < 3; ++c) { p[k][c] = a.src.xyz[3 * si + c]; q[k][c] = a.tgt.xyz[3 * ti + c]; }
  }
#pragma unroll
  for (int u = 0; u < 2; ++u)
#pragma unroll
    for (int v = u + 1; v < 3; ++v) {
      const double ds = __dsqrt_rn(nf_d2(p[u][0], p[u][1], p[u][2], p[v][0], p[v][1], p[v][2]));
      const double dt = __dsqrt_rn(nf_d2(q[u][0], q[u][1], q[u][2], q[v][0], q[v][1], q[v][2]));
      if (ds < __dmul_rn(dt, a.edge_similarity) || dt < __dmul_rn(ds, a.edge_similarity)) return false;
    }
  double E[3][3], F[3][3];
  const double ap = gr_frame(p, E), aq = gr_frame(q, F);
  if (!(ap >= a.min_triangle_area) || !(aq >= a.min_triangle_area)) return false;
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) R[3 * r + c] = nf_dot3(F[0][r], E[0][c], F[1][r], E[1][c], F[2][r], E[2][c]);
  double cp[3], cq[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    cp[c] = __ddiv_rn(__dadd_rn(__dadd_rn(p[0][c], p[1][c]), p[2][c]), 3.0);
    cq[c] = __ddiv_rn(__dadd_rn(__dadd_rn(q[0][c], q[1][c]), q[2][c]), 3.0);
  }
#pragma unroll
  for (int r = 0; r < 3; ++r) t[r] = __dsub_rn(cq[r], nf_dot3(R[3 * r], cp[0], R[3 * r + 1], cp[1], R[3 * r + 2], cp[2]));
  return true;
}

// |R p + t - q|^2, R p + t as ((R_r0 px + R_r1 py) + R_r2 pz) + t_r
__device__ __forceinline__ double gr_res2(const double R[9], const double t[3], const double p[3], const double q[3]) {
  const double x = __dadd_rn(nf_dot3(R[0], p[0], R[1], p[1], R[2], p[2]), t[0]);
  const double y = __dadd_rn(nf_dot3(R[3], p[0], R[4], p[1], R[5], p[2]), t[1]);
  const double z = __dadd_rn(nf_dot3(R[6], p[0], R[7], p[1], R[8], p[2]), t[2]);
  return nf_d2(x, y, z, q[0], q[1], q[2]);
}

// one thread per hypothesis: its inliers (pairs with |T p - q|^2 < tau^2) over tiles of pairs staged in shared memory,
// -1 when rejected (or with fewer than 3 pairs)
__global__ void __launch_bounds__(kGrT) k_gr_hyp(tloam_gr_args a) {
  __shared__ double sp[kGrT][3], sq[kGrT][3];
  const unsigned long long nc = a.state->n_corr;
  const unsigned h = blockIdx.x * kGrT + threadIdx.x;
  double R[9], t[3];
  bool live = h < (unsigned)a.n_hypotheses && nc >= 3;
  if (live) live = gr_hypothesis(a, h, nc, R, t);
  const double tau2 = __dmul_rn(a.tau, a.tau);
  int cnt = 0;
  for (unsigned long long base = 0; base < nc; base += kGrT) {
    __syncthreads();
    const unsigned long long c = base + threadIdx.x;
    if (c < nc) {
      const unsigned long long si = (unsigned long long)a.corr[2 * c], ti = (unsigned long long)a.corr[2 * c + 1];
#pragma unroll
      for (int k = 0; k < 3; ++k) { sp[threadIdx.x][k] = a.src.xyz[3 * si + k]; sq[threadIdx.x][k] = a.tgt.xyz[3 * ti + k]; }
    }
    __syncthreads();
    if (!live) continue;
    const unsigned m = nc - base < kGrT ? (unsigned)(nc - base) : kGrT;
    for (unsigned k = 0; k < m; ++k) cnt += gr_res2(R, t, sp[k], sq[k]) < tau2 ? 1 : 0;
  }
  if (h < (unsigned)a.n_hypotheses) a.hyp_inliers[h] = live ? cnt : -1;
}

// one block: the valid hypotheses and the best (most inliers, the lower index on a tie), its T into the state
__global__ void __launch_bounds__(kGrT) k_gr_best(tloam_gr_args a) {
  __shared__ unsigned long long wkey[kGrT / 32];
  __shared__ unsigned wval[kGrT / 32];
  unsigned long long key = 0;
  unsigned valid = 0;
  for (unsigned h = threadIdx.x; h < (unsigned)a.n_hypotheses; h += kGrT) {
    const int v = a.hyp_inliers[h];
    if (v < 0) continue;
    ++valid;
    const unsigned long long k = ((unsigned long long)(v + 1) << 32) | (0xffffffffu - h);
    key = k > key ? k : key;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long k = __shfl_xor_sync(0xffffffffu, key, o);
    key = k > key ? k : key;
    valid += __shfl_xor_sync(0xffffffffu, valid, o);
  }
  if ((threadIdx.x & 31u) == 0) { wkey[threadIdx.x >> 5] = key; wval[threadIdx.x >> 5] = valid; }
  __syncthreads();
  if (threadIdx.x != 0) return;
  key = 0;
  valid = 0;
  for (unsigned w = 0; w < kGrT / 32; ++w) { key = wkey[w] > key ? wkey[w] : key; valid += wval[w]; }
  tloam_gr_state* s = a.state;
  const unsigned long long nc = s->n_corr;
  s->n_valid = (int)valid;
  double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, t[3] = {0, 0, 0};
  s->best = -1;
  s->best_inliers = 0;
  if (nc < 3) {
    s->term = kGrFewCorrespondences;
  } else if (valid == 0) {
    s->term = kGrNoHypothesis;
  } else {
    const unsigned h = 0xffffffffu - (unsigned)(key & 0xffffffffu);
    s->best = (int)h;
    s->best_inliers = (int)(key >> 32) - 1;
    s->term = kGrIterationLimit;
    gr_hypothesis(a, h, nc, R, t);
  }
  for (int k = 0; k < 9; ++k) s->R[k] = R[k];
  for (int k = 0; k < 3; ++k) s->t[k] = t[k];
}

// ---- refinement ---------------------------------------------------------------------------------------------------------
// cyclic Jacobi of the symmetric 4 x 4 a with nf_jacobi3's rules (at most 32 sweeps over (0,1), (0,2), (0,3), (1,2),
// (1,3), (2,3); a rotation skipped when its entry is 0; done once off <= 1e-32 diag); the eigenvector of the largest
// eigenvalue (the lower index on a tie) to q
__device__ __forceinline__ void gr_jacobi4(double a[4][4], double q[4]) {
  double v[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
  for (int sweep = 0; sweep < 32; ++sweep) {
    double off = 0.0, diag = 0.0;
    #pragma unroll
    for (int p = 0; p < 3; ++p)
      #pragma unroll
      for (int r = p + 1; r < 4; ++r) off = __dadd_rn(off, __dmul_rn(a[p][r], a[p][r]));
    #pragma unroll
    for (int p = 0; p < 4; ++p) diag = __dadd_rn(diag, __dmul_rn(a[p][p], a[p][p]));
    if (off <= __dmul_rn(1e-32, diag) || off == 0.0) break;
    #pragma unroll
    for (int p = 0; p < 3; ++p)
      #pragma unroll
      for (int r = p + 1; r < 4; ++r) {
        if (a[p][r] == 0.0) continue;
        const double theta = __ddiv_rn(__dsub_rn(a[r][r], a[p][p]), __dmul_rn(2.0, a[p][r]));
        const double tt = __ddiv_rn(theta >= 0 ? 1.0 : -1.0, __dadd_rn(fabs(theta), __dsqrt_rn(__dadd_rn(__dmul_rn(theta, theta), 1.0))));
        const double cs = __ddiv_rn(1.0, __dsqrt_rn(__dadd_rn(__dmul_rn(tt, tt), 1.0))), sn = __dmul_rn(tt, cs);
        #pragma unroll
        for (int k = 0; k < 4; ++k) {
          const double akp = a[k][p], akr = a[k][r];
          a[k][p] = __dsub_rn(__dmul_rn(cs, akp), __dmul_rn(sn, akr));
          a[k][r] = __dadd_rn(__dmul_rn(sn, akp), __dmul_rn(cs, akr));
        }
        #pragma unroll
        for (int k = 0; k < 4; ++k) {
          const double apk = a[p][k], ark = a[r][k];
          a[p][k] = __dsub_rn(__dmul_rn(cs, apk), __dmul_rn(sn, ark));
          a[r][k] = __dadd_rn(__dmul_rn(sn, apk), __dmul_rn(cs, ark));
        }
        #pragma unroll
        for (int k = 0; k < 4; ++k) {
          const double vkp = v[k][p], vkr = v[k][r];
          v[k][p] = __dsub_rn(__dmul_rn(cs, vkp), __dmul_rn(sn, vkr));
          v[k][r] = __dadd_rn(__dmul_rn(sn, vkp), __dmul_rn(cs, vkr));
        }
      }
  }
  int b = 0;
  #pragma unroll
  for (int k = 1; k < 4; ++k)
    if (a[k][k] > a[b][b]) b = k;
  #pragma unroll
  for (int k = 0; k < 4; ++k) q[k] = v[k][b];
}

// the least-squares rigid fit of the pairs in set (Horn 1987), on one thread: centroids and the cross-covariance summed in
// pair order, N's largest eigenvector q = (w, x, y, z) normalised, R from q, t = c_q - R c_p
__device__ __forceinline__ void gr_fit(const tloam_gr_args& a, unsigned long long nc, const unsigned char* set, int n, double R[9], double t[3]) {
  double cp[3] = {0, 0, 0}, cq[3] = {0, 0, 0};
  for (unsigned long long c = 0; c < nc; ++c) {
    if (!set[c]) continue;
    const double* p = a.src.xyz + 3ull * a.corr[2 * c];
    const double* q = a.tgt.xyz + 3ull * a.corr[2 * c + 1];
    for (int k = 0; k < 3; ++k) { cp[k] = __dadd_rn(cp[k], p[k]); cq[k] = __dadd_rn(cq[k], q[k]); }
  }
  const double dn = (double)n;
  for (int k = 0; k < 3; ++k) { cp[k] = __ddiv_rn(cp[k], dn); cq[k] = __ddiv_rn(cq[k], dn); }
  double S[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (unsigned long long c = 0; c < nc; ++c) {
    if (!set[c]) continue;
    const double* p = a.src.xyz + 3ull * a.corr[2 * c];
    const double* q = a.tgt.xyz + 3ull * a.corr[2 * c + 1];
    const double dp[3] = {__dsub_rn(p[0], cp[0]), __dsub_rn(p[1], cp[1]), __dsub_rn(p[2], cp[2])};
    const double dq[3] = {__dsub_rn(q[0], cq[0]), __dsub_rn(q[1], cq[1]), __dsub_rn(q[2], cq[2])};
#pragma unroll
    for (int u = 0; u < 3; ++u)
#pragma unroll
      for (int v = 0; v < 3; ++v) S[3 * u + v] = __dadd_rn(S[3 * u + v], __dmul_rn(dp[u], dq[v]));
  }
  const double xx = S[0], xy = S[1], xz = S[2], yx = S[3], yy = S[4], yz = S[5], zx = S[6], zy = S[7], zz = S[8];
  double N[4][4];
  N[0][0] = __dadd_rn(__dadd_rn(xx, yy), zz);
  N[1][1] = __dsub_rn(__dsub_rn(xx, yy), zz);
  N[2][2] = __dsub_rn(__dsub_rn(yy, xx), zz);
  N[3][3] = __dsub_rn(__dsub_rn(zz, xx), yy);
  N[0][1] = N[1][0] = __dsub_rn(yz, zy);
  N[0][2] = N[2][0] = __dsub_rn(zx, xz);
  N[0][3] = N[3][0] = __dsub_rn(xy, yx);
  N[1][2] = N[2][1] = __dadd_rn(xy, yx);
  N[1][3] = N[3][1] = __dadd_rn(zx, xz);
  N[2][3] = N[3][2] = __dadd_rn(yz, zy);
  double q[4];
  gr_jacobi4(N, q);
  const double qn = __dsqrt_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[0], q[0]), __dmul_rn(q[1], q[1])), __dmul_rn(q[2], q[2])),
                                         __dmul_rn(q[3], q[3])));
  const double w = __ddiv_rn(q[0], qn), x = __ddiv_rn(q[1], qn), y = __ddiv_rn(q[2], qn), z = __ddiv_rn(q[3], qn);
  const double ww = __dmul_rn(w, w), xx2 = __dmul_rn(x, x), yy2 = __dmul_rn(y, y), zz2 = __dmul_rn(z, z);
  const double wx = __dmul_rn(w, x), wy = __dmul_rn(w, y), wz = __dmul_rn(w, z);
  const double xy2 = __dmul_rn(x, y), xz2 = __dmul_rn(x, z), yz2 = __dmul_rn(y, z);
  R[0] = __dsub_rn(__dsub_rn(__dadd_rn(ww, xx2), yy2), zz2);
  R[1] = __dmul_rn(2.0, __dsub_rn(xy2, wz));
  R[2] = __dmul_rn(2.0, __dadd_rn(xz2, wy));
  R[3] = __dmul_rn(2.0, __dadd_rn(xy2, wz));
  R[4] = __dsub_rn(__dadd_rn(__dsub_rn(ww, xx2), yy2), zz2);
  R[5] = __dmul_rn(2.0, __dsub_rn(yz2, wx));
  R[6] = __dmul_rn(2.0, __dsub_rn(xz2, wy));
  R[7] = __dmul_rn(2.0, __dadd_rn(yz2, wx));
  R[8] = __dadd_rn(__dsub_rn(__dsub_rn(ww, xx2), yy2), zz2);
  for (int r = 0; r < 3; ++r) t[r] = __dsub_rn(cq[r], nf_dot3(R[3 * r], cp[0], R[3 * r + 1], cp[1], R[3 * r + 2], cp[2]));
}

// the pairs within tau under (R, t) into set (block-wide); returns their count and, with prev, whether set equals prev
__device__ int gr_mark(const tloam_gr_args& a, unsigned long long nc, const double* R, const double* t, unsigned char* set,
                       const unsigned char* prev, int* same) {
  __shared__ int cnt, diff;
  if (threadIdx.x == 0) { cnt = 0; diff = 0; }
  __syncthreads();
  const double tau2 = __dmul_rn(a.tau, a.tau);
  int mine = 0, d = 0;
  for (unsigned long long c = threadIdx.x; c < nc; c += kGrT) {
    const double* p = a.src.xyz + 3ull * a.corr[2 * c];
    const double* q = a.tgt.xyz + 3ull * a.corr[2 * c + 1];
    const unsigned char in = gr_res2(R, t, p, q) < tau2 ? 1 : 0;
    set[c] = in;
    mine += in;
    if (prev && prev[c] != in) d = 1;
  }
  atomicAdd(&cnt, mine);
  if (d) atomicOr(&diff, 1);
  __syncthreads();
  const int n = cnt;
  if (same) *same = diff == 0;
  __syncthreads();
  return n;
}

// one block: S0 = the best hypothesis's inliers; while fewer than max_refine_iterations fits and |S| >= 3: T = fit(S),
// S' = the pairs within tau under T, stop when S' = S; then the inliers, their rmse and the termination into the state
__global__ void __launch_bounds__(kGrT) k_gr_refine(tloam_gr_args a) {
  tloam_gr_state* st = a.state;
  if (st->best < 0) return;
  __shared__ double R[9], t[3];
  const unsigned long long nc = st->n_corr;
  if (threadIdx.x < 9) R[threadIdx.x] = st->R[threadIdx.x];
  if (threadIdx.x < 3) t[threadIdx.x] = st->t[threadIdx.x];
  __syncthreads();
  unsigned char* cur = a.in_set;
  unsigned char* nxt = a.in_set + a.src.n;
  int n = gr_mark(a, nc, R, t, cur, nullptr, nullptr), it = 0, term;
  for (;;) {
    if (it >= a.max_refine_iterations) { term = kGrIterationLimit; break; }
    if (n < 3) { term = kGrFewInliers; break; }
    if (threadIdx.x == 0) {
      double Rn[9], tn[3];
      gr_fit(a, nc, cur, n, Rn, tn);
      for (int k = 0; k < 9; ++k) R[k] = Rn[k];
      for (int k = 0; k < 3; ++k) t[k] = tn[k];
    }
    __syncthreads();
    ++it;
    int same = 0;
    n = gr_mark(a, nc, R, t, nxt, cur, &same);
    unsigned char* w = cur; cur = nxt; nxt = w;
    if (same) { term = kGrConverged; break; }
  }
  if (threadIdx.x != 0) return;
  double e = 0.0;
  for (unsigned long long c = 0; c < nc; ++c)
    if (cur[c]) e = __dadd_rn(e, gr_res2(R, t, a.src.xyz + 3ull * a.corr[2 * c], a.tgt.xyz + 3ull * a.corr[2 * c + 1]));
  st->rmse = n ? __dsqrt_rn(__ddiv_rn(e, (double)n)) : 0.0;
  for (int k = 0; k < 9; ++k) st->R[k] = R[k];
  for (int k = 0; k < 3; ++k) st->t[k] = t[k];
  st->inliers = n;
  st->iterations = it;
  st->term = term;
}

// one thread per source keypoint: whether a target keypoint lies within tau (d2 < tau^2) of T p, by the target's grid;
// the count into the state
__global__ void __launch_bounds__(kGrRows) k_gr_fitness(tloam_gr_args a) {
  const tloam_gr_state* st = a.state;
  const unsigned long long i = (unsigned long long)blockIdx.x * kGrRows + threadIdx.x;
  bool hit = false;
  if (i < a.src.n) {
    const double* p = a.src.xyz + 3 * i;
    const double x = __dadd_rn(nf_dot3(st->R[0], p[0], st->R[1], p[1], st->R[2], p[2]), st->t[0]);
    const double y = __dadd_rn(nf_dot3(st->R[3], p[0], st->R[4], p[1], st->R[5], p[2]), st->t[1]);
    const double z = __dadd_rn(nf_dot3(st->R[6], p[0], st->R[7], p[1], st->R[8], p[2]), st->t[2]);
    const double tau2 = __dmul_rn(a.tau, a.tau), rr = __dmul_ru(a.tau, kLocInflate);
    const tloam_loc_grid& g = a.tgt.grid;
    gr_walk(g, x, y, z, rr, [&](unsigned j) {
      if (!hit && nf_d2(x, y, z, g.sxyz[3ull * j], g.sxyz[3ull * j + 1], g.sxyz[3ull * j + 2]) < tau2) hit = true;
    });
  }
  const unsigned b = __ballot_sync(0xffffffffu, hit);
  if ((threadIdx.x & 31u) == 0 && b) atomicAdd(&a.state->fit_count, (unsigned long long)__popc(b));
}

static unsigned gr_blocks(unsigned long long n, unsigned t) { return (unsigned)((n + t - 1) / t); }

}  // namespace tloam

using namespace tloam;

#define TLOAM_GR_API extern "C" __attribute__((visibility("default")))

TLOAM_GR_API int tloam_gr_run(const tloam_gr_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(a->state, 0, sizeof(tloam_gr_state), a->stream)) != cudaSuccess) return (int)e;
  int nl = 0;
  for (const tloam_gr_side* s : {&a->src, &a->tgt}) {
    if ((e = cudaMemsetAsync(s->spfh, 0, (size_t)s->n * kGrB * sizeof(int), a->stream)) != cudaSuccess) return (int)e;
    k_gr_orient<<<gr_blocks(s->n, kGrRows), kGrRows, 0, a->stream>>>(*s);
    k_gr_spfh<<<gr_blocks(s->n, kGrRows), kGrRows, 0, a->stream>>>(*s, a->feature_radius, *a);
    k_gr_fpfh<<<gr_blocks(s->n, kGrRows), kGrRows, 0, a->stream>>>(*s, a->feature_radius);
    nl += 3;
  }
  k_gr_match<<<gr_blocks(a->src.n, kGrRows), kGrRows, 0, a->stream>>>(a->src, a->tgt, a->src.nn);
  k_gr_match<<<gr_blocks(a->tgt.n, kGrRows), kGrRows, 0, a->stream>>>(a->tgt, a->src, a->tgt.nn);
  k_gr_mutual<<<1, kGrOneBlock, 0, a->stream>>>(*a);
  k_gr_hyp<<<gr_blocks((unsigned long long)a->n_hypotheses, kGrT), kGrT, 0, a->stream>>>(*a);
  k_gr_best<<<1, kGrT, 0, a->stream>>>(*a);
  k_gr_refine<<<1, kGrT, 0, a->stream>>>(*a);
  k_gr_fitness<<<gr_blocks(a->src.n, kGrRows), kGrRows, 0, a->stream>>>(*a);
  *launches = nl + 7;
  return (int)cudaGetLastError();
}
