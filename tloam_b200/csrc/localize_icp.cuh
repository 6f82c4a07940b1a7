// localize_icp.cuh -- the grid search and the point-to-plane ICP of localization in a prior map, as device functions over
// one run's state, partial sums and match records.  localize.cu runs them for one localization (k_loc_*), relocalize.cu
// for a batch of hypotheses (k_rl_*), so every hypothesis is exactly one localization.  The definition is in
// include/tloam_b200.h ("Localization in a prior map").
#pragma once
#include <cuda_runtime.h>
#include <math.h>

#include "ldlt6.cuh"
#include "localize.h"
#include "normal_fit.cuh"
#include "se3.cuh"

namespace tloam {

// the buffers of one run, read where the body uses them: LocRun is the run of tloam_loc_args itself; a batch supplies a
// type with the same members for each of its runs
struct LocRun {
  const tloam_loc_args& a;
  __device__ __forceinline__ tloam_loc_state* state() const { return a.state; }
  __device__ __forceinline__ double* sums() const { return a.sums; }
  __device__ __forceinline__ int* match_index() const { return a.match_index; }
  __device__ __forceinline__ double* match_d2() const { return a.match_d2; }
};

enum { kLocConverged = 0, kLocIterationLimit = 1, kLocFewInliers = 2, kLocSingular = 3, kLocEmpty = 4 };
constexpr unsigned kLocT = TLOAM_LOC_THREADS;
constexpr double kLocInflate = 1.0 + 1e-7;

__device__ __forceinline__ void loc_apply(const tloam_loc_state* s, double qx, double qy, double qz, double& px, double& py,
                                          double& pz) {
  px = __dadd_rn(nf_dot3(s->R[0], qx, s->R[1], qy, s->R[2], qz), s->t[0]);
  py = __dadd_rn(nf_dot3(s->R[3], qx, s->R[4], qy, s->R[5], qz), s->t[1]);
  pz = __dadd_rn(nf_dot3(s->R[6], qx, s->R[7], qy, s->R[8], qz), s->t[2]);
}

__device__ __forceinline__ unsigned long long loc_key(const tloam_loc_grid& g, long long ix, long long iy, long long iz) {
  return ((unsigned long long)ix << (g.bits[1] + g.bits[2])) | ((unsigned long long)iy << g.bits[2]) | (unsigned long long)iz;
}

// the cells of axis d that can hold a row within rr of p: [lo, hi], clipped to the map's cells (empty when lo > hi)
__device__ __forceinline__ void loc_range(const tloam_loc_grid& g, int d, double p, double rr, long long& lo, long long& hi) {
  double l = floor(__ddiv_rn(__dsub_rn(__dsub_rd(p, rr), g.mb[d]), g.cell));
  double h = floor(__ddiv_rn(__dsub_rn(__dadd_ru(p, rr), g.mb[d]), g.cell));
  l = fmax(l, 0.0);
  h = fmin(h, (double)g.top[d]);
  lo = (long long)l;
  hi = h < l ? lo - 1 : (long long)h;
}

// the first cell with key >= k (strict: > k)
__device__ __forceinline__ unsigned loc_bound(const unsigned long long* ckey, unsigned n, unsigned long long k, bool strict) {
  unsigned lo = 0, hi = n;
  while (lo < hi) {
    const unsigned mid = (lo + hi) >> 1;
    const unsigned long long v = ckey[mid];
    if (strict ? v <= k : v < k) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// the sorted positions of column (ix, iy), cells iz_lo .. iz_hi: one run, since the key orders z last
__device__ __forceinline__ void loc_column(const tloam_loc_grid& g, unsigned n_cells, long long ix, long long iy, long long zlo,
                                           long long zhi, unsigned& s, unsigned& e) {
  const unsigned c0 = loc_bound(g.ckey, n_cells, loc_key(g, ix, iy, zlo), false);
  const unsigned c1 = loc_bound(g.ckey, n_cells, loc_key(g, ix, iy, zhi), true);
  s = g.cstart[c0];
  e = g.cstart[c1];
}

// one thread per query row (blockIdx.x: the query block): p = R q + t and its nearest map row within the pass's radius
// (s->r, corr_dist_coarse for the final pass) by (d2, row index), recorded at slot `pass` (the final pass: s->iter) of
// match_index / match_d2.  k_mu_novel (map_update.cu) walks the same cells and columns for an existence test: a change to
// the cell rule here changes it there too.
template <class Run>
__device__ __forceinline__ void loc_match_run(const tloam_loc_args& a, const Run& run, int pass, int final_pass) {
  const tloam_loc_state* s = run.state();
  if (!final_pass && s->done) return;
  const unsigned long long i = blockIdx.x * (unsigned long long)kLocT + threadIdx.x;
  if (i >= a.nq) return;
  const tloam_loc_grid& g = a.grid;
  const unsigned n_cells = (unsigned)g.st->n_vox;
  double px, py, pz;
  loc_apply(s, a.query[3 * i], a.query[3 * i + 1], a.query[3 * i + 2], px, py, pz);
  const double r = final_pass ? a.corr_dist_coarse : s->r;
  const double r2 = __dmul_rn(r, r), rr = __dmul_ru(r, kLocInflate);
  long long lx, hx, ly, hy, lz, hz;
  loc_range(g, 0, px, rr, lx, hx);
  loc_range(g, 1, py, rr, ly, hy);
  loc_range(g, 2, pz, rr, lz, hz);
  double best = INFINITY;
  unsigned bi = 0xffffffffu;
  if (lz <= hz)
    for (long long ix = lx; ix <= hx; ++ix)
      for (long long iy = ly; iy <= hy; ++iy) {
        unsigned j0, j1;
        loc_column(g, n_cells, ix, iy, lz, hz, j0, j1);
        for (unsigned j = j0; j < j1; ++j) {
          const double d2 = nf_d2(px, py, pz, g.sxyz[3ull * j], g.sxyz[3ull * j + 1], g.sxyz[3ull * j + 2]);
          if (d2 <= r2) {
            const unsigned v = g.srow[j];
            if (d2 < best || (d2 == best && v < bi)) { best = d2; bi = v; }
          }
        }
      }
  const size_t slot = (size_t)(final_pass ? s->iter : pass) * a.nq + i;
  run.match_index()[slot] = bi == 0xffffffffu ? -1 : (int)bi;
  run.match_d2()[slot] = best;
}

// one thread per query row: for a match within the inlier radius (s->r, corr_dist_fine for the final pass) whose map row
// has a valid normal n, the row's contribution to H = sum J^T J and g = sum J^T e with e = n . (p - m), J = [n, p x n];
// the contributing rows, sum e^2 over them and sum min(d2, coarse^2) over every row; reduced per block in a fixed order
// into sums[blockIdx.x]
template <class Run>
__device__ __forceinline__ void loc_reduce_run(const tloam_loc_args& a, const Run& run, int pass, int final_pass) {
  const tloam_loc_state* s = run.state();
  if (!final_pass && s->done) return;
  const unsigned long long i = blockIdx.x * (unsigned long long)kLocT + threadIdx.x;
  double v[TLOAM_LOC_SUMS];
#pragma unroll
  for (int k = 0; k < TLOAM_LOC_SUMS; ++k) v[k] = 0.0;
  if (i < a.nq) {
    const size_t slot = (size_t)(final_pass ? s->iter : pass) * a.nq + i;
    const int bi = run.match_index()[slot];
    const double d2 = run.match_d2()[slot];
    const double r = final_pass ? a.corr_dist_fine : s->r;
    v[29] = bi >= 0 ? d2 : __dmul_rn(a.corr_dist_coarse, a.corr_dist_coarse);
    if (bi >= 0 && d2 <= __dmul_rn(r, r) && a.valid[bi]) {
      double p[3];
      loc_apply(s, a.query[3 * i], a.query[3 * i + 1], a.query[3 * i + 2], p[0], p[1], p[2]);
      const double* m = a.map + 3 * (unsigned long long)bi;
      const double* n = a.normal + 3 * (unsigned long long)bi;
      const double e = nf_dot3(n[0], __dsub_rn(p[0], m[0]), n[1], __dsub_rn(p[1], m[1]), n[2], __dsub_rn(p[2], m[2]));
      const double J[6] = {n[0], n[1], n[2], p[1] * n[2] - p[2] * n[1], p[2] * n[0] - p[0] * n[2], p[0] * n[1] - p[1] * n[0]};
#pragma unroll
      for (int u = 0; u < 6; ++u) {
#pragma unroll
        for (int w = 0; w < 6; ++w)
          if (w >= u) v[tri(u, w)] = J[u] * J[w];
        v[21 + u] = J[u] * e;
      }
      v[27] = 1.0;
      v[28] = e * e;
    }
  }
  __shared__ double ws[kLocT / 32][TLOAM_LOC_SUMS];
#pragma unroll
  for (int k = 0; k < TLOAM_LOC_SUMS; ++k) {
    double x = v[k];
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5][k] = x;
  }
  __syncthreads();
  if (threadIdx.x < TLOAM_LOC_SUMS) {
    double x = 0.0;
    for (unsigned w = 0; w < kLocT / 32; ++w) x += ws[w][threadIdx.x];
    run.sums()[blockIdx.x * (size_t)TLOAM_LOC_SUMS + threadIdx.x] = x;
  }
}

// the block partials summed in block order (thread k: entry k)
__device__ void loc_total(const tloam_loc_args& a, const double* sums, double* tot) {
  const unsigned nb = (unsigned)((a.nq + kLocT - 1) / kLocT);
  if (threadIdx.x < TLOAM_LOC_SUMS) {
    double x = 0.0;
    for (unsigned b = 0; b < nb; ++b) x += sums[b * (size_t)TLOAM_LOC_SUMS + threadIdx.x];
    tot[threadIdx.x] = x;
  }
  __syncwarp();
}

// one thread, from a run's totals: delta = -H^-1 g by LDL^T, T <- exp(delta) . T, then the radius schedule and the
// termination
__device__ __forceinline__ void loc_step_solve(tloam_loc_state* s, const double* tot, double eps_translation, double eps_rotation,
                                               double corr_dist_fine, int max_iterations) {
  if (tot[27] < 6.0) { s->term = kLocFewInliers; s->done = 1; return; }
  double A[21], b[6], y[6];
  for (int k = 0; k < 21; ++k) A[k] = tot[k];
  for (int k = 0; k < 6; ++k) b[k] = tot[21 + k];
  if (!ldlt_solve6_packed(A, b, y)) { s->term = kLocSingular; s->done = 1; return; }
  double d[6];
  for (int k = 0; k < 6; ++k) d[k] = -y[k];
  const Pose7 e = se3_exp(d);
  double Re[9];
  quat_to_rot(e, Re);
  const double te[3] = {e.tx, e.ty, e.tz};
  double R[9], t[3];
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) R[3 * r + c] = nf_dot3(Re[3 * r], s->R[c], Re[3 * r + 1], s->R[3 + c], Re[3 * r + 2], s->R[6 + c]);
    t[r] = __dadd_rn(nf_dot3(Re[3 * r], s->t[0], Re[3 * r + 1], s->t[1], Re[3 * r + 2], s->t[2]), te[r]);
  }
  for (int k = 0; k < 9; ++k) s->R[k] = R[k];
  for (int k = 0; k < 3; ++k) s->t[k] = t[k];
  s->iter += 1;
  const double nu = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), nw = sqrt(d[3] * d[3] + d[4] * d[4] + d[5] * d[5]);
  if (nu < eps_translation && nw < eps_rotation) {
    if (s->r == corr_dist_fine) { s->term = kLocConverged; s->done = 1; return; }
    s->r = fmax(s->r * 0.5, corr_dist_fine);
  }
  if (s->iter >= max_iterations) { s->term = kLocIterationLimit; s->done = 1; }
}

// one warp: the final pass's contributing rows, their rmse, the fitness; accepted; T_map_odom = T . O_now^-1:
//   R_M(r, c) = (R_T(r, 0) R_O(c, 0) + R_T(r, 1) R_O(c, 1)) + R_T(r, 2) R_O(c, 2)
//   t_M(r)    = t_T(r) - ((R_M(r, 0) t_O(0) + R_M(r, 1) t_O(1)) + R_M(r, 2) t_O(2))
// and, with kMemory, the prediction's memory: L = T if accepted else G, O = O_now
template <bool kMemory, class Run>
__device__ __forceinline__ void loc_final_run(const tloam_loc_args& a, const Run& run) {
  tloam_loc_state* s = run.state();
  __shared__ double tot[TLOAM_LOC_SUMS];
  loc_total(a, run.sums(), tot);
  if (threadIdx.x != 0) return;
  if (a.nq == 0) {
    s->inliers = 0; s->rmse = 0.0; s->fitness = INFINITY;
  } else {
    s->inliers = (unsigned long long)tot[27];
    s->rmse = tot[27] > 0.0 ? sqrt(tot[28] / tot[27]) : 0.0;
    s->fitness = tot[29] / (double)a.nq;
  }
  s->accepted = s->term == kLocConverged && s->fitness <= a.max_fitness ? 1 : 0;
  double T[16];
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) T[4 * c + r] = s->R[3 * r + c];
    T[12 + r] = s->t[r];
    T[4 * r + 3] = 0.0;
  }
  T[15] = 1.0;
  const double* O = s->odom;
  double* M = s->map_odom;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) M[4 * c + r] = nf_dot3(T[r], O[c], T[4 + r], O[4 + c], T[8 + r], O[8 + c]);
    M[12 + r] = __dsub_rn(T[12 + r], nf_dot3(M[r], O[12], M[4 + r], O[13], M[8 + r], O[14]));
    M[4 * r + 3] = 0.0;
  }
  M[15] = 1.0;
  if (kMemory)
    for (int k = 0; k < 16; ++k) {
      a.memory->L[k] = s->accepted ? T[k] : s->guess[k];
      a.memory->O[k] = O[k];
    }
}

}  // namespace tloam
