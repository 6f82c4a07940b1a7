// loop_verify_submap.cu -- libtloam_b200_loopvs.so: verification of a loop candidate against the submap of the keyframes
// around it (hand-written CUDA for sm_90a).  The target is the union of the window's keyframes in the candidate's sensor
// frame, every target row gets a normal from the covariance of its neighbourhood, and the ICP is loop_verify.cu's with a
// point-to-plane residual over the rows whose match has a valid normal.  The full definition is in include/tloam_b200.h
// ("Loop verification against a submap"); tests/loop_verify_submap_oracle.py restates it in numpy.
//
// Everything up to the first pass's matches is separately rounded __d*_rn in the order the header writes, the neighbourhood
// sums run in ascending row order inside one thread, and the eigen-solve is a fixed cyclic Jacobi, so the target, the
// neighbour counts, the normals and the first pass are bit-reproducible on the host.  The normal equations are reduced in
// a fixed order (warp butterfly, warps in order, blocks in order), so a run is bit-deterministic.
//
// A separate library so that the kernels of libtloam_b200.so and libtloam_b200_loopv.so keep their SASS.
#include <cuda_runtime.h>
#include <math.h>

#include "ldlt6.cuh"
#include "loop_verify_submap.h"
#include "normal_fit.cuh"
#include "se3.cuh"

namespace tloam {

enum { kLvsConverged = 0, kLvsIterationLimit = 1, kLvsFewInliers = 2, kLvsSingular = 3 };
constexpr unsigned kLvsT = TLOAM_LVS_THREADS;
constexpr unsigned kLvsN = TLOAM_LVS_NORMAL_THREADS;

__device__ __forceinline__ double lvs_dot3(double a0, double b0, double a1, double b1, double a2, double b2) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a0, b0), __dmul_rn(a1, b1)), __dmul_rn(a2, b2));
}

__device__ __forceinline__ double lvs_d2(double px, double py, double pz, double mx, double my, double mz) {
  const double dx = __dsub_rn(px, mx), dy = __dsub_rn(py, my), dz = __dsub_rn(pz, mz);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

__device__ __forceinline__ void lvs_apply(const tloam_lv_state* s, double qx, double qy, double qz, double& px, double& py,
                                          double& pz) {
  px = __dadd_rn(lvs_dot3(s->R[0], qx, s->R[1], qy, s->R[2], qz), s->t[0]);
  py = __dadd_rn(lvs_dot3(s->R[3], qx, s->R[4], qy, s->R[5], qz), s->t[1]);
  pz = __dadd_rn(lvs_dot3(s->R[6], qx, s->R[7], qy, s->R[8], qz), s->t[2]);
}

// (d2, index) order; index -1 (no row) is above everything
__device__ __forceinline__ bool lvs_better(double d2, long long j, const tloam_lv_best& b) {
  return j >= 0 && (b.index < 0 || d2 < b.d2 || (d2 == b.d2 && j < b.index));
}

// a thread per window frame w: A_w = O_c^-1 O_(lo + w): R(r, c) = sum_k R_c(k, r) R_j(k, c), t(r) = sum_k R_c(k, r) (t_j(k) -
// t_c(k)); column-major 4 x 4
__global__ void k_lvs_poses(tloam_lvs_args a) {
  const unsigned long long w = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (w > a.hi - a.lo) return;
  const double* Oc = a.poses + 16 * (a.candidate - a.lo);
  const double* Oj = a.poses + 16 * w;
  double* A = a.A + 16 * w;
  const double d[3] = {__dsub_rn(Oj[12], Oc[12]), __dsub_rn(Oj[13], Oc[13]), __dsub_rn(Oj[14], Oc[14])};
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c)
      A[4 * c + r] = lvs_dot3(Oc[4 * r], Oj[4 * c], Oc[4 * r + 1], Oj[4 * c + 1], Oc[4 * r + 2], Oj[4 * c + 2]);
    A[12 + r] = lvs_dot3(Oc[4 * r], d[0], Oc[4 * r + 1], d[1], Oc[4 * r + 2], d[2]);
    A[4 * r + 3] = 0.0;
  }
  A[15] = 1.0;
}

// a thread per target row i: its store row (the window's rows in order, the query's left out), its frame by binary search
// over the window's slice of the keyframe table (the last f with offsets[f] <= row), then A_f p; the candidate's own rows
// are copied
__global__ void __launch_bounds__(kLvsT) k_lvs_assemble(tloam_lvs_args a) {
  const unsigned long long i = (unsigned long long)blockIdx.x * kLvsT + threadIdx.x;
  if (i >= a.nm) return;
  unsigned long long s = a.base + i;
  if (a.query_in_window && s >= a.q0) s += a.nq;
  unsigned long long lo = a.lo, hi = a.hi;
  while (lo < hi) {
    const unsigned long long mid = (lo + hi + 1) / 2;
    if (a.offsets[mid] <= s) lo = mid;
    else hi = mid - 1;
  }
  const double x = a.pts[3 * s], y = a.pts[3 * s + 1], z = a.pts[3 * s + 2];
  double* o = a.target + 3 * i;
  if (lo == a.candidate) { o[0] = x; o[1] = y; o[2] = z; return; }
  const double* A = a.A + 16 * (lo - a.lo);
  for (int r = 0; r < 3; ++r) o[r] = __dadd_rn(lvs_dot3(A[r], x, A[4 + r], y, A[8 + r], z), A[12 + r]);
}

// a thread per target row i; the whole target streamed through shared memory in tiles of kLvsN in ascending row order,
// twice: the first sweep counts the rows within normal_radius and sums them, the second sums the products of their
// offsets from the mean.  Each thread adds its neighbours in ascending row order.
__global__ void __launch_bounds__(kLvsN) k_lvs_normals(tloam_lvs_args a) {
  __shared__ double sx[kLvsN], sy[kLvsN], sz[kLvsN];
  const unsigned long long i = (unsigned long long)blockIdx.x * kLvsN + threadIdx.x;
  const bool have = i < a.nm;
  const double px = have ? a.target[3 * i] : 0.0, py = have ? a.target[3 * i + 1] : 0.0, pz = have ? a.target[3 * i + 2] : 0.0;
  const double r2 = __dmul_rn(a.normal_radius, a.normal_radius);
  int cnt = 0;
  double mx = 0.0, my = 0.0, mz = 0.0;
  double c[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int sweep = 0; sweep < 2; ++sweep) {
    for (unsigned long long base = 0; base < a.nm; base += kLvsN) {
      __syncthreads();
      const unsigned long long j = base + threadIdx.x;
      if (j < a.nm) { sx[threadIdx.x] = a.target[3 * j]; sy[threadIdx.x] = a.target[3 * j + 1]; sz[threadIdx.x] = a.target[3 * j + 2]; }
      __syncthreads();
      const int n = (int)(a.nm - base < kLvsN ? a.nm - base : kLvsN);
      if (!have) continue;
      if (sweep == 0) {
        for (int k = 0; k < n; ++k) {
          const double x = sx[k], y = sy[k], z = sz[k];
          if (lvs_d2(px, py, pz, x, y, z) <= r2) {
            cnt += 1;
            mx = __dadd_rn(mx, x); my = __dadd_rn(my, y); mz = __dadd_rn(mz, z);
          }
        }
      } else {
        for (int k = 0; k < n; ++k) {
          const double x = sx[k], y = sy[k], z = sz[k];
          if (lvs_d2(px, py, pz, x, y, z) <= r2) nf_cov_add(c, x, y, z, mx, my, mz);
        }
      }
    }
    if (sweep == 0) {                   // a row is its own neighbour: cnt >= 1
      const double n = (double)cnt;
      mx = __ddiv_rn(mx, n); my = __ddiv_rn(my, n); mz = __ddiv_rn(mz, n);
    }
  }
  if (!have) return;
  double nv[3];
  const unsigned char ok = nf_finish(cnt, c, a.min_normal_neighbours, a.max_planarity, nv);
  a.normal[3 * i] = nv[0]; a.normal[3 * i + 1] = nv[1]; a.normal[3 * i + 2] = nv[2];
  a.neighbours[i] = cnt;
  a.valid[i] = ok;
}

// grid (query blocks, splits): thread i of block (x, y) takes query row x * kLvsT + i and the rows of slice y of the
// target, streamed through shared memory in tiles of kLvsT; the slice's nearest row (lowest index on a tie) goes to
// part[y * nq + i]
__global__ void __launch_bounds__(kLvsT) k_lvs_match(tloam_lvs_args a, int final_pass) {
  const tloam_lv_state* s = a.state;
  if (!final_pass && s->done) return;
  __shared__ double sx[kLvsT], sy[kLvsT], sz[kLvsT];
  const unsigned long long i = blockIdx.x * (unsigned long long)kLvsT + threadIdx.x;
  const bool have = i < a.nq;
  double px = 0.0, py = 0.0, pz = 0.0;
  if (have) lvs_apply(s, a.pts[3 * (a.q0 + i)], a.pts[3 * (a.q0 + i) + 1], a.pts[3 * (a.q0 + i) + 2], px, py, pz);
  const unsigned long long per = (a.nm + a.splits - 1) / a.splits;
  const unsigned long long j0 = blockIdx.y * per, j1 = j0 + per < a.nm ? j0 + per : a.nm;
  double best = INFINITY;
  long long bi = -1;
  for (unsigned long long base = j0; base < j1; base += kLvsT) {
    __syncthreads();
    const unsigned long long j = base + threadIdx.x;
    if (j < j1) { sx[threadIdx.x] = a.target[3 * j]; sy[threadIdx.x] = a.target[3 * j + 1]; sz[threadIdx.x] = a.target[3 * j + 2]; }
    __syncthreads();
    const int cnt = (int)(j1 - base < kLvsT ? j1 - base : kLvsT);
    if (have)
      for (int k = 0; k < cnt; ++k) {
        const double d2 = lvs_d2(px, py, pz, sx[k], sy[k], sz[k]);
        if (d2 < best) { best = d2; bi = (long long)(base + k); }
      }
  }
  if (have) a.part[blockIdx.y * a.nq + i] = tloam_lv_best{best, bi};
}

// one thread per query row: the slices merged, the pass's match recorded, and, for an inlier (d2 <= r * r) whose match has
// a valid normal n, the row's contribution to H = sum J^T J and g = sum J^T e with e = n . (p - m), J = [n, p x n]; the
// contributing rows, sum e^2 over them and sum d2 over every row; reduced per block in a fixed order into a.sums.
// pass: the slot of match_index / match_d2 (the final pass uses state->iter).
__global__ void __launch_bounds__(kLvsT) k_lvs_reduce(tloam_lvs_args a, int pass, int final_pass) {
  const tloam_lv_state* s = a.state;
  if (!final_pass && s->done) return;
  const unsigned long long i = blockIdx.x * (unsigned long long)kLvsT + threadIdx.x;
  double v[TLOAM_LVS_SUMS];
#pragma unroll
  for (int k = 0; k < TLOAM_LVS_SUMS; ++k) v[k] = 0.0;
  if (i < a.nq) {
    tloam_lv_best b{INFINITY, -1};
    for (unsigned y = 0; y < a.splits; ++y) {
      const tloam_lv_best c = a.part[y * a.nq + i];
      if (lvs_better(c.d2, c.index, b)) b = c;
    }
    const size_t slot = (size_t)(final_pass ? s->iter : pass) * a.nq + i;
    a.match_index[slot] = (int)b.index;
    a.match_d2[slot] = b.d2;
    const double r = final_pass ? a.corr_dist_fine : s->r;
    v[29] = b.d2;
    if (b.index >= 0 && b.d2 <= __dmul_rn(r, r) && a.valid[b.index]) {
      double p[3];
      lvs_apply(s, a.pts[3 * (a.q0 + i)], a.pts[3 * (a.q0 + i) + 1], a.pts[3 * (a.q0 + i) + 2], p[0], p[1], p[2]);
      const double* m = a.target + 3 * (unsigned long long)b.index;
      const double* n = a.normal + 3 * (unsigned long long)b.index;
      const double e = lvs_dot3(n[0], __dsub_rn(p[0], m[0]), n[1], __dsub_rn(p[1], m[1]), n[2], __dsub_rn(p[2], m[2]));
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
  __shared__ double ws[kLvsT / 32][TLOAM_LVS_SUMS];
#pragma unroll
  for (int k = 0; k < TLOAM_LVS_SUMS; ++k) {
    double x = v[k];
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5][k] = x;
  }
  __syncthreads();
  if (threadIdx.x < TLOAM_LVS_SUMS) {
    double x = 0.0;
    for (unsigned w = 0; w < kLvsT / 32; ++w) x += ws[w][threadIdx.x];
    a.sums[blockIdx.x * (size_t)TLOAM_LVS_SUMS + threadIdx.x] = x;
  }
}

// the block partials summed in block order (thread k: entry k)
__device__ void lvs_total(const tloam_lvs_args& a, double* tot) {
  const unsigned nb = (unsigned)((a.nq + kLvsT - 1) / kLvsT);
  if (threadIdx.x < TLOAM_LVS_SUMS) {
    double x = 0.0;
    for (unsigned b = 0; b < nb; ++b) x += a.sums[b * (size_t)TLOAM_LVS_SUMS + threadIdx.x];
    tot[threadIdx.x] = x;
  }
  __syncwarp();
}

// one warp: delta = -H^-1 g by LDL^T, T <- exp(delta) . T, then the radius schedule and the termination
__global__ void k_lvs_step(tloam_lvs_args a) {
  tloam_lv_state* s = a.state;
  if (s->done) return;
  __shared__ double tot[TLOAM_LVS_SUMS];
  lvs_total(a, tot);
  if (threadIdx.x != 0) return;
  if (tot[27] < 6.0) { s->term = kLvsFewInliers; s->done = 1; return; }
  double A[21], b[6], y[6];
  for (int k = 0; k < 21; ++k) A[k] = tot[k];
  for (int k = 0; k < 6; ++k) b[k] = tot[21 + k];
  if (!ldlt_solve6_packed(A, b, y)) { s->term = kLvsSingular; s->done = 1; return; }
  double d[6];
  for (int k = 0; k < 6; ++k) d[k] = -y[k];
  const Pose7 e = se3_exp(d);
  double Re[9];
  quat_to_rot(e, Re);
  const double te[3] = {e.tx, e.ty, e.tz};
  double R[9], t[3];
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) R[3 * r + c] = lvs_dot3(Re[3 * r], s->R[c], Re[3 * r + 1], s->R[3 + c], Re[3 * r + 2], s->R[6 + c]);
    t[r] = __dadd_rn(lvs_dot3(Re[3 * r], s->t[0], Re[3 * r + 1], s->t[1], Re[3 * r + 2], s->t[2]), te[r]);
  }
  for (int k = 0; k < 9; ++k) s->R[k] = R[k];
  for (int k = 0; k < 3; ++k) s->t[k] = t[k];
  s->iter += 1;
  const double nu = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), nw = sqrt(d[3] * d[3] + d[4] * d[4] + d[5] * d[5]);
  if (nu < a.eps_translation && nw < a.eps_rotation) {
    if (s->r == a.corr_dist_fine) { s->term = kLvsConverged; s->done = 1; return; }
    s->r = fmax(s->r * 0.5, a.corr_dist_fine);
  }
  if (s->iter >= a.max_iterations) { s->term = kLvsIterationLimit; s->done = 1; }
}

// one warp: the final pass's contributing rows, the rmse of their point-to-plane residual, fitness = mean d2 over every
// query row
__global__ void k_lvs_final(tloam_lvs_args a) {
  tloam_lv_state* s = a.state;
  __shared__ double tot[TLOAM_LVS_SUMS];
  lvs_total(a, tot);
  if (threadIdx.x != 0) return;
  s->inliers = (unsigned long long)tot[27];
  s->rmse = tot[27] > 0.0 ? sqrt(tot[28] / tot[27]) : 0.0;
  s->fitness = tot[29] / (double)a.nq;
}

}  // namespace tloam

using namespace tloam;

#define TLOAM_LVS_API extern "C" __attribute__((visibility("default")))

TLOAM_LVS_API int tloam_lvs_verify(const tloam_lvs_args* a, int* launches) {
  cudaError_t e = cudaSetDevice(a->device);
  *launches = 0;
  if (e != cudaSuccess) return (int)e;
  const unsigned n_win = (unsigned)(a->hi - a->lo + 1);
  k_lvs_poses<<<(n_win + 127) / 128, 128, 0, a->stream>>>(*a);
  k_lvs_assemble<<<(unsigned)((a->nm + kLvsT - 1) / kLvsT), kLvsT, 0, a->stream>>>(*a);
  k_lvs_normals<<<(unsigned)((a->nm + kLvsN - 1) / kLvsN), kLvsN, 0, a->stream>>>(*a);
  *launches += 3;
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  const unsigned qb = (unsigned)((a->nq + kLvsT - 1) / kLvsT);
  const dim3 grid(qb, a->splits);
  for (int k = 0; k <= a->max_iterations; ++k) {
    const int fin = k == a->max_iterations;
    k_lvs_match<<<grid, kLvsT, 0, a->stream>>>(*a, fin);
    k_lvs_reduce<<<qb, kLvsT, 0, a->stream>>>(*a, k, fin);
    if (fin) k_lvs_final<<<1, 32, 0, a->stream>>>(*a);
    else k_lvs_step<<<1, 32, 0, a->stream>>>(*a);
    *launches += 3;
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  }
  return (int)cudaSuccess;
}
