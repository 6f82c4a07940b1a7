// loop_verify.cu -- libtloam_b200_loopv.so: geometric verification of loop candidates on the device (hand-written CUDA for
// sm_90a).  A point-to-point ICP of one down-sampled keyframe (the query Q) against another (the candidate M), Gauss-Newton
// on SE(3) with a left perturbation and a correspondence radius that halves down to its fine value; plus the commit that
// closes each keyframe slot of the store libtloam_b200.so fills.  The full definition is in include/tloam_b200.h ("Loop
// verification"); tests/loop_verify_oracle.py restates it in numpy.
//
// The correspondence of a query row is an exact brute-force nearest neighbour over the whole candidate keyframe: p = R q + t
// and d2 = ((px - mx)^2 + (py - my)^2) + (pz - mz)^2 are separately rounded __d*_rn, the lowest index wins a tie, so the
// first pass (at the caller's T) is bit-reproducible on the host.  The normal equations are reduced in a fixed order
// (warp butterfly, warps in order, blocks in order), so a run is bit-deterministic.
//
// A separate library so that the kernels of libtloam_b200.so and libtloam_b200_loop.so keep their SASS.
#include <cuda_runtime.h>
#include <math.h>

#include "ldlt6.cuh"
#include "loop_verify.h"
#include "se3.cuh"

namespace tloam {

enum { kLvConverged = 0, kLvIterationLimit = 1, kLvFewInliers = 2, kLvSingular = 3 };
constexpr unsigned kLvT = TLOAM_LV_THREADS;

__device__ __forceinline__ void lv_apply(const tloam_lv_state* s, double qx, double qy, double qz, double& px, double& py,
                                         double& pz) {
  px = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(s->R[0], qx), __dmul_rn(s->R[1], qy)), __dmul_rn(s->R[2], qz)), s->t[0]);
  py = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(s->R[3], qx), __dmul_rn(s->R[4], qy)), __dmul_rn(s->R[5], qz)), s->t[1]);
  pz = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(s->R[6], qx), __dmul_rn(s->R[7], qy)), __dmul_rn(s->R[8], qz)), s->t[2]);
}

// (d2, index) order; index -1 (no row) is above everything
__device__ __forceinline__ bool lv_better(double d2, long long j, const tloam_lv_best& b) {
  return j >= 0 && (b.index < 0 || d2 < b.d2 || (d2 == b.d2 && j < b.index));
}

// grid (query blocks, splits): thread i of block (x, y) takes query row x * kLvT + i and the rows of slice y of M, streamed
// through shared memory in tiles of kLvT; the slice's nearest row (lowest index on a tie) goes to part[y * nq + i]
__global__ void __launch_bounds__(kLvT) k_lv_match(tloam_lv_args a, int final_pass) {
  const tloam_lv_state* s = a.state;
  if (!final_pass && s->done) return;
  __shared__ double sx[kLvT], sy[kLvT], sz[kLvT];
  const unsigned long long i = blockIdx.x * (unsigned long long)kLvT + threadIdx.x;
  const bool have = i < a.nq;
  double px = 0.0, py = 0.0, pz = 0.0;
  if (have) lv_apply(s, a.pts[3 * (a.q0 + i)], a.pts[3 * (a.q0 + i) + 1], a.pts[3 * (a.q0 + i) + 2], px, py, pz);
  const unsigned long long per = (a.nm + a.splits - 1) / a.splits;
  const unsigned long long j0 = blockIdx.y * per, j1 = j0 + per < a.nm ? j0 + per : a.nm;
  double best = INFINITY;
  long long bi = -1;
  for (unsigned long long base = j0; base < j1; base += kLvT) {
    __syncthreads();
    const unsigned long long j = base + threadIdx.x;
    if (j < j1) {
      const double* m = a.pts + 3 * (a.m0 + j);
      sx[threadIdx.x] = m[0]; sy[threadIdx.x] = m[1]; sz[threadIdx.x] = m[2];
    }
    __syncthreads();
    const int cnt = (int)(j1 - base < kLvT ? j1 - base : kLvT);
    if (have)
      for (int k = 0; k < cnt; ++k) {
        const double dx = __dsub_rn(px, sx[k]), dy = __dsub_rn(py, sy[k]), dz = __dsub_rn(pz, sz[k]);
        const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
        if (d2 < best) { best = d2; bi = (long long)(base + k); }
      }
  }
  if (have) a.part[blockIdx.y * a.nq + i] = tloam_lv_best{best, bi};
}

// one thread per query row: the slices merged, the pass's match recorded, and the row's contribution to H = sum J^T J,
// g = sum J^T e (inliers: d2 <= r * r), the inlier count, sum d2 over the inliers and over every row, reduced per block
// in a fixed order into a.sums.  pass: the slot of match_index / match_d2 (the final pass uses state->iter).
__global__ void __launch_bounds__(kLvT) k_lv_reduce(tloam_lv_args a, int pass, int final_pass) {
  const tloam_lv_state* s = a.state;
  if (!final_pass && s->done) return;
  const unsigned long long i = blockIdx.x * (unsigned long long)kLvT + threadIdx.x;
  double v[TLOAM_LV_SUMS];
#pragma unroll
  for (int k = 0; k < TLOAM_LV_SUMS; ++k) v[k] = 0.0;
  if (i < a.nq) {
    tloam_lv_best b{INFINITY, -1};
    for (unsigned y = 0; y < a.splits; ++y) {
      const tloam_lv_best c = a.part[y * a.nq + i];
      if (lv_better(c.d2, c.index, b)) b = c;
    }
    const size_t slot = (size_t)(final_pass ? s->iter : pass) * a.nq + i;
    a.match_index[slot] = (int)b.index;
    a.match_d2[slot] = b.d2;
    const double r = final_pass ? a.corr_dist_fine : s->r;
    v[29] = b.d2;
    if (b.index >= 0 && b.d2 <= __dmul_rn(r, r)) {
      double p[3];
      lv_apply(s, a.pts[3 * (a.q0 + i)], a.pts[3 * (a.q0 + i) + 1], a.pts[3 * (a.q0 + i) + 2], p[0], p[1], p[2]);
      const double* m = a.pts + 3 * (a.m0 + (unsigned long long)b.index);
      const double e[3] = {__dsub_rn(p[0], m[0]), __dsub_rn(p[1], m[1]), __dsub_rn(p[2], m[2])};
      // J = [I, -[p]x]
      const double J[3][6] = {{1.0, 0.0, 0.0, 0.0, p[2], -p[1]}, {0.0, 1.0, 0.0, -p[2], 0.0, p[0]}, {0.0, 0.0, 1.0, p[1], -p[0], 0.0}};
#pragma unroll
      for (int u = 0; u < 6; ++u) {
#pragma unroll
        for (int w = 0; w < 6; ++w)
          if (w >= u) v[tri(u, w)] = J[0][u] * J[0][w] + J[1][u] * J[1][w] + J[2][u] * J[2][w];
        v[21 + u] = J[0][u] * e[0] + J[1][u] * e[1] + J[2][u] * e[2];
      }
      v[27] = 1.0;
      v[28] = b.d2;
    }
  }
  __shared__ double ws[kLvT / 32][TLOAM_LV_SUMS];
#pragma unroll
  for (int k = 0; k < TLOAM_LV_SUMS; ++k) {
    double x = v[k];
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5][k] = x;
  }
  __syncthreads();
  if (threadIdx.x < TLOAM_LV_SUMS) {
    double x = 0.0;
    for (unsigned w = 0; w < kLvT / 32; ++w) x += ws[w][threadIdx.x];
    a.sums[blockIdx.x * (size_t)TLOAM_LV_SUMS + threadIdx.x] = x;
  }
}

// the block partials summed in block order (thread k: entry k)
__device__ void lv_total(const tloam_lv_args& a, double* tot) {
  const unsigned nb = (unsigned)((a.nq + kLvT - 1) / kLvT);
  if (threadIdx.x < TLOAM_LV_SUMS) {
    double x = 0.0;
    for (unsigned b = 0; b < nb; ++b) x += a.sums[b * (size_t)TLOAM_LV_SUMS + threadIdx.x];
    tot[threadIdx.x] = x;
  }
  __syncwarp();
}

// one warp: delta = -H^-1 g by LDL^T, T <- exp(delta) . T, then the radius schedule and the termination
__global__ void k_lv_step(tloam_lv_args a) {
  tloam_lv_state* s = a.state;
  if (s->done) return;
  __shared__ double tot[TLOAM_LV_SUMS];
  lv_total(a, tot);
  if (threadIdx.x != 0) return;
  if (tot[27] < 6.0) { s->term = kLvFewInliers; s->done = 1; return; }
  double A[21], b[6], y[6];
  for (int k = 0; k < 21; ++k) A[k] = tot[k];
  for (int k = 0; k < 6; ++k) b[k] = tot[21 + k];
  if (!ldlt_solve6_packed(A, b, y)) { s->term = kLvSingular; s->done = 1; return; }
  double d[6];
  for (int k = 0; k < 6; ++k) d[k] = -y[k];
  const Pose7 e = se3_exp(d);
  double Re[9];
  quat_to_rot(e, Re);
  const double te[3] = {e.tx, e.ty, e.tz};
  double R[9], t[3];
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c)
      R[3 * r + c] = __dadd_rn(__dadd_rn(__dmul_rn(Re[3 * r], s->R[c]), __dmul_rn(Re[3 * r + 1], s->R[3 + c])),
                               __dmul_rn(Re[3 * r + 2], s->R[6 + c]));
    t[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(Re[3 * r], s->t[0]), __dmul_rn(Re[3 * r + 1], s->t[1])),
                               __dmul_rn(Re[3 * r + 2], s->t[2])), te[r]);
  }
  for (int k = 0; k < 9; ++k) s->R[k] = R[k];
  for (int k = 0; k < 3; ++k) s->t[k] = t[k];
  s->iter += 1;
  const double nu = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), nw = sqrt(d[3] * d[3] + d[4] * d[4] + d[5] * d[5]);
  if (nu < a.eps_translation && nw < a.eps_rotation) {
    if (s->r == a.corr_dist_fine) { s->term = kLvConverged; s->done = 1; return; }
    s->r = fmax(s->r * 0.5, a.corr_dist_fine);
  }
  if (s->iter >= a.max_iterations) { s->term = kLvIterationLimit; s->done = 1; }
}

// one warp: the final pass's inliers, rmse over them, fitness = mean d2 over every query row
__global__ void k_lv_final(tloam_lv_args a) {
  tloam_lv_state* s = a.state;
  __shared__ double tot[TLOAM_LV_SUMS];
  lv_total(a, tot);
  if (threadIdx.x != 0) return;
  s->inliers = (unsigned long long)tot[27];
  s->rmse = tot[27] > 0.0 ? sqrt(tot[28] / tot[27]) : 0.0;
  s->fitness = tot[29] / (double)a.nq;
}

__global__ void k_lv_commit(const unsigned* n_vox, const unsigned* refused, unsigned long long* count, unsigned long long* frames,
                            unsigned* flags, unsigned long long* offsets, unsigned long long cap) {
  if (threadIdx.x != 0) return;
  unsigned long long end = *count + (*refused ? 0u : *n_vox);
  if (end > cap) { *flags |= 2u; end = *count; }
  *count = end;
  *frames += 1ull;
  offsets[*frames] = end;
}

}  // namespace tloam

using namespace tloam;

#define TLOAM_LV_API extern "C" __attribute__((visibility("default")))

TLOAM_LV_API int tloam_lv_verify(const tloam_lv_args* a, int* launches) {
  cudaError_t e = cudaSetDevice(a->device);
  *launches = 0;
  if (e != cudaSuccess) return (int)e;
  const unsigned qb = (unsigned)((a->nq + kLvT - 1) / kLvT);
  const dim3 grid(qb, a->splits);
  for (int k = 0; k <= a->max_iterations; ++k) {
    const int fin = k == a->max_iterations;
    k_lv_match<<<grid, kLvT, 0, a->stream>>>(*a, fin);
    k_lv_reduce<<<qb, kLvT, 0, a->stream>>>(*a, k, fin);
    if (fin) k_lv_final<<<1, 32, 0, a->stream>>>(*a);
    else k_lv_step<<<1, 32, 0, a->stream>>>(*a);
    *launches += 3;
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  }
  return (int)cudaSuccess;
}

TLOAM_LV_API int tloam_lv_commit(const unsigned* n_vox, const unsigned* refused, unsigned long long* count, unsigned long long* frames,
                                 unsigned* flags, unsigned long long* offsets, unsigned long long cap, int device, cudaStream_t stream) {
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) return (int)e;
  k_lv_commit<<<1, 32, 0, stream>>>(n_vox, refused, count, frames, flags, offsets, cap);
  return (int)cudaGetLastError();
}
