// registration.cuh -- device side of the TLS scan-to-map registration (sm_90a).
//
// Reference path: tloam::LocalRegistration::scanMatching, ref: src/models/registration/registration.cpp:879-1133
// and everything it calls (factor builders :427-635, :714-778; cost functors :19-117; fitBestPlane :303-368;
// updateWeight :858-876; PoseSE3Parameterization :162-179) plus the Ceres 2.0 trust-region loop configured at
// :1036-1047 (DOGLEG / SUBSPACE_DOGLEG, DENSE_QR, CauchyLoss(1.0), max_num_iterations 4).
//
// Execution model (one frame = a fixed sequence of small kernels on one stream, zero host round trips):
//   k_begin_frame                      log(predict), Q1 re-init, GNC/solver state reset
//   for outer in 0..max_iterations-1:
//     k_correspond                     lazy GNC weight update + T*p + voxel-hash kNN + line/plane fit
//     k_eval<first>                    caps (prefix over index order) + residual/Jacobian/Cauchy + 6x6
//                                      normal-equation reduction (warp butterfly -> block -> cluster of 8 through
//                                      distributed shared memory); the LAST cluster leader to finish sums the
//                                      per-cluster partials in a fixed order and advances the trust-region
//                                      state machine (solver.cuh), producing the next candidate pose
//     k_eval x ceres_max_num_iterations  same kernel at the candidate pose (accept / reject / converge)
// Every kernel exits immediately when the state says its work is not needed (solve terminated early,
// frame converged), so the launch sequence is static and graph-capturable.
#pragma once
#include <stddef.h>
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>
#include <stdint.h>

#include "../../include/tloam_b200.h"
#include "map_grid.cuh"
#include "se3.cuh"
#include "ldlt6.cuh"

namespace tloam {

constexpr int kBlk = 128;     // threads per block for all per-feature kernels
constexpr int kNRed = 36;     // 21 (H upper) + 6 (g) + 1 (cost) + 4 (slot sum per cloud) + 4 (factors per cloud)
constexpr int kEvalGridCap = 592;   // caps the rows of the final partial sum; a constant (not the SM count) so that the
                                    // reduction tree, and with it the result, is the same on every device
#ifndef TLOAM_EVAL_CLUSTER
#define TLOAM_EVAL_CLUSTER 8
#endif
constexpr int kEvalCluster = TLOAM_EVAL_CLUSTER;     // k_eval runs in clusters of 8 blocks (portable maximum)
constexpr int kEdge = 0, kSphere = 1, kPlanar = 2, kGround = 3;

// flags per feature written by k_correspond
constexpr unsigned char kFlagCand = 1;     // passes every test of the factor builder (subject to the cap)
constexpr unsigned char kFlagCounted = 2;  // advances the builder's counter (edge_num / sphere_sum / ...)

enum Phase : int { kPhaseIter0 = 0, kPhaseCand = 1 };

__device__ __forceinline__ unsigned long long gtime_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

struct FrameState {
  // ---- pose ----
  double x[6];        // accepted tangent = the reference's `parameters` (translation, rotation)
  Pose7 xq;           // exp(x)
  double cand[6];
  Pose7 candq;
  Pose7 evalq;        // pose the next k_eval evaluates at
  // ---- trust-region state (Ceres TrustRegionMinimizer + DoglegStrategy) ----
  int phase, iter, num_invalid, reuse;
  int sub_1d, used_gn, last_cand_valid, outer;
  int sub_valid, model_ok, pad0, pad1;
  double radius, mu_lm, x_cost, x_norm, model_cost_change, step_norm, gn_norm;
  double scale[6], H[21], g[6];
  double d2[6], y[6];                        // Gauss-Newton model (see solver.cuh: GnModel)
  double D[6], sgrad[6], gn[6], sub_basis[12], sub_g[2], sub_B[4];   // filled lazily (subspace dogleg only)
  double last_cand[6], last_cand_cost;
  Pose7 last_candq;
  // ---- GNC state ----
  double mu, mu_used, th1, th2, c2, planar_prev;
  double slot_sum[4];
  // ---- outputs ----
  double result[16];
  int frame_done, status;   // directly after `result`: the host fetches the three with ONE copy
  double fitness, rmse;     // getFitnessScore of this frame's scan (k_fitness_reduce), fetched with the same copy
  unsigned map_bricks[4];   // occupied bricks per cloud of the map this frame registered against (k_begin_frame), idem
  double curr_pose[16], last_pose[16];
};
static_assert(offsetof(FrameState, frame_done) == offsetof(FrameState, result) + 16 * sizeof(double), "result + flags must be contiguous");
static_assert(sizeof(FrameState) % 8 == 0, "FrameState is copied in 8-byte words");


struct DeviceCtx {
  GridDesc grid[4];
  const double* origin;         // -> MapHeader::origin inside the map blob (device memory)
  const unsigned long long* map_flags;   // -> MapHeader::build_flags
  const unsigned* tgt_cnt[4];   // device-side point counts of the map clouds (sync-free submap chain), or nullptr
  const unsigned* map_bricks;   // -> MapHeader::nbricks
  double r2[4];                 // squared search radius per cloud
  int n[4];                     // features per cloud
  int pad_off[4];               // first padded feature index of each cloud (multiple of kBlk)
  int blk_off[5];               // block ranges per cloud
  int maxnum[4];
  int factor_num, max_iterations, ceres_max_it;
  int dense_mask;               // bit c: cloud c is searched by k_correspond_dense (dense map), not by k_correspond
  double edge_dir_thres, cost_threshold, gnc_factor, noise_bound, fitness_thres;
  double reinit_dir[3];
  double initial_radius;        // Ceres options.initial_trust_region_radius (default 1e4; a test knob otherwise)
  // per-feature SoA (padded)
  const double *px, *py, *pz;
  double *w, *slot;
  double* prim[6];
  unsigned char *flags, *active;
  int* blk_count;               // [2][blocks] (double-buffered by outer&1): `counted` features per 128-feature block
  double* partial;              // [blocks][kNRed]
  unsigned* counter;            // last-block ticket
  int blk_cap;                  // stride between the two blk_count buffers
  unsigned long long* dbg;      // in-kernel timers (profiling mode only, else nullptr)
  FrameState* st;
  tloam_b200_stats* stats;      // device copy of the trace
};

__device__ __forceinline__ bool cloud_enabled(const DeviceCtx& c, int cloud) {
  // factor_num 4: planar, ground, edge, sphere; 3: planar, ground, edge; 2: planar, ground  (ref: :979-1016)
  if (cloud == kPlanar || cloud == kGround) return c.factor_num >= 2 && c.factor_num <= 4;
  if (cloud == kEdge) return c.factor_num >= 3 && c.factor_num <= 4;
  return c.factor_num == 4;
}

__device__ __forceinline__ int cloud_of_block(const DeviceCtx& c, int b) {
  return (b >= c.blk_off[3]) ? 3 : (b >= c.blk_off[2]) ? 2 : (b >= c.blk_off[1]) ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------
// Primitive fits
// ------------------------------------------------------------------------------------------------
// fitBestPlane, ref: registration.cpp:303-368 (closed form, sub-determinant weighted normal).
__device__ __forceinline__ void fit_best_plane(const double (*q)[3], int n, double nd[4]) {
  const double inv = 1.0 / (double)n;
  double cx = 0, cy = 0, cz = 0;
  for (int i = 0; i < n; ++i) { cx += q[i][0]; cy += q[i][1]; cz += q[i][2]; }
  cx /= (double)n; cy /= (double)n; cz /= (double)n;
  double xx = 0, xy = 0, xz = 0, yy = 0, yz = 0, zz = 0;
  for (int i = 0; i < n; ++i) {
    const double dx = q[i][0] - cx, dy = q[i][1] - cy, dz = q[i][2] - cz;
    xx += dx * dx; xy += dx * dy; xz += dx * dz; yy += dy * dy; yz += dy * dz; zz += dz * dz;
  }
  (void)inv;
  const double tn = (double)n;
  xx /= tn; xy /= tn; xz /= tn; yy /= tn; yz /= tn; zz /= tn;
  double wx = 0, wy = 0, wz = 0;
  {
    const double det = yy * zz - yz * yz;
    const double ax = det, ay = xz * yz - xy * zz, az = xy * yz - xz * yy;
    double wgt = det * det;
    if (wx * ax + wy * ay + wz * az < 0.0) wgt = -wgt;
    wx += ax * wgt; wy += ay * wgt; wz += az * wgt;
  }
  {
    const double det = xx * zz - xz * xz;
    const double ax = xz * yz - xy * zz, ay = det, az = xy * xz - yz * xx;
    double wgt = det * det;
    if (wx * ax + wy * ay + wz * az < 0.0) wgt = -wgt;
    wx += ax * wgt; wy += ay * wgt; wz += az * wgt;
  }
  {
    const double det = xx * yy - xy * xy;
    const double ax = xy * yz - xz * yy, ay = xy * xz - yz * xx, az = det;
    double wgt = det * det;
    if (wx * ax + wy * ay + wz * az < 0.0) wgt = -wgt;
    wx += ax * wgt; wy += ay * wgt; wz += az * wgt;
  }
  const double nn = sqrt(wx * wx + wy * wy + wz * wz);
  if (nn == 0.0) { nd[0] = nd[1] = nd[2] = nd[3] = 0.0; return; }
  wx /= nn; wy /= nn; wz /= nn;
  nd[0] = wx; nd[1] = wy; nd[2] = wz; nd[3] = -(wx * cx + wy * cy + wz * cz);
}

// Symmetric 3x3 eigen-decomposition by cyclic Jacobi rotations (FP64, to round-off). Stands in for
// Eigen::SelfAdjointEigenSolver<Matrix3d>::compute (ref: registration.cpp:476-479). Returns the largest
// eigenvalue's eigenvector in v and the three eigenvalues (ascending) in ev.
__device__ __forceinline__ void sym_eig3_max(double a00, double a01, double a02, double a11, double a12, double a22,
                                             double ev[3], double v[3]) {
  double A[3][3] = {{a00, a01, a02}, {a01, a11, a12}, {a02, a12, a22}};
  double V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int sweep = 0; sweep < 32; ++sweep) {
    const double off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2];
    const double dg = A[0][0] * A[0][0] + A[1][1] * A[1][1] + A[2][2] * A[2][2];
    if (off <= 1e-32 * dg || off == 0.0) break;
#pragma unroll
    for (int pq = 0; pq < 3; ++pq) {
      const int p = (pq == 2) ? 1 : 0;
      const int q = (pq == 0) ? 1 : 2;
      const double apq = A[p][q];
      if (apq == 0.0) continue;
      const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
      const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
      const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double akp = A[k][p], akq = A[k][q];
        A[k][p] = c * akp - s * akq;
        A[k][q] = s * akp + c * akq;
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double apk = A[p][k], aqk = A[q][k];
        A[p][k] = c * apk - s * aqk;
        A[q][k] = s * apk + c * aqk;
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double vkp = V[k][p], vkq = V[k][q];
        V[k][p] = c * vkp - s * vkq;
        V[k][q] = s * vkp + c * vkq;
      }
    }
  }
  // sort the three diagonal entries ascending, track the column of the maximum
  double e0 = A[0][0], e1 = A[1][1], e2 = A[2][2];
  int imax = 0;
  double emax = e0;
  if (e1 > emax) { emax = e1; imax = 1; }
  if (e2 > emax) { emax = e2; imax = 2; }
  const double lo = fmin(e0, fmin(e1, e2));
  const double mid = e0 + e1 + e2 - lo - emax;
  ev[0] = lo; ev[1] = mid; ev[2] = emax;
  v[0] = V[0][imax]; v[1] = V[1][imax]; v[2] = V[2][imax];
}

// ------------------------------------------------------------------------------------------------
// Cost functors (rows of J are row-major 1x6: translation 3, rotation 3). c = T*p computed by the caller.
// ------------------------------------------------------------------------------------------------
// PointToPlaneErr::Evaluate, ref: registration.cpp:96-117. Residual NOT weighted, Jacobian weighted.
__device__ __forceinline__ void functor_plane(const double c[3], const double n[3], double d, double w, double& r,
                                              double J[6]) {
  r = n[0] * c[0] + n[1] * c[1] + n[2] * c[2] + d;
  J[0] = n[0] * w; J[1] = n[1] * w; J[2] = n[2] * w;
  // n^T * (-hat(c) * w) = w * (c x n)^T
  J[3] = (c[1] * n[2] - c[2] * n[1]) * w;
  J[4] = (c[2] * n[0] - c[0] * n[2]) * w;
  J[5] = (c[0] * n[1] - c[1] * n[0]) * w;
}

// PointToPointErr::Evaluate, ref: registration.cpp:19-47.  r = w (q - c), J = w [-I | hat(c)].
__device__ __forceinline__ void functor_point(const double c[3], const double q[3], double w, double r[3], double J[18]) {
  r[0] = (q[0] - c[0]) * w; r[1] = (q[1] - c[1]) * w; r[2] = (q[2] - c[2]) * w;
  J[0] = -w;  J[1] = 0.0; J[2] = 0.0; J[3] = 0.0;        J[4] = -c[2] * w;  J[5] = c[1] * w;
  J[6] = 0.0; J[7] = -w;  J[8] = 0.0; J[9] = c[2] * w;   J[10] = 0.0;       J[11] = -c[0] * w;
  J[12] = 0.0; J[13] = 0.0; J[14] = -w; J[15] = -c[1] * w; J[16] = c[0] * w; J[17] = 0.0;
}

// PointToLineErr::Evaluate, ref: registration.cpp:55-88.
// r = w (c-a)x(c-b)/|a-b| ,  J = hat(b-a) * w [I | -hat(c)] / |a-b|.
__device__ __forceinline__ void functor_line(const double c[3], const double a[3], const double b[3], double w,
                                             double r[3], double J[18]) {
  const double ux = c[0] - a[0], uy = c[1] - a[1], uz = c[2] - a[2];
  const double vx = c[0] - b[0], vy = c[1] - b[1], vz = c[2] - b[2];
  const double dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
  // NOTE the reference divides every entry by |a-b| (x / den * w); here one reciprocal is shared, which differs
  // from the reference's rounding by <= 1 ulp per entry.
  const double inv = 1.0 / sqrt(dx * dx + dy * dy + dz * dz);
  r[0] = (uy * vz - uz * vy) * inv * w;
  r[1] = (uz * vx - ux * vz) * inv * w;
  r[2] = (ux * vy - uy * vx) * inv * w;
  // S = hat(b - a) ; M = [I*w | -hat(c)*w] ; J = S*M/den
  const double ex = -dx, ey = -dy, ez = -dz;  // b - a
  const double S[9] = {0.0, -ez, ey, ez, 0.0, -ex, -ey, ex, 0.0};
  const double M[18] = {w,   0.0, 0.0, 0.0,       c[2] * w,  -c[1] * w,
                        0.0, w,   0.0, -c[2] * w, 0.0,       c[0] * w,
                        0.0, 0.0, w,   c[1] * w,  -c[0] * w, 0.0};
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 6; ++j)
      J[i * 6 + j] = (S[i * 3 + 0] * M[0 * 6 + j] + S[i * 3 + 1] * M[1 * 6 + j] + S[i * 3 + 2] * M[2 * 6 + j]) * inv;
}

}  // namespace tloam
