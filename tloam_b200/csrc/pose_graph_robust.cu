// pose_graph_robust.cu -- libtloam_b200_pgr.so: graduated non-convexity with a truncated-least-squares cost over the loop
// edges of the pose graph (hand-written CUDA for sm_90a).  The full definition is in include/tloam_b200.h ("Robust pose
// graph"); tests/pose_graph_robust_oracle.py restates it in numpy.
//
// Between two weighted Gauss-Newton stages (libtloam_b200_pg.so) the host launches k_pgr_residual, the unweighted
// rho_l = r_l^T Omega_loop r_l of every loop edge at the accepted poses, and k_pgr_weights, T-LOAM's updateWeight over them
// (ref: src/models/registration/registration.cpp:858-876, mu_0 at :1027-1033, the thresholds at :1049-1050).  The
// residual is recomputed rather than read from the edge buffer, which after a reverted step holds the candidate poses'.
// No atomics: the reductions run in a fixed order, so a run is bit-deterministic.
//
// A separate library so that the kernels of libtloam_b200.so keep their SASS and libtloam_b200_pg.so its eight kernels.
#include <cuda_runtime.h>
#include <math.h>

#include "pose_graph.cuh"
#include "pose_graph_robust.h"
#include "se3.cuh"

namespace tloam {

constexpr unsigned kPgrT = 256;
constexpr int kPgSingular = 3;        // tloam_pg_state::term of a stage that met a singular solve: the weights stay

__device__ __forceinline__ bool pgr_singular(const tloam_pgr_args& a) { return a.pg_state->done && a.pg_state->term == kPgSingular; }

// one thread per loop edge: rho = r^T Omega_loop r, r = log(Z^-1 T_i^-1 T_j) at T[cur], in k_pg_linearize's operation order.
// Both kernels do nothing after a singular stage, which ends the run
__global__ void __launch_bounds__(kPgrT) k_pgr_residual(tloam_pgr_args a) {
  const unsigned long long l = blockIdx.x * (unsigned long long)kPgrT + threadIdx.x;
  if (l >= a.L || pgr_singular(a)) return;
  const double* T = a.T + 16ull * a.N * (unsigned)a.pg_state->cur;
  const long long i = a.loop_ij[2 * l], j = a.loop_ij[2 * l + 1];
  double Z[16];
  for (int k = 0; k < 16; ++k) Z[k] = a.loop_Z[16 * l + k];
  double X[16], E[16];
  pg_inv_mul(T + 16 * i, T + 16 * j, X);
  pg_inv_mul(Z, X, E);
  Pose7 p;
  pose_from_matrix(E, p);
  double r[6];
  se3_log(p, r);
  double c = 0.0;
  for (int k = 0; k < 6; ++k) c += a.w_loop[k] * r[k] * r[k];
  a.rho[l] = c;
}

// one block.  first: max rho (a fixed tree); max <= c2 leaves every weight at 1 and sets all_inliers, else
// mu = c2 / (2 max - c2) (<= 0: 1e-10).  Otherwise mu = gnc_factor mu.  Then per edge: rho == 0 -> 1, rho >= th1 -> 0,
// rho <= th2 -> 1, else sqrt(c2 mu (mu + 1) / rho) - mu, with th1 = (mu + 1) / mu c2, th2 = mu / (mu + 1) c2; and the
// counts of weights exactly 1 and exactly 0
__global__ void __launch_bounds__(kPgrT) k_pgr_weights(tloam_pgr_args a, int first) {
  if (pgr_singular(a)) return;
  tloam_pgr_state* g = a.state;
  __shared__ double sm[kPgrT];
  __shared__ int si[kPgrT], sr[kPgrT];
  __shared__ double s_mu;
  __shared__ int s_all;
  const unsigned t = threadIdx.x;
  const double c2 = a.chi2_threshold;
  if (first) {
    double m = 0.0;
    for (unsigned long long l = t; l < a.L; l += kPgrT) m = fmax(m, a.rho[l]);
    sm[t] = m;
    __syncthreads();
    for (unsigned o = kPgrT / 2; o > 0; o >>= 1) {
      if (t < o) sm[t] = fmax(sm[t], sm[t + o]);
      __syncthreads();
    }
    if (t == 0) {
      const double mx = sm[0];
      double mu = c2 / (2.0 * mx - c2);
      if (mu <= 0.0) mu = 1e-10;
      g->max_rho = mx;
      s_all = mx <= c2;
      s_mu = s_all ? 0.0 : mu;
    }
  } else if (t == 0) {
    s_all = 0;
    s_mu = a.gnc_factor * g->mu;
  }
  __syncthreads();
  if (s_all) {
    if (t == 0) { g->all_inliers = 1; g->mu = 0.0; g->binary = 1; g->inliers = (int)a.L; g->rejected = 0; }
    return;
  }
  const double mu = s_mu, th1 = (mu + 1.0) / mu * c2, th2 = mu / (mu + 1.0) * c2;
  int ni = 0, nr = 0;
  for (unsigned long long l = t; l < a.L; l += kPgrT) {
    const double rho = a.rho[l];
    double w;
    if (rho == 0.0) w = 1.0;
    else if (rho >= th1) w = 0.0;
    else if (rho <= th2) w = 1.0;
    else w = sqrt(c2 * mu * (mu + 1.0) / rho) - mu;
    a.w[l] = w;
    ni += w == 1.0;
    nr += w == 0.0;
  }
  si[t] = ni; sr[t] = nr;
  __syncthreads();
  for (unsigned o = kPgrT / 2; o > 0; o >>= 1) {
    if (t < o) { si[t] += si[t + o]; sr[t] += sr[t + o]; }
    __syncthreads();
  }
  if (t == 0) {
    g->all_inliers = 0;
    g->mu = mu;
    g->inliers = si[0]; g->rejected = sr[0];
    g->binary = (unsigned long long)(si[0] + sr[0]) == a.L;
  }
}

}  // namespace tloam

using namespace tloam;

extern "C" __attribute__((visibility("default"))) int tloam_pgr_update(const tloam_pgr_args* a, int first, int* launches) {
  cudaError_t e = cudaSetDevice(a->device);
  *launches = 0;
  if (e != cudaSuccess) return (int)e;
  const unsigned gl = (unsigned)((a->L + kPgrT - 1) / kPgrT);
  k_pgr_residual<<<gl, kPgrT, 0, a->stream>>>(*a);
  k_pgr_weights<<<1, kPgrT, 0, a->stream>>>(*a, first);
  *launches = 2;
  return (int)cudaGetLastError();
}
