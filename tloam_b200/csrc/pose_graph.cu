// pose_graph.cu -- libtloam_b200_pg.so: Gauss-Newton over a pose graph on the device (hand-written CUDA for sm_90a).  The
// nodes are the loop frames' odometry poses, the edges the odometry chain and the accepted loop verifications.  The full
// definition is in include/tloam_b200.h ("Pose graph"); tests/pose_graph_oracle.py restates it in numpy.
//
// The normal matrix is H = M + B^T Omega_L B: M the block-tridiagonal chain (node 0 fixed), B the L loop rows.  It is
// solved exactly by Woodbury: a block LDL^T of M along the chain, Y = M^-1 [B^T | b] (one thread per column, sequential
// along the chain), the capacitance S = Omega_L^-1 + B Y by a dense Cholesky (one cooperative grid), then
// delta = u - Y S^-1 B u.  No atomics: every sum runs in a fixed order, so a run is bit-deterministic.
//
// A separate library so that the kernels of libtloam_b200.so keep their SASS.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <math.h>

#include "ldlt6.cuh"
#include "pose_graph.cuh"
#include "pose_graph.h"
#include "se3.cuh"

namespace cg = cooperative_groups;

namespace tloam {

enum { kPgConverged = 0, kPgIterationLimit = 1, kPgCostIncreased = 2, kPgSingular = 3 };
constexpr unsigned kPgT = 256;

__device__ __forceinline__ const double* pg_T(const tloam_pg_args& a, int buf) { return a.T + 16ull * a.N * (unsigned)buf; }

// one thread per edge (odometry edges first): r = log(Z^-1 T_i^-1 T_j), A = Ad(T_j^-1), r^T Omega r.  candidate: read the
// round's candidate poses T[cur ^ 1], else T[cur].  With loop_w, loop edge l stores sqrt(w_l) A and sqrt(w_l) r, so every
// later kernel solves the weighted system and the cost term is w_l r^T Omega r
__global__ void __launch_bounds__(kPgT) k_pg_linearize(tloam_pg_args a, int candidate) {
  const tloam_pg_state* s = a.state;
  if (candidate && s->done) return;
  const unsigned long long e = blockIdx.x * (unsigned long long)kPgT + threadIdx.x;
  const unsigned long long no = a.N - 1;
  if (e >= no + a.L) return;
  const double* T = pg_T(a, candidate ? s->cur ^ 1 : s->cur);
  long long i, j;
  double Z[16];
  const double* w;
  if (e < no) {
    i = (long long)e; j = i + 1;
    pg_inv_mul(a.O + 16 * i, a.O + 16 * j, Z);
    w = a.w_odom;
  } else {
    i = a.loop_ij[2 * (e - no)]; j = a.loop_ij[2 * (e - no) + 1];
    for (int k = 0; k < 16; ++k) Z[k] = a.loop_Z[16 * (e - no) + k];
    w = a.w_loop;
  }
  double X[16], E[16];
  pg_inv_mul(T + 16 * i, T + 16 * j, X);
  pg_inv_mul(Z, X, E);
  Pose7 p;
  pose_from_matrix(E, p);
  double r[6];
  se3_log(p, r);
  double* out = a.edge + e * TLOAM_PG_EDGE;
  // Ad(T_j^-1) = [[R, [t]x R], [0, R]] with R = R_j^T, t = -R_j^T t_j
  const double* Tj = T + 16 * j;
  double R[9], t[3];
  for (int u = 0; u < 3; ++u)
    for (int v = 0; v < 3; ++v) R[3 * u + v] = PGM(Tj, v, u);
  for (int u = 0; u < 3; ++u) t[u] = -(R[3 * u] * PGM(Tj, 0, 3) + R[3 * u + 1] * PGM(Tj, 1, 3) + R[3 * u + 2] * PGM(Tj, 2, 3));
  const double tx[9] = {0.0, -t[2], t[1], t[2], 0.0, -t[0], -t[1], t[0], 0.0};
  for (int u = 0; u < 3; ++u)
    for (int v = 0; v < 3; ++v) {
      out[6 * u + v] = R[3 * u + v];
      out[6 * u + v + 3] = tx[3 * u] * R[v] + tx[3 * u + 1] * R[3 + v] + tx[3 * u + 2] * R[6 + v];
      out[6 * (u + 3) + v] = 0.0;
      out[6 * (u + 3) + v + 3] = R[3 * u + v];
    }
  if (a.loop_w && e >= no) {
    const double sw = sqrt(a.loop_w[e - no]);
    for (int k = 0; k < 36; ++k) out[k] *= sw;
    for (int k = 0; k < 6; ++k) r[k] *= sw;
  }
  double c = 0.0;
  for (int k = 0; k < 6; ++k) {
    out[36 + k] = r[k];
    c += w[k] * r[k] * r[k];
  }
  out[42] = c;
  out[43] = 0.0;
}

// P_k = A^T Omega_odom A of odometry edge (k - 1, k), entry (u, v)
__device__ __forceinline__ double pg_podom(const tloam_pg_args& a, unsigned long long k, int u, int v) {
  const double* A = a.edge + (k - 1) * TLOAM_PG_EDGE;
  double x = 0.0;
  for (int m = 0; m < 6; ++m) x += A[6 * m + u] * a.w_odom[m] * A[6 * m + v];
  return x;
}

// one block of 64: the block LDL^T of M along the chain.  D_k = P_k + P_{k+1}, S_1 = D_1, S_k = D_k - P_k S_{k-1}^-1 P_k;
// per node it stores W_k = P_k S_{k-1}^-1, S_k^-1 (six LDL^T solves) and P_{k+1}
__global__ void __launch_bounds__(64) k_pg_chain_factor(tloam_pg_args a) {
  tloam_pg_state* s = a.state;
  if (s->done) return;
  __shared__ double P0[36], P1[36], X[36], Sp[21], Si[36];
  __shared__ int bad;
  const int t = threadIdx.x, u = t / 6, v = t % 6;
  const unsigned long long N = a.N;
  if (t < 36) { P0[t] = pg_podom(a, 1, u, v); X[t] = 0.0; }
  if (t == 0) bad = 0;
  __syncthreads();
  for (unsigned long long k = 1; k < N; ++k) {
    if (t < 36) P1[t] = k + 1 < N ? pg_podom(a, k + 1, u, v) : 0.0;
    __syncthreads();
    if (t < 36 && u <= v) {
      double x = 0.0;
      for (int m = 0; m < 6; ++m) x += P0[6 * u + m] * X[6 * m + v];
      Sp[tri(u, v)] = (P0[t] + P1[t]) - x;
    }
    __syncthreads();
    if (t < 6) {
      double A[21], e[6], y[6];
      for (int m = 0; m < 21; ++m) A[m] = Sp[m];
      for (int m = 0; m < 6; ++m) e[m] = m == t ? 1.0 : 0.0;
      if (!ldlt_solve6_packed(A, e, y)) bad = 1;
      for (int m = 0; m < 6; ++m) Si[6 * m + t] = y[m];
    }
    __syncthreads();
    if (bad) {
      if (t == 0) { s->term = kPgSingular; s->done = 1; }
      return;
    }
    double x = 0.0;
    double* ck = a.chain + k * TLOAM_PG_CHAIN;
    if (t < 36) {
      for (int m = 0; m < 6; ++m) x += Si[6 * u + m] * P1[6 * m + v];        // X_{k+1} = S_k^-1 P_{k+1}
      ck[36 + t] = Si[t];
      ck[72 + t] = P1[t];
      if (k + 1 < N) a.chain[(k + 1) * TLOAM_PG_CHAIN + 6 * v + u] = x;     // W_{k+1} = X_{k+1}^T
    }
    __syncthreads();
    if (t < 36) { X[t] = x; P0[t] = P1[t]; }
    __syncthreads();
  }
}

// one thread per node k >= 1: b_k = -g_k, g_k = sum over the edges at k of +-A^T Omega r (+ where k is j): odometry edge
// (k - 1, k), odometry edge (k, k + 1), then the loop edges in order
__global__ void __launch_bounds__(kPgT) k_pg_rhs(tloam_pg_args a) {
  if (a.state->done) return;
  const unsigned long long k = blockIdx.x * (unsigned long long)kPgT + threadIdx.x;
  if (k == 0 || k >= a.N) return;
  double g[6] = {0, 0, 0, 0, 0, 0};
  auto add = [&](unsigned long long e, const double* w, double sign) {
    const double* A = a.edge + e * TLOAM_PG_EDGE;
    double wr[6];
    for (int m = 0; m < 6; ++m) wr[m] = w[m] * A[36 + m];
    for (int q = 0; q < 6; ++q) {
      double x = 0.0;
      for (int m = 0; m < 6; ++m) x += A[6 * m + q] * wr[m];
      g[q] += sign * x;
    }
  };
  const unsigned long long no = a.N - 1;
  add(k - 1, a.w_odom, 1.0);
  if (k < no) add(k, a.w_odom, -1.0);
  for (unsigned long long l = 0; l < a.L; ++l) {
    if ((unsigned long long)a.loop_ij[2 * l + 1] == k) add(no + l, a.w_loop, 1.0);
    else if ((unsigned long long)a.loop_ij[2 * l] == k) add(no + l, a.w_loop, -1.0);
  }
  for (int q = 0; q < 6; ++q) a.b[6 * k + q] = -g[q];
}

// one thread per column of [B^T | b]: forward y_k = rhs_k + W_k y_{k-1}, backward x_k = S_k^-1 (y_k + P_{k+1} x_{k+1}).
// Column 6 e + p of B^T holds row p of A_e at node j_e and its negative at node i_e (node 0 has no row)
__global__ void __launch_bounds__(128) k_pg_chain_solve(tloam_pg_args a) {
  if (a.state->done) return;
  const unsigned long long nl = 6 * a.L, ncol = nl + 1;
  const unsigned long long col = blockIdx.x * 128ull + threadIdx.x;
  if (col >= ncol) return;
  const unsigned long long N = a.N, no = N - 1;
  const bool isb = col == nl;
  unsigned long long li = 0, lj = 0;
  const double* Ae = nullptr;
  if (!isb) {
    const unsigned long long e = col / 6;
    li = (unsigned long long)a.loop_ij[2 * e]; lj = (unsigned long long)a.loop_ij[2 * e + 1];
    Ae = a.edge + (no + e) * TLOAM_PG_EDGE + 6 * (col % 6);
  }
  double y[6] = {0, 0, 0, 0, 0, 0};
  for (unsigned long long k = 1; k < N; ++k) {
    double r[6];
    if (isb) {
      for (int q = 0; q < 6; ++q) r[q] = a.b[6 * k + q];
    } else {
      for (int q = 0; q < 6; ++q) r[q] = k == lj ? Ae[q] : (k == li ? -Ae[q] : 0.0);
    }
    const double* W = a.chain + k * TLOAM_PG_CHAIN;
    double ny[6];
    for (int q = 0; q < 6; ++q) {
      double x = r[q];
      if (k > 1)
        for (int m = 0; m < 6; ++m) x += W[6 * q + m] * y[m];
      ny[q] = x;
    }
    for (int q = 0; q < 6; ++q) {
      y[q] = ny[q];
      a.Y[(6 * (k - 1) + q) * ncol + col] = ny[q];
    }
  }
  double x[6] = {0, 0, 0, 0, 0, 0};
  for (unsigned long long k = no; k >= 1; --k) {
    const double* ck = a.chain + k * TLOAM_PG_CHAIN;
    double v[6];
    for (int q = 0; q < 6; ++q) {
      double t = a.Y[(6 * (k - 1) + q) * ncol + col];
      if (k < no)
        for (int m = 0; m < 6; ++m) t += ck[72 + 6 * q + m] * x[m];
      v[q] = t;
    }
    for (int q = 0; q < 6; ++q) {
      double t = 0.0;
      for (int m = 0; m < 6; ++m) t += ck[36 + 6 * q + m] * v[m];
      x[q] = t;
    }
    for (int q = 0; q < 6; ++q) a.Y[(6 * (k - 1) + q) * ncol + col] = x[q];
  }
}

// one thread per entry (row 6 e + p, column c) of [Omega_L^-1 + B Y | B u]: sum_q A_e[p][q] (Y[j_e, q][c] - Y[i_e, q][c]);
// rows stride over grid y, so any number of loop edges fits the grid
__global__ void __launch_bounds__(kPgT) k_pg_capacitance(tloam_pg_args a) {
  if (a.state->done) return;
  const unsigned long long nl = 6 * a.L, ncol = nl + 1, no = a.N - 1;
  const unsigned long long c = blockIdx.x * (unsigned long long)kPgT + threadIdx.x;
  if (c >= ncol) return;
  for (unsigned long long row = blockIdx.y; row < nl; row += gridDim.y) {
    const unsigned long long e = row / 6, p = row % 6;
    const long long li = a.loop_ij[2 * e], lj = a.loop_ij[2 * e + 1];
    const double* A = a.edge + (no + e) * TLOAM_PG_EDGE + 6 * p;
    double x = 0.0;
    for (int q = 0; q < 6; ++q) {
      const double yj = lj > 0 ? a.Y[(6 * (lj - 1) + q) * ncol + c] : 0.0;
      const double yi = li > 0 ? a.Y[(6 * (li - 1) + q) * ncol + c] : 0.0;
      x += A[q] * (yj - yi);
    }
    if (c == row) x += 1.0 / a.w_loop[p];
    a.S[row * ncol + c] = x;
  }
}

// one cooperative grid: right-looking Cholesky of the lower triangle of S's first 6L columns (column k scaled, then the
// trailing lower triangle updated, warps over rows, lanes over columns; L(k, i) is mirrored into the upper triangle so the
// update reads it contiguously), then block 0 solves S z = B u
__global__ void __launch_bounds__(kPgT) k_pg_dense_chol(tloam_pg_args a) {
  cg::grid_group grid = cg::this_grid();
  tloam_pg_state* s = a.state;
  const int done = s->done;
  grid.sync();                                   // every block has read done before anyone may write it
  if (done) return;
  const unsigned long long n = 6 * a.L, ld = n + 1;
  double* S = a.S;
  const unsigned long long gt = blockIdx.x * (unsigned long long)kPgT + threadIdx.x, gn = (unsigned long long)gridDim.x * kPgT;
  const unsigned long long warp = gt / 32, nwarps = gn / 32;
  const unsigned lane = threadIdx.x & 31;
  bool ok = true;
  for (unsigned long long k = 0; k < n; ++k) {
    const double d = S[k * ld + k];
    if (!(d > 0.0) || !isfinite(d)) { ok = false; break; }   // every block reads the same d: all leave together
    const double l = sqrt(d);
    for (unsigned long long i = k + 1 + gt; i < n; i += gn) {
      const double v = S[i * ld + k] / l;
      S[i * ld + k] = v;
      S[k * ld + i] = v;
    }
    grid.sync();
    if (gt == 0) S[k * ld + k] = l;
    for (unsigned long long i = k + 1 + warp; i < n; i += nwarps) {
      const double lik = S[i * ld + k];
      for (unsigned long long j = k + 1 + lane; j <= i; j += 32) S[i * ld + j] -= lik * S[k * ld + j];
    }
    grid.sync();
  }
  if (!ok) {
    if (gt == 0) { s->term = kPgSingular; s->done = 1; }
    return;
  }
  if (blockIdx.x != 0) return;
  double* z = a.z;
  for (unsigned long long i = threadIdx.x; i < n; i += kPgT) z[i] = S[i * ld + n];
  __syncthreads();
  for (unsigned long long k = 0; k < n; ++k) {                  // L w = c
    const double zk = z[k] / S[k * ld + k];
    __syncthreads();
    if (threadIdx.x == 0) z[k] = zk;
    for (unsigned long long i = k + 1 + threadIdx.x; i < n; i += kPgT) z[i] -= S[i * ld + k] * zk;
    __syncthreads();
  }
  for (unsigned long long kk = 0; kk < n; ++kk) {              // L^T z = w
    const unsigned long long k = n - 1 - kk;
    const double zk = z[k] / S[k * ld + k];
    __syncthreads();
    if (threadIdx.x == 0) z[k] = zk;
    for (unsigned long long i = threadIdx.x; i < k; i += kPgT) z[i] -= S[k * ld + i] * zk;
    __syncthreads();
  }
}

// one warp per node: delta = u - Y z over its six rows (lanes over the columns, a fixed butterfly), then the candidate
// T[cur ^ 1]_k = exp(delta) T[cur]_k (node 0 copied) and the node's largest step components
__global__ void __launch_bounds__(kPgT) k_pg_update(tloam_pg_args a) {
  const tloam_pg_state* s = a.state;
  if (s->done) return;
  const unsigned long long k = (blockIdx.x * (unsigned long long)kPgT + threadIdx.x) / 32;
  const unsigned lane = threadIdx.x & 31;
  if (k >= a.N) return;
  const double* Tc = pg_T(a, s->cur) + 16 * k;
  double* Tn = a.T + 16ull * a.N * (unsigned)(s->cur ^ 1) + 16 * k;
  if (k == 0) {
    if (lane < 16) Tn[lane] = Tc[lane];
    if (lane == 0) { a.norms[0] = 0.0; a.norms[1] = 0.0; }
    return;
  }
  const unsigned long long nl = 6 * a.L, ncol = nl + 1;
  double d[6];
  for (int q = 0; q < 6; ++q) {
    const double* row = a.Y + (6 * (k - 1) + q) * ncol;
    double x = 0.0;
    for (unsigned long long c = lane; c < nl; c += 32) x += row[c] * a.z[c];
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    d[q] = row[nl] - x;
  }
  if (lane != 0) return;
  const Pose7 e = se3_exp(d);
  double Re[9];
  quat_to_rot(e, Re);
  const double te[3] = {e.tx, e.ty, e.tz};
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) PGM(Tn, r, c) = Re[3 * r] * PGM(Tc, 0, c) + Re[3 * r + 1] * PGM(Tc, 1, c) + Re[3 * r + 2] * PGM(Tc, 2, c);
    PGM(Tn, r, 3) = Re[3 * r] * PGM(Tc, 0, 3) + Re[3 * r + 1] * PGM(Tc, 1, 3) + Re[3 * r + 2] * PGM(Tc, 2, 3) + te[r];
    PGM(Tn, 3, r) = 0.0;
  }
  PGM(Tn, 3, 3) = 1.0;
  a.norms[2 * k] = fmax(fmax(fabs(d[0]), fabs(d[1])), fabs(d[2]));
  a.norms[2 * k + 1] = fmax(fmax(fabs(d[3]), fabs(d[4])), fabs(d[5]));
}

// one block: the cost sum_e r^T Omega r (thread-strided partials, then a fixed tree) and, after a step, the step's largest
// components and the termination: a step below both eps converges; else a cost that is not <= the current one reverts the
// step and stops; else the step is accepted and the run stops at max_iterations
__global__ void __launch_bounds__(kPgT) k_pg_accept(tloam_pg_args a, int initial) {
  tloam_pg_state* s = a.state;
  if (!initial && s->done) return;
  __shared__ double sc[kPgT], st[kPgT], sr[kPgT];
  const unsigned long long E = a.N - 1 + a.L;
  double c = 0.0, nt = 0.0, nr = 0.0;
  for (unsigned long long e = threadIdx.x; e < E; e += kPgT) c += a.edge[e * TLOAM_PG_EDGE + 42];
  if (!initial)
    for (unsigned long long k = threadIdx.x; k < a.N; k += kPgT) { nt = fmax(nt, a.norms[2 * k]); nr = fmax(nr, a.norms[2 * k + 1]); }
  sc[threadIdx.x] = c; st[threadIdx.x] = nt; sr[threadIdx.x] = nr;
  __syncthreads();
  for (unsigned o = kPgT / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      sc[threadIdx.x] += sc[threadIdx.x + o];
      st[threadIdx.x] = fmax(st[threadIdx.x], st[threadIdx.x + o]);
      sr[threadIdx.x] = fmax(sr[threadIdx.x], sr[threadIdx.x + o]);
    }
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  const double cost = sc[0];
  if (initial) { s->cost = cost; s->initial_cost = cost; return; }
  s->step_t = st[0]; s->step_r = sr[0];
  const bool small = st[0] < a.eps_translation && sr[0] < a.eps_rotation;
  if (!small && !(cost <= s->cost)) { s->term = kPgCostIncreased; s->done = 1; return; }
  s->cur ^= 1;
  s->cost = cost;
  s->iter += 1;
  if (small) { s->term = kPgConverged; s->done = 1; }
  else if (s->iter >= a.max_iterations) { s->term = kPgIterationLimit; s->done = 1; }
}

}  // namespace tloam

using namespace tloam;

#define TLOAM_PG_API extern "C" __attribute__((visibility("default")))

TLOAM_PG_API int tloam_pg_chol_blocks(int device, unsigned* blocks) {
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) return (int)e;
  int per = 0, sms = 0;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, k_pg_dense_chol, kPgT, 0)) != cudaSuccess) return (int)e;
  if ((e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device)) != cudaSuccess) return (int)e;
  *blocks = (unsigned)(sms * (per < 2 ? per : 2));
  return *blocks ? (int)cudaSuccess : (int)cudaErrorCooperativeLaunchTooLarge;
}

TLOAM_PG_API int tloam_pg_optimize(const tloam_pg_args* a, int* launches) {
  cudaError_t e = cudaSetDevice(a->device);
  *launches = 0;
  if (e != cudaSuccess) return (int)e;
  const unsigned long long E = a->N - 1 + a->L, nl = 6 * a->L, ncol = nl + 1;
  const unsigned ge = (unsigned)((E + kPgT - 1) / kPgT), gn = (unsigned)((a->N + kPgT - 1) / kPgT);
  const unsigned gw = (unsigned)((32 * a->N + kPgT - 1) / kPgT), gc = (unsigned)((ncol + kPgT - 1) / kPgT);
  const unsigned gs = (unsigned)((ncol + 127) / 128);
  tloam_pg_args args = *a;
  k_pg_linearize<<<ge, kPgT, 0, a->stream>>>(args, 0);
  k_pg_accept<<<1, kPgT, 0, a->stream>>>(args, 1);
  *launches += 2;
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  void* params[] = {&args};
  for (int it = 0; it < a->max_iterations; ++it) {
    k_pg_chain_factor<<<1, 64, 0, a->stream>>>(args);
    k_pg_rhs<<<gn, kPgT, 0, a->stream>>>(args);
    k_pg_chain_solve<<<gs, 128, 0, a->stream>>>(args);
    k_pg_capacitance<<<dim3(gc, (unsigned)(nl < 65535 ? nl : 65535)), kPgT, 0, a->stream>>>(args);
    if ((e = cudaLaunchCooperativeKernel((const void*)k_pg_dense_chol, dim3(a->chol_blocks), dim3(kPgT), params, 0, a->stream)) !=
        cudaSuccess)
      return (int)e;
    k_pg_update<<<gw, kPgT, 0, a->stream>>>(args);
    k_pg_linearize<<<ge, kPgT, 0, a->stream>>>(args, 1);
    k_pg_accept<<<1, kPgT, 0, a->stream>>>(args, 0);
    *launches += 8;
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  }
  return (int)cudaSuccess;
}
