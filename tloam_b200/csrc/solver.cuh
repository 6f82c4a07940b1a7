// solver.cuh -- on-device trust-region state machine, run by the LAST block of k_eval.
//
// Restates, for ONE 6-parameter block, the control flow of Ceres Solver 2.0
//   TrustRegionMinimizer::Minimize / IterationZero / ComputeTrustRegionStep / HandleSuccessfulStep /
//   HandleInvalidStep / ParameterToleranceReached / FunctionToleranceReached (trust_region_minimizer.cc),
//   DoglegStrategy with SUBSPACE_DOGLEG (dogleg_strategy.cc), TrustRegionStepEvaluator (monotonic),
// with the options the reference sets (ref: registration.cpp:1036-1047) and Ceres defaults otherwise,
// followed by the reference's GNC bookkeeping (ref: registration.cpp:1049-1121).
//
// Everything Ceres derives from the Jacobian is derived here from the 6x6 normal equations
// H = J^T J, g = J^T r (robustified, unscaled) that k_eval reduces: with S = jacobi scaling,
//   J_s^T J_s = S H S,  J_s^T r = S g,  ||J_s col||^2 = (S H S)_jj,
//   model_cost_change = -(g_s . step + step^T H_s step / 2),
//   DENSE_QR on [J_s ; sqrt(mu) D] y = [r ; 0]  ==  (H_s + mu D^2) y = g_s  (solved by Cholesky, FP64).
//
// The work is one long chain of dependent FP64 operations (~15 cycles each), so it is split over the warps of
// the block (measured: 29k cycles single-threaded):
//   phase A, concurrently   warp 1: gradient-tolerance quantity |x - Plus(x,-g)|_inf for the state that would
//                                   be current if this evaluation is accepted
//                           warp 2: Gauss-Newton model (diagonal, scaled gradient, Cholesky solve) from the
//                                   freshly reduced H, g  -- speculative, used iff the step is accepted
//                           warp 3: cand = log(candidate pose) (the candidate was handed to the kernels as a
//                                   pose; its tangent is only needed for tolerance tests and the trace)
//   phase B, thread 0       accept / reject / convergence logic, dogleg step, next candidate pose.
#pragma once
#include "registration.cuh"
#include "ldlt6.cuh"

namespace tloam {

__device__ __forceinline__ double norm6(const double* v) {
  double s = 0.0;
  for (int i = 0; i < 6; ++i) s += v[i] * v[i];
  return sqrt(s);
}

// The same factorisation with ROLLED loops on arrays in shared memory (w: 21 + 4 * 6 doubles of scratch).  Same
// operations in the same order (bit-identical); ~10x fewer static instructions.  Built to test whether the unrolled form
// is bound by instruction fetch (the solver runs once per launch on one SM with a cold instruction cache): it is not --
// measured 11.3k cycles against 5.0k, every operand pays the shared-memory latency.  Kept for A/B only
// (TLOAM_SOLVER_ROLLED_MODEL).
__device__ __noinline__ bool ldlt_solve6_rolled(double* a, const double* b, double* yout, double* w) {
  double* d = w; double* dinv = w + 6; double* z = w + 12;
  bool ok = true;
#pragma unroll 1
  for (int j = 0; j < 6; ++j) {
    double s = a[tri(j, j)];
#pragma unroll 1
    for (int k = 0; k < j; ++k) s -= a[tri(k, j)] * a[tri(k, j)] * d[k];
    d[j] = s;
    ok = ok && (s > 0.0) && isfinite(s);
    const double di = 1.0 / s;
    dinv[j] = di;
#pragma unroll 1
    for (int i = j + 1; i < 6; ++i) {
      double t = a[tri(j, i)];
#pragma unroll 1
      for (int k = 0; k < j; ++k) t -= a[tri(k, i)] * a[tri(k, j)] * d[k];
      a[tri(j, i)] = t * di;
    }
  }
  if (!ok) return false;
#pragma unroll 1
  for (int i = 0; i < 6; ++i) {
    double t = b[i];
#pragma unroll 1
    for (int k = 0; k < i; ++k) t -= a[tri(k, i)] * z[k];
    z[i] = t;
  }
  bool fin = true;
#pragma unroll 1
  for (int ii = 0; ii < 6; ++ii) {
    const int i = 5 - ii;
    double t = z[i] * dinv[i];
#pragma unroll 1
    for (int k = i + 1; k < 6; ++k) t -= a[tri(i, k)] * yout[k];
    yout[i] = t;
    fin = fin && isfinite(t);
  }
  return fin;
}

// minimise 0.5 y^T B y + g^T y on |y| = radius (2-D): the boundary problem of the subspace dogleg
// (dogleg_strategy.cc FindMinimumOnTrustRegionBoundary). Angular bracketing + bisection on f'.
__device__ __noinline__ void min_on_boundary_2d(const double B[4], const double g[2], double radius, double y[2]) {
  const double b01 = 0.5 * (B[1] + B[2]);
  double best_t = 0.0, best_f = DBL_MAX;
  const int N = 1024;
  const double two_pi = 6.283185307179586476925;
  auto f = [&](double t) {
    double s, c; sincos(t, &s, &c);
    c *= radius; s *= radius;
    return 0.5 * (B[0] * c * c + 2.0 * b01 * c * s + B[3] * s * s) + g[0] * c + g[1] * s;
  };
  auto df = [&](double t) {
    double s, c; sincos(t, &s, &c);
    return radius * radius * ((B[3] - B[0]) * c * s + b01 * (c * c - s * s)) + radius * (-g[0] * s + g[1] * c);
  };
  double d_prev = df(0.0), f_prev = f(0.0);
  for (int i = 0; i < N; ++i) {
    const double t0 = two_pi * i / N, t1 = two_pi * (i + 1) / N;
    const double d1 = df(t1), f1 = f(t1);
    double cand_t, cand_f;
    if (d_prev < 0.0 && d1 > 0.0) {
      double lo = t0, hi = t1;
      for (int it = 0; it < 100; ++it) {
        const double mid = 0.5 * (lo + hi);
        if (df(mid) < 0.0) lo = mid; else hi = mid;
      }
      cand_t = 0.5 * (lo + hi); cand_f = f(cand_t);
    } else if (f_prev < f1) { cand_t = t0; cand_f = f_prev; }
    else { cand_t = t1; cand_f = f1; }
    if (cand_f < best_f) { best_f = cand_f; best_t = cand_t; }
    d_prev = d1; f_prev = f1;
  }
  double s, c; sincos(best_t, &s, &c);
  y[0] = radius * c; y[1] = radius * s;
}

// Gauss-Newton model of DoglegStrategy::ComputeStep (first call after an accepted / invalid step), reduced to
// what the common path needs.  With D^2_i = clamp((S H S)_ii), the regularised Gauss-Newton solve is
//   (S H S + mu D^2) y = S g,   gauss_newton_step = -D.y,   dogleg step inside the radius = gn / D = -y,
// so neither D nor the scaled gradient is needed unless the step leaves the trust region (computed lazily in
// compute_subspace).  |D.y| = sqrt(sum D^2_i y_i^2): one square root.
struct GnModel {
  double scale[6];     // jacobi scaling used
  double d2[6];        // clamped squared column norms of the scaled Jacobian (= D^2)
  double y[6];         // solution of the regularised normal equations
  double gn_norm, mu_lm;
  int ok;              // 0 = LINEAR_SOLVER_FAILURE
  int pad;
};

__device__ __forceinline__ void gn_model(const double H[21], const double g[6], const double scale[6], double mu_lm,
                                         GnModel& m) {
  double gs[6], d2[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    gs[i] = scale[i] * g[i];
    d2[i] = fmin(fmax(scale[i] * H[tri(i, i)] * scale[i], 1e-6), 1e32);          // min/max_lm_diagonal of (S H S)_ii
  }
  bool ok = false;
  double y[6] = {0, 0, 0, 0, 0, 0};
  while (mu_lm < 1.0) {                                         // kMaxMu
    double A[21];                                               // (S H S + mu D^2), packed upper triangle, rebuilt per try
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
      for (int j = i; j < 6; ++j) A[tri(i, j)] = scale[i] * H[tri(i, j)] * scale[j];
#pragma unroll
    for (int i = 0; i < 6; ++i) A[tri(i, i)] += mu_lm * d2[i];
    if (ldlt_solve6_packed(A, gs, y)) { ok = true; break; }
    mu_lm *= 10.0;                                              // mu_increase_factor_
  }
  double n2 = 0.0;
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    m.scale[i] = scale[i];
    m.d2[i] = d2[i];
    m.y[i] = ok ? y[i] : 0.0;
    n2 += d2[i] * m.y[i] * m.y[i];
  }
  m.gn_norm = sqrt(n2);
  m.mu_lm = mu_lm;
  m.ok = ok ? 1 : 0;
}

// gn_model with the rolled factorisation; ws: 21 + 6 + 6 + 18 doubles of shared-memory scratch
__device__ __forceinline__ void gn_model_rolled(const double H[21], const double g[6], const double scale[6], double mu_lm,
                                                GnModel& m, double* ws) {
  double* A = ws; double* gs = ws + 21; double* y = ws + 27; double* w = ws + 33;
  double d2[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    gs[i] = scale[i] * g[i];
    d2[i] = fmin(fmax(scale[i] * H[tri(i, i)] * scale[i], 1e-6), 1e32);          // min/max_lm_diagonal of (S H S)_ii
    y[i] = 0.0;
  }
  bool ok = false;
  while (mu_lm < 1.0) {                                         // kMaxMu
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
      for (int j = i; j < 6; ++j) A[tri(i, j)] = scale[i] * H[tri(i, j)] * scale[j];
#pragma unroll
    for (int i = 0; i < 6; ++i) A[tri(i, i)] += mu_lm * d2[i];
    if (ldlt_solve6_rolled(A, gs, y, w)) { ok = true; break; }
    mu_lm *= 10.0;                                              // mu_increase_factor_
  }
  double n2 = 0.0;
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    m.scale[i] = scale[i];
    m.d2[i] = d2[i];
    m.y[i] = ok ? y[i] : 0.0;
    n2 += d2[i] * m.y[i] * m.y[i];
  }
  m.gn_norm = sqrt(n2);
  m.mu_lm = mu_lm;
  m.ok = ok ? 1 : 0;
}

// The same model by ONE WARP (all 32 lanes call; lanes 0..5 own one column of the packed upper triangle each, every
// lane returns the full result).  Every element goes through the same operations in the same order as in
// ldlt_solve6_packed / gn_model (sums over k ascending, (L L) d, six reciprocals), so the result is bit-identical; what
// changes is that the 15 off-diagonal eliminations of a column, and the column's products, run side by side instead of
// one after the other -- the serial form was 4.9k cycles of mostly instruction fetch and dependent FP64 latency.
__device__ __forceinline__ void gn_model_warp(const double* Hs /* shared: packed H[21] */, const double g[6], const double scale[6],
                                              double mu_lm, GnModel& m) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int me = lane < 6 ? lane : 5;                       // lanes >= 6 shadow lane 5 (their results are never read)
  double gs[6], d2[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    gs[i] = scale[i] * g[i];
    d2[i] = fmin(fmax(scale[i] * Hs[tri(i, i)] * scale[i], 1e-6), 1e32);          // min/max_lm_diagonal of (S H S)_ii
  }
  // my column of S H S: entries (k, me), k <= me
  double hcol[6], sme = scale[0];
#pragma unroll
  for (int k = 0; k < 6; ++k) { hcol[k] = Hs[tri(k < me ? k : me, me)]; if (k == me) sme = scale[k]; }
  bool ok = false;
  double y[6] = {0, 0, 0, 0, 0, 0};
  while (mu_lm < 1.0) {                                         // kMaxMu
    double col[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      col[k] = scale[k] * hcol[k] * sme;                        // A[tri(k, me)] = scale[k] * H[tri(k, me)] * scale[me]
      if (k == me) col[k] += mu_lm * d2[k];
    }
    double d[6], dinv[6];
    bool pos = true;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      double s = col[j];                                        // lane j: its diagonal entry
#pragma unroll
      for (int k = 0; k < 6; ++k)
        if (k < j) s -= col[k] * col[k] * d[k];
      d[j] = __shfl_sync(full, s, j);
      pos = pos && (d[j] > 0.0) && isfinite(d[j]);
      dinv[j] = 1.0 / d[j];
      double t = col[j];                                        // lanes i > j: entry (j, i)
#pragma unroll
      for (int k = 0; k < 6; ++k)
        if (k < j) {
          const double ljk = __shfl_sync(full, col[k], j);      // entry (k, j) = L(j, k)
          t -= col[k] * ljk * d[k];
        }
      if (me > j) col[j] = t * dinv[j];
    }
    if (pos) {
      // forward substitution: step i takes lane i's value
      double z[6];
      double mygs = gs[0];
#pragma unroll
      for (int k = 0; k < 6; ++k) if (k == me) mygs = gs[k];
#pragma unroll
      for (int i = 0; i < 6; ++i) {
        double t = mygs;
#pragma unroll
        for (int k = 0; k < 6; ++k)
          if (k < i) t -= col[k] * z[k];
        z[i] = __shfl_sync(full, t, i);
      }
      // row me of the factor: entry (me, k), k > me, lives in lane k's column
      double rowv[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        rowv[k] = 0.0;
#pragma unroll
        for (int i = 0; i < 6; ++i)
          if (i < k) { const double v = __shfl_sync(full, col[i], k); if (i == me) rowv[k] = v; }
      }
      double myz = z[0], mydinv = dinv[0];
#pragma unroll
      for (int k = 0; k < 6; ++k) if (k == me) { myz = z[k]; mydinv = dinv[k]; }
#pragma unroll
      for (int ii = 0; ii < 6; ++ii) {
        const int i = 5 - ii;
        double t = myz * mydinv;
#pragma unroll
        for (int k = 0; k < 6; ++k)
          if (k > i) t -= rowv[k] * y[k];
        y[i] = __shfl_sync(full, t, i);
      }
      bool fin = true;
#pragma unroll
      for (int i = 0; i < 6; ++i) fin = fin && isfinite(y[i]);
      if (fin) { ok = true; break; }
    }
    mu_lm *= 10.0;                                              // mu_increase_factor_
  }
  double n2 = 0.0;
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    m.scale[i] = scale[i];
    m.d2[i] = d2[i];
    m.y[i] = ok ? y[i] : 0.0;
    n2 += d2[i] * m.y[i] * m.y[i];
  }
  m.gn_norm = sqrt(n2);
  m.mu_lm = mu_lm;
  m.ok = ok ? 1 : 0;
}

// single out-of-line copies of the Lie-group routines (the solver is instruction-fetch bound: keep it small)
#ifndef TLOAM_SOLVER_INLINE_LIE
#define TLOAM_SOLVER_INLINE_LIE 0
#endif
#if TLOAM_SOLVER_INLINE_LIE
#define TL_LIE_INLINE __forceinline__
#else
#define TL_LIE_INLINE __noinline__
#endif
__device__ TL_LIE_INLINE void s_exp(const double a[6], Pose7* out) { *out = se3_exp(a); }
__device__ TL_LIE_INLINE void s_log(const Pose7* p, double out[6]) { se3_log(*p, out); }
__device__ TL_LIE_INLINE void s_mul(const Pose7* a, const Pose7* b, Pose7* out) { *out = se3_mul(*a, *b); }

struct SolverIO {
  const DeviceCtx* ctx;
  FrameState* st;
  tloam_b200_stats* tr;
};

// profiling-mode stage timer: accumulates SM cycles since the previous stamp into dbg[slot]
#define TL_STAMP(io, slot)                                                        \
  do {                                                                            \
    if ((io).ctx->dbg) {                                                          \
      const long long now__ = clock64();                                          \
      (io).ctx->dbg[slot] += (unsigned long long)(now__ - (long long)(io).ctx->dbg[15]); \
      (io).ctx->dbg[15] = (unsigned long long)now__;                              \
    }                                                                             \
  } while (0)

__device__ __forceinline__ tloam_b200_outer_trace* outer_trace(const SolverIO& io) {
  return (io.tr && io.st->outer < TLOAM_B200_MAX_OUTER) ? &io.tr->outer[io.st->outer] : nullptr;
}
__device__ __forceinline__ tloam_b200_inner_trace* inner_trace(const SolverIO& io) {
  tloam_b200_outer_trace* ot = outer_trace(io);
  const int it = io.st->iter;
  return (ot && it >= 1 && it <= TLOAM_B200_MAX_INNER) ? &ot->inner[it - 1] : nullptr;
}

// |x - Plus(x, -g)|_inf  (TrustRegionMinimizer::EvaluateGradientAndJacobian), for pose P with tangent x
__device__ __noinline__ double gradient_max_norm(const Pose7& P, const double x[6], const double g[6]) {
  double ng[6], proj[6];
  for (int i = 0; i < 6; ++i) ng[i] = -g[i];
  Pose7 e, em;
  s_exp(ng, &e);
  s_mul(&e, &P, &em);
  s_log(&em, proj);
  double m = 0.0;
  for (int i = 0; i < 6; ++i) m = fmax(m, fabs(x[i] - proj[i]));
  return m;
}

__device__ __noinline__ void finish_frame(const SolverIO& io) {
  FrameState* st = io.st;
  Pose7 fin;
  s_exp(st->x, &fin);                                   // ref: registration.cpp:1124
  pose_to_matrix(fin, st->result);
  for (int i = 0; i < 16; ++i) st->curr_pose[i] = st->result[i];
  if (io.tr) for (int i = 0; i < 6; ++i) io.tr->x_final[i] = st->x[i];
  st->frame_done = 1;
}

// The Ceres solve of this outer iteration is over: GNC bookkeeping, ref: registration.cpp:1049-1121.
__device__ __noinline__ void end_of_solve(const SolverIO& io, int termination) {
  FrameState* st = io.st;
  const DeviceCtx& c = *io.ctx;
  tloam_b200_outer_trace* ot = outer_trace(io);
  const double mu = st->mu;
  st->th1 = (mu + 1.0) / mu * st->c2;                   // :1049
  st->th2 = mu / (mu + 1.0) * st->c2;                   // :1050
  st->mu_used = mu;
  if (ot) {
    ot->termination = termination;
    ot->final_cost = st->x_cost;
    ot->n_inner = st->iter;
    for (int i = 0; i < 6; ++i) ot->x_end[i] = st->x[i];
    ot->mu = mu; ot->th1 = st->th1; ot->th2 = st->th2;
    for (int k = 0; k < 4; ++k) ot->slot_sum[k] = st->slot_sum[k];
  }
  st->mu = mu * exp((double)(st->outer + 1) * c.gnc_factor);   // :1089
  if (io.tr) io.tr->n_outer = st->outer + 1;
  const double planar_cost = st->slot_sum[kPlanar];            // :1094
  const double diff = fabs(planar_cost - st->planar_prev);     // :1096
  if (diff < c.cost_threshold) {                               // :1108
    if (io.tr) io.tr->converged_early = 1;
    finish_frame(io);
    return;
  }
  st->planar_prev = planar_cost;                               // :1113
  st->outer += 1;
  if (st->outer >= c.max_iterations) { finish_frame(io); return; }
  st->phase = kPhaseIter0;        // next: k_correspond (weights updated + slots zeroed there), then k_eval<first>
  st->evalq = st->xq;
}

__device__ __forceinline__ void install_model(FrameState* st, const GnModel& m) {
  for (int i = 0; i < 6; ++i) { st->d2[i] = m.d2[i]; st->y[i] = m.y[i]; }
  st->gn_norm = m.gn_norm;
  st->mu_lm = m.mu_lm;
  st->sub_valid = 0;
}

// subspace model (DoglegStrategy::ComputeSubspaceModel): orthonormal basis of span{sgrad, gn} and the 2x2
// model in it.  Only needed when the Gauss-Newton step leaves the trust region, so it is computed lazily.
__device__ __noinline__ bool compute_subspace(FrameState* st) {
  for (int i = 0; i < 6; ++i) {               // the lazily needed vectors of the full model
    st->D[i] = sqrt(st->d2[i]);
    st->sgrad[i] = st->scale[i] * st->g[i] / st->D[i];
    st->gn[i] = -st->D[i] * st->y[i];
  }
  const double n0 = norm6(st->sgrad), n1 = st->gn_norm;
  const double* first = (n0 >= n1) ? st->sgrad : st->gn;
  const double* second = (n0 >= n1) ? st->gn : st->sgrad;
  const double nf = fmax(n0, n1);
  if (nf == 0.0) return false;
  double u0[6], u1[6], pr = 0.0;
  for (int i = 0; i < 6; ++i) { u0[i] = first[i] / nf; pr += u0[i] * second[i]; }
  for (int i = 0; i < 6; ++i) u1[i] = second[i] - pr * u0[i];
  const double n2 = norm6(u1);
  st->sub_1d = !(n2 > nf * 6.0 * DBL_EPSILON);
  if (!st->sub_1d) {
    double t0[6], t1[6];
    st->sub_g[0] = st->sub_g[1] = 0.0;
    for (int i = 0; i < 6; ++i) {
      u1[i] /= n2;
      st->sub_basis[i] = u0[i]; st->sub_basis[6 + i] = u1[i];
      st->sub_g[0] += u0[i] * st->sgrad[i]; st->sub_g[1] += u1[i] * st->sgrad[i];
      t0[i] = u0[i] / st->D[i]; t1[i] = u1[i] / st->D[i];
    }
    double b00 = 0, b01 = 0, b11 = 0;
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j < 6; ++j) {
        const double h = ((i <= j) ? st->H[tri(i, j)] : st->H[tri(j, i)]) * st->scale[i] * st->scale[j];
        b00 += t0[i] * h * t0[j];
        b01 += t0[i] * h * t1[j];
        b11 += t1[i] * h * t1[j];
      }
    st->sub_B[0] = b00; st->sub_B[1] = st->sub_B[2] = b01; st->sub_B[3] = b11;
  }
  st->sub_valid = 1;
  return true;
}

// Loop "compute step -> candidate" until a candidate needs a fresh evaluation (returns with
// phase = kPhaseCand) or the solve terminates (end_of_solve called).
__device__ __forceinline__ void advance(const SolverIO& io) {
  FrameState* st = io.st;
  const DeviceCtx& c = *io.ctx;
  while (true) {
    if (st->iter >= c.ceres_max_it) { end_of_solve(io, 0); return; }   // MaxSolverIterationsReached
    st->iter += 1;
    tloam_b200_inner_trace* it = inner_trace(io);
    bool solver_ok = st->model_ok != 0;
    if (!st->reuse) {                                                  // only after an invalid step
      st->reuse = 1;
      GnModel m;
      double H[21], g[6], sc[6];
      for (int i = 0; i < 21; ++i) H[i] = st->H[i];
      for (int i = 0; i < 6; ++i) { g[i] = st->g[i]; sc[i] = st->scale[i]; }
      gn_model(H, g, sc, st->mu_lm, m);
      install_model(st, m);
      st->model_ok = m.ok;
      solver_ok = m.ok != 0;
    }
    double step[6] = {0, 0, 0, 0, 0, 0};
    if (solver_ok) {                                                   // ComputeSubspaceDoglegStep
      if (st->gn_norm <= st->radius) {
        for (int i = 0; i < 6; ++i) step[i] = -st->y[i];              // gauss_newton_step / D
        st->step_norm = st->gn_norm; st->used_gn = 1;
      } else {
        if (!st->sub_valid) solver_ok = compute_subspace(st);
        if (solver_ok) {
          if (st->sub_1d) {
            const double gnm = norm6(st->sgrad);
            for (int i = 0; i < 6; ++i) step[i] = -(st->radius / gnm) * st->sgrad[i] / st->D[i];
          } else {
            double y2[2];
            min_on_boundary_2d(st->sub_B, st->sub_g, st->radius, y2);
            for (int i = 0; i < 6; ++i) step[i] = (st->sub_basis[i] * y2[0] + st->sub_basis[6 + i] * y2[1]) / st->D[i];
          }
          st->step_norm = st->radius; st->used_gn = 0;
        }
      }
    }
    // model cost change = -(g_s.step + step^T H_s step / 2)
    double mcc = 0.0;
    bool valid = false;
    if (solver_ok) {
      double v[6], lin = 0.0, quad = 0.0;
      for (int i = 0; i < 6; ++i) { v[i] = st->scale[i] * step[i]; lin += st->g[i] * v[i]; }
      for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) quad += v[i] * ((i <= j) ? st->H[tri(i, j)] : st->H[tri(j, i)]) * v[j];
      mcc = -(lin + 0.5 * quad);
      valid = mcc > 0.0;
    }
    st->model_cost_change = mcc;
    if (it) {
      it->radius = st->radius; it->step_norm_scaled = st->step_norm; it->used_gauss_newton = st->used_gn;
      it->model_cost_change = mcc; it->accepted = 0; it->relative_decrease = 0.0; it->candidate_cost = 0.0;
    }
    if (!valid) {                                                      // HandleInvalidStep
      st->num_invalid += 1;
      if (it) it->accepted = -1;
      if (st->num_invalid >= 5) { end_of_solve(io, 6); return; }
      st->mu_lm *= 10.0; st->reuse = 0;                                // StepIsInvalid
      continue;
    }
    st->num_invalid = 0;
    double delta[6];
    for (int i = 0; i < 6; ++i) delta[i] = step[i] * st->scale[i];     // undo the Jacobi scaling
    Pose7 ed, cq;
    s_exp(delta, &ed);
    s_mul(&ed, &st->xq, &cq);                                          // Plus: exp(delta) * exp(x)
    bool same = st->last_cand_valid != 0;
    same = same && cq.qw == st->last_candq.qw && cq.qx == st->last_candq.qx && cq.qy == st->last_candq.qy &&
           cq.qz == st->last_candq.qz && cq.tx == st->last_candq.tx && cq.ty == st->last_candq.ty &&
           cq.tz == st->last_candq.tz;
    if (same) {
      // identical to the candidate that was just evaluated and rejected (reuse_ = true and the
      // Gauss-Newton step still fits the halved radius): the evaluation, both tolerance tests and the step
      // quality repeat exactly, so the step is rejected again without re-running the kernel.
      if (it) {
        for (int i = 0; i < 6; ++i) it->x_candidate[i] = st->last_cand[i];
        it->candidate_cost = st->last_cand_cost;
        it->relative_decrease = (st->x_cost - st->last_cand_cost) / mcc;
        it->accepted = 0;
      }
      st->radius *= 0.5; st->reuse = 1;                                // StepRejected
      if (st->radius <= 1e-32) { end_of_solve(io, 4); return; }
      continue;
    }
    st->candq = cq;            // its tangent (cand) is computed by warp 3 of the next evaluation
    st->evalq = cq;
    st->phase = kPhaseCand;
    return;
  }
}

struct SolverShared {
  GnModel model;
  double proj[6];      // Plus(x, -g) for the state that becomes current if this evaluation is accepted
  double cand[6];      // log(candidate pose)
  // speculative first trip through advance() for the state that becomes current if this evaluation is accepted and
  // the Gauss-Newton step of the fresh model fits the trust region: model cost change and next candidate pose
  double spec_mcc;
  Pose7 spec_cq;
  int spec_ok, pad;
  double ldlt_ws[51];  // scratch of the rolled LDL^T (gn_model_rolled)
  FrameState backup;   // state before advance(), for the (practically never taken) gradient-tolerance exit
};

__device__ __forceinline__ void bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void bar_arrive(int id, int nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Entered by ALL threads of the last block (kBlk = 128 = 4 warps) after the per-block partials have been summed
// into tot[kNRed].  `st` is a shared-memory copy of ctx.st (the caller writes it back).
//
//   warp 3 : cand = log(candidate pose)                                    -> named barrier 1
//   warp 1 : proj = Plus(x', -g') = log(exp(-g') * P')                     -> named barrier 2
//            (x', P', g' = tangent, pose, gradient of the state that is current after an accepted step)
//   warp 2 : Gauss-Newton model from the fresh H, g, then -- still in registers -- the first trip through advance()
//            that follows an accepted evaluation in the common case (Gauss-Newton step inside the trust region):
//            model cost change and next candidate pose exp(delta) * P'     -> named barrier 3
//            (everything speculative: used iff the evaluation is accepted, same operations in the same order
//            as advance(), so the results are bit-identical to the serial path)
//   warp 0 : wait 1 | tolerance tests, accept / reject | wait 3 | install the model, take the speculative step or
//            fall back to advance() (rejected step, dogleg, invalid step) | wait 2 | gradient-tolerance test
// Measured before the split (thread 0 did model -> decision -> advance() in sequence): 14k cycles per active
// evaluation = 3.5k model + 2.1k decision + 6.2k advance() + tail.
// The gradient-tolerance test (|x' - proj|_inf <= 1e-10) comes BEFORE advance() in Ceres; it practically never
// fires (it needs |g| ~ 1e-10), so advance() runs first on a backed-up state and is undone if it does fire.
__device__ __noinline__ void solver_on_eval(const DeviceCtx& ctx, FrameState* st, const double* tot, SolverShared* sh) {
  SolverIO io{&ctx, st, ctx.stats};
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool iter0 = st->phase == kPhaseIter0;
  // inputs of the helper warps are copied to registers before anybody mutates the state
  Pose7 P = iter0 ? st->xq : st->candq;
  double g[6];
  for (int i = 0; i < 6; ++i) g[i] = tot[21 + i];
  __syncthreads();
  long long ta0 = 0;
  if (ctx.dbg) ta0 = clock64();

  if (warp == 3) {
    if (lane == 0 && !iter0) {
      s_log(&P, sh->cand);
      if (ctx.dbg) ctx.dbg[7] += (unsigned long long)(clock64() - ta0);
    }
    __syncwarp();
    bar_arrive(1, 64);
    return;
  }
  if (warp == 1) {
    if (lane == 0) {
      double ng[6];
      for (int i = 0; i < 6; ++i) ng[i] = -g[i];
      Pose7 e, em;
      s_exp(ng, &e);
      s_mul(&e, &P, &em);
      s_log(&em, sh->proj);
      if (ctx.dbg) ctx.dbg[5] += (unsigned long long)(clock64() - ta0);
    }
    __syncwarp();
    bar_arrive(2, 64);
    return;
  }
  if (warp == 2) {
    double sc[6];
    for (int i = 0; i < 6; ++i)
      sc[i] = iter0 ? 1.0 / (1.0 + sqrt(tot[tri(i, i)])) : st->scale[i];            // jacobi scaling (iteration 0 only)
    const double mu0 = iter0 ? 1e-8 : fmax(1e-8, 2.0 * st->mu_lm / 10.0);          // kMinMu / StepAccepted
#ifndef TLOAM_SOLVER_WARP_MODEL
#define TLOAM_SOLVER_WARP_MODEL 0    // 1: gn_model_warp (measured: 6.1k cycles vs 4.9k for the serial form -- more instructions)
#endif
    GnModel m;
    if (TLOAM_SOLVER_WARP_MODEL) gn_model_warp(tot, g, sc, mu0, m);               // the whole warp
    if (lane == 0) {
      double H[21];
      for (int i = 0; i < 21; ++i) H[i] = tot[i];
#ifndef TLOAM_SOLVER_ROLLED_MODEL
#define TLOAM_SOLVER_ROLLED_MODEL 0   // 1: gn_model_rolled (measured: 11.3k cycles vs 5.0k -- shared-memory latency on every operand)
#endif
      if (!TLOAM_SOLVER_WARP_MODEL) {
        if (TLOAM_SOLVER_ROLLED_MODEL) gn_model_rolled(H, g, sc, mu0, m, sh->ldlt_ws);
        else gn_model(H, g, sc, mu0, m);
      }
      sh->model = m;
      if (ctx.dbg) ctx.dbg[6] += (unsigned long long)(clock64() - ta0);
      int ok = 0;
      if (m.ok) {
        // advance() for "accepted, Gauss-Newton step inside the radius": step = -y, model cost change, Plus
        double step[6], v[6], lin = 0.0, quad = 0.0;
        for (int i = 0; i < 6; ++i) step[i] = -m.y[i];
        for (int i = 0; i < 6; ++i) { v[i] = sc[i] * step[i]; lin += g[i] * v[i]; }
        for (int i = 0; i < 6; ++i)
          for (int j = 0; j < 6; ++j) quad += v[i] * ((i <= j) ? H[tri(i, j)] : H[tri(j, i)]) * v[j];
        sh->spec_mcc = -(lin + 0.5 * quad);
        double delta[6];
        for (int i = 0; i < 6; ++i) delta[i] = step[i] * sc[i];
        Pose7 ed, cq;
        s_exp(delta, &ed);
        s_mul(&ed, &P, &cq);
        sh->spec_cq = cq;
        ok = 1;
      }
      sh->spec_ok = ok;
      if (ctx.dbg) ctx.dbg[13] += (unsigned long long)(clock64() - ta0);
    }
    __syncwarp();
    bar_arrive(3, 64);
    return;
  }
  if (warp != 0) return;

  // ------------------------------- warp 0 -------------------------------
  if (lane == 0 && ctx.dbg) ctx.dbg[15] = (unsigned long long)clock64();
  bar_sync(1, 64);                                                       // cand is ready

  // 0 = solve ended, 1 = go on with advance() and then the deferred gradient-tolerance test,
  // 2 = go on with advance(), no gradient test (step rejected)
  int go = 0, copy_hg = 0, trace_h0 = 0, take_scale = 0, take_model = 0;
  if (lane == 0) {
    const double cost = tot[27];
    for (int k = 0; k < 4; ++k) st->slot_sum[k] = tot[28 + k];
    tloam_b200_outer_trace* ot = outer_trace(io);
    if (!isfinite(cost)) {
      st->status = TLOAM_B200_ERR_NUMERIC;
      finish_frame(io);
    } else if (iter0) {
      // ---- IterationZero ----
      st->iter = 0; st->num_invalid = 0; st->last_cand_valid = 0;
      st->radius = ctx.initial_radius;                                   // initial_trust_region_radius
      int nf_total = 0;
      for (int k = 0; k < 4; ++k) {
        const int nf = (int)(tot[32 + k] + 0.5);
        nf_total += nf;
        if (ot) ot->n_factors[k] = nf;
      }
      st->x_cost = cost;
      copy_hg = 1;                                                       // H, g <- tot (done by the whole warp below)
      if (ot) ot->initial_cost = cost;
      trace_h0 = ot != nullptr;
      st->mu_lm = 1e-8; st->reuse = 0; st->model_ok = 0;
      if (nf_total == 0) {
        take_scale = 1;                                                  // the scaling is part of the state either way
        end_of_solve(io, 5);                                             // no residual blocks
      } else {
        st->x_norm = norm6(st->x);
        take_scale = 1; take_model = 1;                                  // after barrier 3 (the model is warp 2's)
        go = 1;
      }
    } else {
      // ---- the evaluation was at the candidate ----
      for (int i = 0; i < 6; ++i) st->cand[i] = sh->cand[i];
      tloam_b200_inner_trace* it = inner_trace(io);
      if (it) {
        it->candidate_cost = cost;
        for (int i = 0; i < 6; ++i) it->x_candidate[i] = st->cand[i];
      }
      double d[6];
      for (int i = 0; i < 6; ++i) d[i] = st->x[i] - st->cand[i];
      if (norm6(d) <= 1e-8 * (st->x_norm + 1e-8)) {                      // ParameterToleranceReached
        if (it) it->accepted = 2;
        end_of_solve(io, 2);
      } else if (fabs(st->x_cost - cost) <= 1e-6 * st->x_cost) {         // FunctionToleranceReached
        if (it) it->accepted = 2;
        end_of_solve(io, 1);
      } else {
        const double rel = (st->x_cost - cost) / st->model_cost_change;  // StepQuality (monotonic)
        if (it) it->relative_decrease = rel;
        if (rel > 1e-3) {                                                // min_relative_decrease
          // HandleSuccessfulStep
          for (int i = 0; i < 6; ++i) st->x[i] = st->cand[i];
          st->xq = st->candq;
          st->x_norm = norm6(st->x);
          st->x_cost = cost;
          copy_hg = 1;
          if (rel < 0.25) st->radius *= 0.5;                             // DoglegStrategy::StepAccepted
          if (rel > 0.75) st->radius = fmax(st->radius, 3.0 * st->step_norm);
          st->last_cand_valid = 0;
          if (it) it->accepted = 1;
          take_model = 1;                                                // speculative model becomes current (after barrier 3)
          go = 1;
        } else {
          st->radius *= 0.5; st->reuse = 1;                              // StepRejected
          for (int i = 0; i < 6; ++i) st->last_cand[i] = st->cand[i];
          st->last_candq = st->candq;
          st->last_cand_cost = cost; st->last_cand_valid = 1;
          if (it) it->accepted = 0;
          go = 2;
        }
        if (go != 0 && st->radius <= 1e-32 && go == 2) { end_of_solve(io, 4); go = 0; }   // MinTrustRegionRadiusReached
      }
    }
    TL_STAMP(io, 11);
  }
  go = __shfl_sync(0xffffffffu, go, 0);
  copy_hg = __shfl_sync(0xffffffffu, copy_hg, 0);
  trace_h0 = __shfl_sync(0xffffffffu, trace_h0, 0);
  take_scale = __shfl_sync(0xffffffffu, take_scale, 0);
  take_model = __shfl_sync(0xffffffffu, take_model, 0);
  if (copy_hg) {                                                         // lane-parallel: H (21) + g (6) <- tot
    if (lane < 27) { if (lane < 21) st->H[lane] = tot[lane]; else st->g[lane - 21] = tot[lane]; }
    __syncwarp();
  }
  if (trace_h0) {                                                        // lane-parallel trace of the iteration-0 system
    tloam_b200_outer_trace* ot = outer_trace(io);
    for (int e = lane; e < 36; e += 32) { const int i = e / 6, j = e % 6; ot->H0[e] = (i <= j) ? tot[tri(i, j)] : tot[tri(j, i)]; }
    if (lane < 6) { ot->x_start[lane] = st->x[lane]; ot->g0[lane] = tot[21 + lane]; }
    __syncwarp();
  }
  if (go == 1) {
    // back up the state (warp-wide copy) while warp 2 is still busy: everything the deferred gradient-tolerance exit
    // needs (x, cost, radius, GNC bookkeeping) is final here; the Gauss-Newton model installed below is not part of it
    const unsigned long long* src = reinterpret_cast<const unsigned long long*>(st);
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(&sh->backup);
    for (unsigned i = lane; i < sizeof(FrameState) / 8; i += 32) dst[i] = src[i];
    __syncwarp();
  }
  bar_sync(3, 64);                                                       // model + speculative step are ready
  if (take_scale && lane < 6) st->scale[lane] = sh->model.scale[lane];
  if (take_model) {                                                      // install_model(), one lane per entry
    if (lane < 6) { st->d2[lane] = sh->model.d2[lane]; st->y[lane] = sh->model.y[lane]; }
    if (lane == 6) { st->gn_norm = sh->model.gn_norm; st->mu_lm = sh->model.mu_lm; }
    if (lane == 7) { st->sub_valid = 0; st->model_ok = sh->model.ok; st->reuse = 1; }
  }
  __syncwarp();
  if (lane == 0 && go != 0) {
    // after an accepted step Ceres tests the radius AFTER the gradient tolerance; the gradient test is deferred
    // (below), so the radius test of the accepted branch is applied there as well
    if (go == 2 || st->radius > 1e-32) {
      // the speculative step IS advance()'s first trip when: accepted (reuse = 1, no rejected candidate on record),
      // iterations left, model solved, Gauss-Newton step inside the (updated) radius, valid step
#ifndef TLOAM_SOLVER_NO_SPEC
#define TLOAM_SOLVER_NO_SPEC 0       // 1: always take the serial advance() (A/B and bit-identity check of the speculative step)
#endif
      if (!TLOAM_SOLVER_NO_SPEC && go == 1 && st->iter < ctx.ceres_max_it && sh->spec_ok && st->model_ok && st->gn_norm <= st->radius &&
          sh->spec_mcc > 0.0) {
        st->iter += 1;
        st->step_norm = st->gn_norm; st->used_gn = 1;
        st->model_cost_change = sh->spec_mcc;
        tloam_b200_inner_trace* it = inner_trace(io);
        if (it) {
          it->radius = st->radius; it->step_norm_scaled = st->step_norm; it->used_gauss_newton = 1;
          it->model_cost_change = sh->spec_mcc; it->accepted = 0; it->relative_decrease = 0.0; it->candidate_cost = 0.0;
        }
        st->num_invalid = 0;
        st->candq = sh->spec_cq;
        st->evalq = sh->spec_cq;
        st->phase = kPhaseCand;
      } else {
        advance(io);
      }
    }
    TL_STAMP(io, 12);
  }
  __syncwarp();
  bar_sync(2, 64);                                                       // proj is ready
  int undo = 0;
  if (lane == 0 && go == 1) {
    const FrameState* b = &sh->backup;                                   // x' = tangent of the accepted state
    double gmax = 0.0;
    for (int i = 0; i < 6; ++i) gmax = fmax(gmax, fabs(b->x[i] - sh->proj[i]));
    if (gmax <= 1e-10) undo = 3;                                         // GradientToleranceReached
    else if (b->radius <= 1e-32) undo = 4;                               // MinTrustRegionRadiusReached
  }
  undo = __shfl_sync(0xffffffffu, undo, 0);
  if (undo != 0) {
    const unsigned long long* src = reinterpret_cast<const unsigned long long*>(&sh->backup);
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(st);
    for (unsigned i = lane; i < sizeof(FrameState) / 8; i += 32) dst[i] = src[i];
    __syncwarp();
    if (lane == 0) end_of_solve(io, undo);
  }
}

}  // namespace tloam
