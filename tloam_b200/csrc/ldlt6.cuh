// ldlt6.cuh -- the packed 6x6 LDL^T solve shared by the registration solver (solver.cuh) and loop verification
// (loop_verify.cu).  Header-only and kernel-free, so including it adds no kernel to a library.
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace tloam {

// upper-triangle index of (i,j), i <= j, row-major packed (21 entries)
__host__ __device__ __forceinline__ int tri(int i, int j) { return i * 6 - (i * (i - 1)) / 2 + (j - i); }

// LDL^T solve of the SPD 6x6 system A y = b on the PACKED upper triangle (21 entries, tri(i,j), i <= j), IN PLACE: the
// factor overwrites A (L(i,j), i > j, lands in a[tri(j,i)]).  Fully unrolled with compile-time indices only, so the
// whole factorisation lives in registers: the previous full-matrix form kept A / L / H_s (3 x 36 doubles) in LOCAL
// memory (221 LDL/STL in the SASS of k_eval, most of the 3.5k cycles of the Gauss-Newton model).  Same operations in
// the same order as before (sum over k ascending, (L L) d), six reciprocals, no square roots.  Returns false if a
// pivot is not positive / finite.
__device__ __forceinline__ bool ldlt_solve6_packed(double a[21], const double b[6], double y[6]) {
  // every loop runs over the constant range 0..5 with the triangular bounds as (compile-time) predicates: loops whose
  // bounds depend on an outer unrolled variable were left rolled by the front end, which put `a` in local memory
  double d[6], dinv[6];
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    double s = a[tri(j, j)];
#pragma unroll
    for (int k = 0; k < 6; ++k)
      if (k < j) s -= a[tri(k, j)] * a[tri(k, j)] * d[k];
    d[j] = s;
    ok = ok && (s > 0.0) && isfinite(s);
    dinv[j] = 1.0 / s;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      if (i > j) {
        double t = a[tri(j, i)];
#pragma unroll
        for (int k = 0; k < 6; ++k)
          if (k < j) t -= a[tri(k, i)] * a[tri(k, j)] * d[k];
        a[tri(j, i)] = t * dinv[j];
      }
    }
  }
  if (!ok) return false;
  double z[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    double t = b[i];
#pragma unroll
    for (int k = 0; k < 6; ++k)
      if (k < i) t -= a[tri(k, i)] * z[k];
    z[i] = t;
  }
#pragma unroll
  for (int ii = 0; ii < 6; ++ii) {
    const int i = 5 - ii;
    double t = z[i] * dinv[i];
#pragma unroll
    for (int k = 0; k < 6; ++k)
      if (k > i) t -= a[tri(i, k)] * y[k];
    y[i] = t;
  }
  bool fin = true;
#pragma unroll
  for (int i = 0; i < 6; ++i) fin = fin && isfinite(y[i]);
  return fin;
}

}  // namespace tloam
