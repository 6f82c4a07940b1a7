// normal_fit.cuh -- the per-row normal of a neighbourhood (include/tloam_b200.h, "Loop verification against a submap",
// Normals): the covariance sums, their quotient by the count, the cyclic Jacobi eigen-solve and the validity rule, every
// operation a separately rounded intrinsic.  Shared by libtloam_b200_loopvs.so (loop_verify_submap.cu, neighbours from an
// exhaustive scan) and libtloam_b200_loc.so (localize.cu, neighbours from the prior map's grid), so the rule lives in one
// place.  Device functions only: no kernel is defined here.
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace tloam {

__device__ __forceinline__ double nf_dot3(double a0, double b0, double a1, double b1, double a2, double b2) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a0, b0), __dmul_rn(a1, b1)), __dmul_rn(a2, b2));
}

__device__ __forceinline__ double nf_d2(double px, double py, double pz, double mx, double my, double mz) {
  const double dx = __dsub_rn(px, mx), dy = __dsub_rn(py, my), dz = __dsub_rn(pz, mz);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// c (xx, xy, xz, yy, yz, zz) += the products of neighbour (x, y, z)'s offsets from the mean
__device__ __forceinline__ void nf_cov_add(double c[6], double x, double y, double z, double mx, double my, double mz) {
  const double dx = __dsub_rn(x, mx), dy = __dsub_rn(y, my), dz = __dsub_rn(z, mz);
  c[0] = __dadd_rn(c[0], __dmul_rn(dx, dx)); c[1] = __dadd_rn(c[1], __dmul_rn(dx, dy));
  c[2] = __dadd_rn(c[2], __dmul_rn(dx, dz)); c[3] = __dadd_rn(c[3], __dmul_rn(dy, dy));
  c[4] = __dadd_rn(c[4], __dmul_rn(dy, dz)); c[5] = __dadd_rn(c[5], __dmul_rn(dz, dz));
}

// cyclic Jacobi of the symmetric c (xx, xy, xz, yy, yz, zz): at most 32 sweeps over (0,1), (0,2), (1,2), a rotation
// skipped when its entry is 0, done once off <= 1e-32 diag; eigenvalues ascending by three compare-exchanges (ties keep
// the lower axis first), nvec the eigenvector of the least.  Every operation separately rounded.
__device__ __forceinline__ void nf_jacobi3(const double c[6], double eig[3], double nvec[3]) {
  double a[3][3] = {{c[0], c[1], c[2]}, {c[1], c[3], c[4]}, {c[2], c[4], c[5]}};
  double v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
#pragma unroll 1
  for (int sweep = 0; sweep < 32; ++sweep) {
    const double off = nf_dot3(a[0][1], a[0][1], a[0][2], a[0][2], a[1][2], a[1][2]);
    const double diag = nf_dot3(a[0][0], a[0][0], a[1][1], a[1][1], a[2][2], a[2][2]);
    if (off <= __dmul_rn(1e-32, diag) || off == 0.0) break;
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
      for (int q = p + 1; q < 3; ++q) {
        if (a[p][q] == 0.0) continue;
        const double theta = __ddiv_rn(__dsub_rn(a[q][q], a[p][p]), __dmul_rn(2.0, a[p][q]));
        const double t = __ddiv_rn(theta >= 0 ? 1.0 : -1.0, __dadd_rn(fabs(theta), __dsqrt_rn(__dadd_rn(__dmul_rn(theta, theta), 1.0))));
        const double cs = __ddiv_rn(1.0, __dsqrt_rn(__dadd_rn(__dmul_rn(t, t), 1.0))), sn = __dmul_rn(t, cs);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double akp = a[k][p], akq = a[k][q];
          a[k][p] = __dsub_rn(__dmul_rn(cs, akp), __dmul_rn(sn, akq));
          a[k][q] = __dadd_rn(__dmul_rn(sn, akp), __dmul_rn(cs, akq));
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double apk = a[p][k], aqk = a[q][k];
          a[p][k] = __dsub_rn(__dmul_rn(cs, apk), __dmul_rn(sn, aqk));
          a[q][k] = __dadd_rn(__dmul_rn(sn, apk), __dmul_rn(cs, aqk));
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double vkp = v[k][p], vkq = v[k][q];
          v[k][p] = __dsub_rn(__dmul_rn(cs, vkp), __dmul_rn(sn, vkq));
          v[k][q] = __dadd_rn(__dmul_rn(sn, vkp), __dmul_rn(cs, vkq));
        }
      }
  }
  double d0 = a[0][0], d1 = a[1][1], d2 = a[2][2];
  double n0[3] = {v[0][0], v[1][0], v[2][0]}, n1[3] = {v[0][1], v[1][1], v[2][1]}, n2[3] = {v[0][2], v[1][2], v[2][2]};
  auto cswap = [](double& da, double& db, double* na, double* nb) {
    if (db < da) {
      const double t = da; da = db; db = t;
      for (int r = 0; r < 3; ++r) { const double u = na[r]; na[r] = nb[r]; nb[r] = u; }
    }
  };
  cswap(d0, d1, n0, n1);
  cswap(d1, d2, n1, n2);
  cswap(d0, d1, n0, n1);
  eig[0] = d0; eig[1] = d1; eig[2] = d2;
  nvec[0] = n0[0]; nvec[1] = n0[1]; nvec[2] = n0[2];
}

// the covariance sums c of cnt >= 1 neighbours divided by cnt, the eigen-solve, and the normal and its validity
__device__ __forceinline__ unsigned char nf_finish(int cnt, double c[6], int min_normal_neighbours, double max_planarity,
                                                   double nv[3]) {
  const double n = (double)cnt;
#pragma unroll
  for (int k = 0; k < 6; ++k) c[k] = __ddiv_rn(c[k], n);
  double eig[3];
  nf_jacobi3(c, eig, nv);
  return cnt >= min_normal_neighbours && eig[0] <= __dmul_rn(max_planarity, eig[1]) ? 1 : 0;
}

}  // namespace tloam
