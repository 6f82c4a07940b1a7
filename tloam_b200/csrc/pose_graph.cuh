// pose_graph.cuh -- the rigid-matrix helper the pose-graph kernels share (pose_graph.cu, pose_graph_robust.cu), so that the
// robust back end evaluates a loop edge's residual with the operation order of k_pg_linearize.
#pragma once

namespace tloam {

#define PGM(m, r, c) (m)[4 * (c) + (r)]

// C = A^-1 B of rigid column-major 4 x 4 matrices: R_A^T R_B, R_A^T (t_B - t_A)
__device__ void pg_inv_mul(const double* A, const double* B, double* C) {
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) PGM(C, r, c) = PGM(A, 0, r) * PGM(B, 0, c) + PGM(A, 1, r) * PGM(B, 1, c) + PGM(A, 2, r) * PGM(B, 2, c);
    PGM(C, r, 3) = PGM(A, 0, r) * (PGM(B, 0, 3) - PGM(A, 0, 3)) + PGM(A, 1, r) * (PGM(B, 1, 3) - PGM(A, 1, 3)) +
                   PGM(A, 2, r) * (PGM(B, 2, 3) - PGM(A, 2, 3));
    PGM(C, 3, r) = 0.0;
  }
  PGM(C, 3, 3) = 1.0;
}

}  // namespace tloam
