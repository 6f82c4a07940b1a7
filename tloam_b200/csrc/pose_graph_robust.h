// pose_graph_robust.h -- the C launcher of libtloam_b200_pgr.so (pose_graph_robust.cu): the loop edges' residuals and
// their graduated-non-convexity weights with a truncated-least-squares cost (include/tloam_b200.h, "Robust pose graph").
// The weighted Gauss-Newton stages themselves run in libtloam_b200_pg.so (tloam_pg_args::loop_w).
//
// libtloam_b200.so loads that library with dlopen on the first robust optimisation and resolves this symbol; nothing here
// defines a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer is a device pointer,
// the launcher enqueues its work on `stream` of `device`, and nothing synchronises.  The return value is a cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "pose_graph.h"

#ifdef __cplusplus
extern "C" {
#endif

// the device-side GNC state: written by k_pgr_weights, read by the host after every stage
typedef struct tloam_pgr_state {
  double mu;                          // the mu of the last weight update
  double max_rho;                     // max_l rho_l at the first update
  int all_inliers;                    // first update only: max rho <= chi2_threshold (the weights stay 1)
  int binary;                         // every weight exactly 0 or 1
  int inliers, rejected;              // weights == 1, == 0
} tloam_pgr_state;

typedef struct tloam_pgr_args {
  const double* T;                    // 2 x N poses as in tloam_pg_args; the residuals are taken at T[pg_state->cur]
  const tloam_pg_state* pg_state;
  const long long* loop_ij;           // L x (i, j)
  const double* loop_Z;               // L x 16
  unsigned long long N, L;
  double w_loop[6];                   // the diagonal of Omega_loop
  double chi2_threshold, gnc_factor;
  double* rho;                        // L: r^T Omega_loop r, unweighted
  double* w;                          // L: the weights, updated in place
  tloam_pgr_state* state;
  int device;
  cudaStream_t stream;
} tloam_pgr_args;

// k_pgr_residual (one thread per loop edge) -> k_pgr_weights (one block).  first: mu_0 from max rho (or all_inliers), else
// mu <- gnc_factor mu; then the TLS update of every weight.  *launches (host) receives the kernel count.
int tloam_pgr_update(const tloam_pgr_args* a, int first, int* launches);

typedef int (*tloam_pgr_update_fn)(const tloam_pgr_args*, int, int*);

#ifdef __cplusplus
}
#endif
