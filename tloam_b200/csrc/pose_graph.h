// pose_graph.h -- the C launcher of libtloam_b200_pg.so (pose_graph.cu): Gauss-Newton over a pose graph of odometry and
// verified loop edges (include/tloam_b200.h, "Pose graph").
//
// libtloam_b200.so loads that library with dlopen on the first pose-graph call and resolves this symbol; nothing here
// defines a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer is a device pointer,
// the launcher enqueues its work on `stream` of `device`, and nothing synchronises.  The return value is a cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TLOAM_PG_EDGE 44              // per edge: A = Ad(T_j^-1) (36, row-major), r (6), r^T Omega r, unused
#define TLOAM_PG_CHAIN 108            // per node k >= 1: W_k (36), S_k^-1 (36), P_{k+1} (36), all row-major

// the device-side state of one optimisation.  T[cur] holds the accepted poses; a round writes its candidate to T[cur ^ 1]
typedef struct tloam_pg_state {
  int cur, done, term, iter;
  double cost, initial_cost;          // at T[cur]; at the odometry poses
  double step_t, step_r;              // the last step's largest |upsilon| / |omega| component
} tloam_pg_state;

typedef struct tloam_pg_args {
  const double* O;                    // N odometry poses, column-major 4 x 4
  double* T;                          // 2 x N poses, column-major 4 x 4 (buffer b at T + 16 N b)
  const long long* loop_ij;           // L x (candidate i, query j)
  const double* loop_Z;               // L x 16: Z = T_i^-1 T_j measured, column-major
  const double* loop_w;               // L: the loop edges' weights in [0, 1], read by k_pg_linearize only; null: all 1
  unsigned long long N, L;
  double w_odom[6], w_loop[6];        // the diagonals of Omega_odom and Omega_loop, (upsilon, omega) order
  double eps_translation, eps_rotation;
  int max_iterations;
  unsigned chol_blocks;               // k_pg_dense_chol's cooperative grid
  tloam_pg_state* state;              // initialised by the caller: T[cur] = the start poses (O for a plain run), the rest 0
  double* edge;                       // (N - 1 + L) x TLOAM_PG_EDGE; odometry edge k - 1 is (k - 1, k)
  double* chain;                      // N x TLOAM_PG_CHAIN (slot 0 unused)
  double* b;                          // N x 6: -g (slot 0 unused)
  double* Y;                          // 6 (N - 1) x (6 L + 1), row-major: M^-1 [B^T | b]
  double* S;                          // 6 L x (6 L + 1), row-major: [Omega_loop^-1 + B Y | B u], factored in place
  double* z;                          // 6 L: S^-1 B u
  double* norms;                      // N x 2: per node max |upsilon|, max |omega| of the step
  int device;
  cudaStream_t stream;
} tloam_pg_args;

// k_pg_linearize -> k_pg_accept at the odometry poses, then max_iterations rounds of k_pg_chain_factor -> k_pg_rhs ->
// k_pg_chain_solve -> k_pg_capacitance -> k_pg_dense_chol -> k_pg_update -> k_pg_linearize -> k_pg_accept (a round after
// termination does nothing).  *launches (host) receives the kernel count.
int tloam_pg_optimize(const tloam_pg_args* a, int* launches);
// the cooperative grid k_pg_dense_chol may use on `device` (co-resident blocks)
int tloam_pg_chol_blocks(int device, unsigned* blocks);

typedef int (*tloam_pg_optimize_fn)(const tloam_pg_args*, int*);
typedef int (*tloam_pg_chol_blocks_fn)(int, unsigned*);

#ifdef __cplusplus
}
#endif
