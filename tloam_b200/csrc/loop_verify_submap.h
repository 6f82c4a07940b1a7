// loop_verify_submap.h -- the C launcher of libtloam_b200_loopvs.so (loop_verify_submap.cu): the verification of a loop
// candidate against the submap of the keyframes around it, with a point-to-plane residual (include/tloam_b200.h, "Loop
// verification against a submap").
//
// libtloam_b200.so loads that library with dlopen on the first submap verification call and resolves this symbol; nothing
// here defines a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer is a device
// pointer unless marked, the launcher enqueues its work on `stream` of `device`, and nothing synchronises.  The return
// value is a cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "loop_verify.h"

#ifdef __cplusplus
extern "C" {
#endif

#define TLOAM_LVS_THREADS 256         // queries per block of the correspondence search
#define TLOAM_LVS_NORMAL_THREADS 128  // target rows per block of the normal estimation
#define TLOAM_LVS_SUMS 32             // per-block partials: H (21, packed upper triangle), g (6), contributing rows, sum e^2
                                      // over them, sum d2 of every query, two unused
#define TLOAM_LVS_MAX_HALF_WINDOW 50

typedef struct tloam_lvs_args {
  const double* pts;                  // the keyframe store (FP64 xyz)
  const unsigned long long* offsets;  // the keyframe table: keyframe f = rows [offsets[f], offsets[f + 1])
  unsigned long long lo, hi;          // the window's frames
  unsigned long long candidate;
  unsigned long long q0, nq;          // the query keyframe Q: rows q0 .. q0 + nq - 1
  int query_in_window;                // Q's rows lie inside the window's rows of the store and are left out
  unsigned long long base;            // offsets[lo] (known to the host)
  unsigned long long nm;              // target rows
  const double* poses;                // pose of frame lo + w at poses + 16 w (column-major 4 x 4)
  double* A;                          // (hi - lo + 1) x 16: A_w = O_c^-1 O_(lo + w)
  double* target;                     // nm x 3
  double* normal;                     // nm x 3
  unsigned char* valid;               // nm
  int* neighbours;                    // nm
  double normal_radius, max_planarity;
  int min_normal_neighbours;
  double corr_dist_coarse, corr_dist_fine, eps_translation, eps_rotation;
  int max_iterations;
  unsigned splits;                    // the target is searched in this many slices (grid y)
  tloam_lv_state* state;              // initialised by the caller (T = guess, r = coarse, the rest 0)
  tloam_lv_best* part;                // splits x nq
  double* sums;                       // ceil(nq / TLOAM_LVS_THREADS) x TLOAM_LVS_SUMS
  int* match_index;                   // (max_iterations + 1) x nq: pass k's nearest target row (-1: none)
  double* match_d2;                   // the same passes' d2
  int device;
  cudaStream_t stream;
} tloam_lvs_args;

// k_lvs_poses -> k_lvs_assemble -> k_lvs_normals, then max_iterations rounds of k_lvs_match -> k_lvs_reduce -> k_lvs_step (a
// round after termination does nothing) and the final pass at r = corr_dist_fine (k_lvs_match -> k_lvs_reduce ->
// k_lvs_final).  *launches (host) receives the kernel count.
int tloam_lvs_verify(const tloam_lvs_args* a, int* launches);

typedef int (*tloam_lvs_verify_fn)(const tloam_lvs_args*, int*);

#ifdef __cplusplus
}
#endif
