// relocalize.h -- the C launcher of libtloam_b200_reloc.so (relocalize.cu): relocalization in a prior map, a Scan Context
// search over a saved session's places and the best candidates refined by the localization's ICP in one batch
// (include/tloam_b200.h, "Relocalization in a prior map").
//
// libtloam_b200.so loads that library with dlopen on tloam_b200_relocalize_enable and resolves the symbol; nothing here
// defines a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer is a device pointer,
// the launcher enqueues its work on `stream` of `device`, and nothing synchronises.  The return value is a cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "localize.h"

#ifdef __cplusplus
extern "C" {
#endif

#define TLOAM_RL_MAX_K 64             // top_k at most

// the candidates and the selection, written on the device
typedef struct tloam_rl_top {
  int n;                              // hypotheses (<= top_k)
  int winner;                         // -1 without hypotheses
  int ambiguous, accepted;
  long long place[TLOAM_RL_MAX_K];
  long long shift[TLOAM_RL_MAX_K];
  double distance[TLOAM_RL_MAX_K];
} tloam_rl_top;

typedef struct tloam_rl_args {
  tloam_loc_args loc;                 // the map, its index, the query, O_now, the memory and the ICP's schedule (its
                                      // state, sums and match records are unused: each hypothesis has its own below)
  const double* qdesc;                // the query's descriptor slot (TLOAM_SC_SLOT_DOUBLES)
  const double* places;               // n_places slots
  const double* poses;                // n_places x 16, column-major
  unsigned long long n_places;
  int n_ring, n_sector;
  const double* dirs;                 // (n_sector - 1) x 2: the sector boundaries' (cos, sin)
  double* place_distance;             // n_places: each place's best distance
  long long* place_shift;             // n_places: and its shift
  int top_k;
  double max_distance, distinct_translation, cos_distinct_rotation, ambiguity_ratio;
  tloam_loc_state* states;            // top_k runs (set by the host: radius, termination, done)
  double* sums;                       // top_k x ceil(nq / TLOAM_LOC_THREADS) x TLOAM_LOC_SUMS
  int* match_index;                   // top_k x (max_iterations + 1) x nq
  double* match_d2;
  tloam_rl_top* top;
  int device;
  cudaStream_t stream;
} tloam_rl_args;

// k_rl_search (every place's best distance and shift), k_rl_topk, k_rl_guess, max_iterations rounds of k_rl_match ->
// k_rl_reduce -> k_rl_step over every hypothesis, the final pass (k_rl_match -> k_rl_reduce -> k_rl_final), then k_rl_select
int tloam_rl_run(const tloam_rl_args* a, int* launches);

typedef int (*tloam_rl_run_fn)(const tloam_rl_args*, int*);

#ifdef __cplusplus
}
#endif
