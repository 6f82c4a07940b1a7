// map_update.h -- the C launchers of libtloam_b200_mapu.so (map_update.cu): updating a prior map from localized frames
// (include/tloam_b200.h, "Updating a prior map").
//
// libtloam_b200.so loads that library with dlopen on tloam_b200_map_update_enable and resolves these symbols; nothing here
// defines a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  The free-space votes are
// tloam_gmd_vote of libtloam_b200_gmd.so and the prior rows' part of the build tloam_gmd_static, called by the host.  Every
// pointer is a device pointer unless marked, each launcher enqueues its work on `stream` of `device`, and nothing
// synchronises.  The return value is a cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "localize.h"
#include "map_merge.h"

#ifdef __cplusplus
extern "C" {
#endif

#define TLOAM_MU_MAX_BLOCKS 1024      // blocks of an order-preserving compaction

typedef struct tloam_mu_add_args {
  tloam_loc_grid grid;                // the prior map's index
  const double* query;                // nq x 3: the localization's query (sensor frame)
  unsigned long long nq;
  const tloam_loc_state* state;       // the localization's final state: p = T q by loc_apply
  double radius;                      // novel_radius
  unsigned long long n_prior;         // the prior map's rows
  double* pose;                       // 16: T, column-major (written by k_mu_pose for the votes)
  unsigned long long* prior_count;    // 1: n_prior (written by k_mu_pose for the votes)
  unsigned char* flag;                // nq: the row is new
  double* p;                          // nq x 3: T q
  unsigned* block_counts;             // TLOAM_MU_MAX_BLOCKS
  unsigned long long* base;           // 1: the additions' count before the append
  unsigned long long* count;          // 1: the additions' count (in and out)
  double* add_xyz;                    // the additions: xyz, frame number, counters
  unsigned* add_frame;
  unsigned* add_through;
  unsigned* add_hits;
  unsigned frame;                     // this add's frame number
  int device;
  cudaStream_t stream;
} tloam_mu_add_args;

// k_mu_pose: T column-major from the state, and n_prior, for the two tloam_gmd_vote calls
int tloam_mu_pose(const tloam_mu_add_args* a, int* launches);
// k_mu_novel -> k_mu_count -> k_mu_scatter: the query rows with no prior row within radius, as T q, appended to the
// additions in query order with this add's frame number and counters (0, 0)
int tloam_mu_novel(const tloam_mu_add_args* a, int* launches);

typedef struct tloam_mu_build_args {
  const double* add_xyz;              // n_add x 3
  const unsigned* add_frame;
  const unsigned* add_through;
  const unsigned* add_hits;
  unsigned long long n_add;           // host value, < 2^32
  unsigned min_through;
  unsigned min_frames;
  // set by the host between tloam_mu_bounds and tloam_mu_sort (the merge's rule)
  double mb[3];
  double voxel;
  int bits[3];
  unsigned long long n_sel;           // the kept additions (the state's value)
  void* scratch;                      // tloam_mu_scratch_bytes(n_add)
  tloam_gmm_state* state;             // in scratch (tloam_mu_state_of)
  // tloam_mu_average
  unsigned long long n_vox;
  unsigned long long* count;          // 1: in, the rows already in out_xyz (the kept prior rows); out, the cloud's rows
  double* out_xyz;                    // the built cloud: the kept prior rows, then the supported voxels
  int device;
  cudaStream_t stream;
} tloam_mu_build_args;

size_t tloam_mu_scratch_bytes(unsigned long long n_add);
tloam_gmm_state* tloam_mu_state_of(void* scratch, unsigned long long n_add);
// clears the state, then k_mu_bounds: the kept additions' count, bounds and non-finite flag
int tloam_mu_bounds(const tloam_mu_build_args* a, int* launches);
// k_mu_keys, the shared stable radix sort, the heads: the voxel starts and state->n_vox
int tloam_mu_sort(const tloam_mu_build_args* a, int* launches);
// k_mu_average (averages, distinct frames, the min_frames test), then k_mu_count -> k_mu_scatter of the supported voxels
// in ascending key order behind *count rows
int tloam_mu_average(const tloam_mu_build_args* a, int* launches);

typedef int (*tloam_mu_add_fn)(const tloam_mu_add_args*, int*);
typedef size_t (*tloam_mu_scratch_bytes_fn)(unsigned long long);
typedef tloam_gmm_state* (*tloam_mu_state_of_fn)(void*, unsigned long long);
typedef int (*tloam_mu_build_fn)(const tloam_mu_build_args*, int*);

#ifdef __cplusplus
}
#endif
