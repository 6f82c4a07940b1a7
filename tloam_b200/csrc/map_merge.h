// map_merge.h -- the C launchers of libtloam_b200_gmm.so (map_merge.cu): the global map merged into one voxel grid,
// VoxelDownSample of the whole map or of its static rows (include/tloam_b200.h, "Merged global map").
//
// libtloam_b200.so loads that library with dlopen on the first merge and resolves these symbols; nothing here defines a
// kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer is a device pointer unless
// marked, each launcher enqueues its work on `stream` of `device`, and nothing synchronises.  The return value is a
// cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

// what tloam_gmm_bounds leaves for the host (one copy home)
typedef struct tloam_gmm_state {
  unsigned long long lo[3];           // complemented ordered encodings of the selected rows' min (0 = none)
  unsigned long long hi[3];           // ordered encodings of their max (0 = none)
  unsigned long long n_sel;           // selected rows
  unsigned long long n_vox;           // voxels (written by tloam_gmm_sort)
  unsigned nonfinite;                 // a selected row has a NaN or infinite coordinate
} tloam_gmm_state;

typedef struct tloam_gmm_args {
  const double* map;                  // count x 3
  const double* intensity;            // count, or null (no channel)
  const unsigned* through;            // with hits: the removal's counters (static_only), or null (every row)
  const unsigned* hits;
  unsigned min_through;
  unsigned long long count;           // the map's rows (host value, < 2^32)
  // set by the host between tloam_gmm_bounds and tloam_gmm_sort
  double mb[3];                       // min - voxel * 0.5 per axis
  double voxel;
  int bits[3];                        // bits of ix, iy, iz in the key (0 .. 21)
  unsigned long long n_sel;           // selected rows (the state's value)
  void* scratch;                      // tloam_gmm_scratch_bytes(count) bytes
  tloam_gmm_state* state;             // in scratch (tloam_gmm_state_of)
  // tloam_gmm_average
  unsigned long long n_vox;
  double* out_xyz;                    // n_vox x 3
  double* out_intensity;              // n_vox, null without a channel
  int device;
  cudaStream_t stream;
} tloam_gmm_args;

// the scratch of a merge over `count` map rows: two key / row buffers (24 B per row), the radix histograms and the state
size_t tloam_gmm_scratch_bytes(unsigned long long count);
tloam_gmm_state* tloam_gmm_state_of(void* scratch, unsigned long long count);
// clears the state, then k_gmm_bounds: the selected rows' count, bounds and non-finite flag
int tloam_gmm_bounds(const tloam_gmm_args* a, int* launches);
// k_gmm_keys, the stable LSD radix sort (k_gmm_hist -> k_gmm_offsets -> k_gmm_scatter per 8-bit digit), then
// k_gmm_head_count -> k_gmm_head_scatter: the voxel starts and state->n_vox
int tloam_gmm_sort(const tloam_gmm_args* a, int* launches);
// k_gmm_average: voxel j's averages at position j
int tloam_gmm_average(const tloam_gmm_args* a, int* launches);

typedef size_t (*tloam_gmm_scratch_bytes_fn)(unsigned long long);
typedef tloam_gmm_state* (*tloam_gmm_state_of_fn)(void*, unsigned long long);
typedef int (*tloam_gmm_launch_fn)(const tloam_gmm_args*, int*);

#ifdef __cplusplus
}
#endif
