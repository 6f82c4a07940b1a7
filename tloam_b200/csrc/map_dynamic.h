// map_dynamic.h -- the C launchers of libtloam_b200_gmd.so (map_dynamic.cu): dynamic-point removal for the global map,
// free-space votes from every appended scan's range image (include/tloam_b200.h, "Dynamic-point removal").
//
// libtloam_b200.so loads that library with dlopen when removal is enabled and resolves these symbols; nothing here defines
// a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer is a device pointer unless
// marked, each launcher enqueues its work on `stream` of `device`, and nothing synchronises.  The return value is a
// cudaError_t.  Poses are column-major 4 x 4.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct tloam_gmd_params {
  int n_rows, n_cols;                 // the range image
  int wr, wc;                         // the window's half extents (rows clipped, columns wrapped)
  double margin_abs, margin_rel;
  double min_range, max_range;
  const double* row_bounds;           // n_rows + 1: b_k
  const double* col_bounds;           // (n_cols - 1) x 2: (cos, sin) of the sector boundaries
} tloam_gmd_params;

typedef struct tloam_gmd_vote_args {
  tloam_gmd_params p;
  const double* scan;                 // n x 3: the append's sensor-frame rows, read before the append transforms them
  unsigned n;
  const double* pose;                 // 16: the pose the append places its block at
  const double* map;                  // the map, rows [0, *count) voted on
  const unsigned long long* count;    // the map's row count before the append (device)
  unsigned* through;
  unsigned* hits;
  unsigned long long* image;          // n_rows x n_cols: ordered bits of the minimum r, +inf = empty
  double* window;                     // n_rows x n_cols: the window minimum, NaN = unknown
  int device;
  cudaStream_t stream;
} tloam_gmd_vote_args;

// k_gmd_clear -> k_gmd_bin -> k_gmd_window -> k_gmd_vote.  *launches (host) receives the kernel count.
int tloam_gmd_vote(const tloam_gmd_vote_args* a, int* launches);

typedef struct tloam_gmd_static_args {
  const double* map;                  // count x 3
  const double* intensity;            // count, or null
  const unsigned* through;
  const unsigned* hits;
  unsigned long long count;           // the map's rows (host value)
  unsigned min_through;
  unsigned* block_counts;             // tloam_gmd_static_blocks(count) entries
  unsigned long long* total;          // 1: the static rows
  double* out_xyz;                    // count x 3
  double* out_intensity;              // count, or null
  int device;
  cudaStream_t stream;
} tloam_gmd_static_args;

// the blocks of the compaction (at most 1024)
unsigned tloam_gmd_static_blocks(unsigned long long count);
// k_gmd_count -> k_gmd_scatter: the non-dynamic rows in row order.  *launches (host) receives the kernel count.
int tloam_gmd_static(const tloam_gmd_static_args* a, int* launches);

typedef int (*tloam_gmd_vote_fn)(const tloam_gmd_vote_args*, int*);
typedef unsigned (*tloam_gmd_static_blocks_fn)(unsigned long long);
typedef int (*tloam_gmd_static_fn)(const tloam_gmd_static_args*, int*);

#ifdef __cplusplus
}
#endif
