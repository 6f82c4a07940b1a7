// occupancy.h -- the C launchers of libtloam_b200_occ.so (occupancy.cu): the 2D occupancy grid of the global map
// (include/tloam_b200.h, "Occupancy grid").
//
// libtloam_b200.so loads that library with dlopen on tloam_b200_occupancy_enable and resolves these symbols; nothing here
// defines a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer is a device pointer
// unless marked, each launcher enqueues its work on `stream` of `device`, and nothing synchronises.  The return value is a
// cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TLOAM_OCC_SLOT 4              // doubles per sector of a frame's scan: the obstacle's x, y, z, then the floor's range

typedef struct tloam_occ_params {
  int n_cols;                         // sectors
  double z_lo, z_hi;                  // the obstacle band (sensor frame)
  double min_range, max_range;
  const double* dirs;                 // 2 (n_cols - 1): Scan Context's sector boundaries (cos, sin of 2 pi k / n_cols)
} tloam_occ_params;

// the 2D scan of one append: k_occ_clear -> k_occ_bin -> k_occ_pick -> k_occ_final, into slot *frames (the device frame
// count the append's k_gmap_commit advances, so a refused append leaves its slot to the next one)
typedef struct tloam_occ_capture_args {
  tloam_occ_params p;
  const double* scan;                 // n x 3, sensor frame
  unsigned n;
  const double* pose;                 // 16: the pose the block is placed at (column-major)
  const unsigned long long* frames;   // 1: the slot
  unsigned long long cap;             // slots
  double* scans;                      // cap x n_cols x TLOAM_OCC_SLOT
  double* poses;                      // cap x 16
  int device;
  cudaStream_t stream;
} tloam_occ_capture_args;

int tloam_occ_capture(const tloam_occ_capture_args* a, int* launches);

typedef struct tloam_occ_build_args {
  tloam_occ_params p;
  double free_margin, resolution;
  double W;                           // the window half-width: max_range + max(|z_lo|, |z_hi|) + resolution
  const double* scans;                // n_frames x n_cols x TLOAM_OCC_SLOT
  const double* poses;                // n_frames x 16: the build poses
  unsigned long long n_frames;        // > 0
  double* extent;                     // 4: min t_x, min t_y, max t_x, max t_y (tloam_occ_extent)
  // set by the host between tloam_occ_extent and tloam_occ_rasterise
  double origin_x, origin_y;
  unsigned width, height;
  int nwin;                           // candidate cells per axis of a frame's window (a superset of the |c - t| <= W test)
  unsigned* occupied;                 // width x height, row-major from (0, 0), i along x
  unsigned* free_count;
  signed char* cells;
  unsigned long long* dropped;        // 1
  int device;
  cudaStream_t stream;
} tloam_occ_build_args;

// k_occ_extent: the build poses' translation bounds
int tloam_occ_extent(const tloam_occ_build_args* a, int* launches);
// clears the counters, then k_occ_free (one thread per frame and window cell), k_occ_hits (one per frame and sector) and
// k_occ_value (one per cell)
int tloam_occ_rasterise(const tloam_occ_build_args* a, int* launches);

typedef int (*tloam_occ_capture_fn)(const tloam_occ_capture_args*, int*);
typedef int (*tloam_occ_build_fn)(const tloam_occ_build_args*, int*);

#ifdef __cplusplus
}
#endif
