// distance.h -- the C launchers of libtloam_b200_dist.so (distance.cu): the distance field and the inflated costmap of an
// occupancy grid (include/tloam_b200.h, "Distance field and costmap").
//
// libtloam_b200.so loads that library with dlopen on the first distance call and resolves these symbols; nothing here
// defines a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer is a device pointer,
// each launcher enqueues its work on `stream` of `device`, and nothing synchronises.  The return value is a cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TLOAM_DIST_BAND 64            // rows per band of the column pass
#define TLOAM_DIST_INF 0xFFFFFFFFu    // no cell of the other class

typedef struct tloam_dist_build_args {
  const signed char* cells;           // width x height, row-major from (0, 0), i along x: nav_msgs/OccupancyGrid's values
  unsigned width, height;             // >= 1 each, (width - 1)^2 + (height - 1)^2 < 2^32 - 1
  double resolution;
  unsigned* bands;                    // width x ceil(height / TLOAM_DIST_BAND) x 4: per column and band, the first and last
                                      // obstacle row and the first and last other row (TLOAM_DIST_INF: none)
  unsigned* g;                        // width x height: the column distance to the nearest cell of the other class
  unsigned short* stack;              // width x height x 2: the row pass's two envelopes (obstacle and other sources)
  unsigned* sq;                       // width x height: the squared distance in cells
  float* sd;                          // width x height: the signed distance in m
  const unsigned char* table;         // r2 + 1: the cost c of a non-obstacle cell by sq
  unsigned r2;                        // R_c^2
  unsigned char* costs;               // width x height
  signed char* values;                // width x height
  unsigned long long* obstacles;      // 1
  int device;
  cudaStream_t stream;
} tloam_dist_build_args;

// k_dist_bands (one thread per column and band), k_dist_cols (the same: the column distance g), k_dist_rows (one thread
// per row: the two lower envelopes of g^2 + (i - k)^2, then sq) and k_dist_cost (one per cell: sd, cost, value, and the
// obstacle count)
int tloam_dist_build(const tloam_dist_build_args* a, int* launches);

typedef struct tloam_dist_query_args {
  const float* sd;                    // width x height
  unsigned width, height;
  double origin_x, origin_y, resolution;
  int finite;                         // 0: the field holds an infinite value, and every point gives NaN
  const double* xy;                   // n x 2
  unsigned long long n;
  double* distance;                   // n
  double* gradient;                   // n x 2
  int device;
  cudaStream_t stream;
} tloam_dist_query_args;

// k_dist_query: one thread per point
int tloam_dist_query(const tloam_dist_query_args* a, int* launches);

typedef int (*tloam_dist_build_fn)(const tloam_dist_build_args*, int*);
typedef int (*tloam_dist_query_fn)(const tloam_dist_query_args*, int*);

#ifdef __cplusplus
}
#endif
