// map_correct.h -- the C launchers of libtloam_b200_gmc.so (map_correct.cu): the global map's per-frame pose tables and
// the loop-closure correction that moves every frame's block to its pose-graph pose (include/tloam_b200.h, "Loop-corrected
// global map").
//
// libtloam_b200.so loads that library with dlopen when tracking is enabled and resolves these symbols; nothing here defines
// a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer is a device pointer unless
// marked, each launcher enqueues its work on `stream` of `device`, and nothing synchronises.  The return value is a
// cudaError_t.  Poses are column-major 4 x 4.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct tloam_gmc_mat {
  double m[16];
} tloam_gmc_mat;

// k_gmc_pose (one warp): O[f] = src, P[f] = M src (M null, host: a copy of src) at f = *frames, the slot the append is
// about to commit (a refused frame's slot is overwritten by the next append); pose = P[f], the pose k_gmap_transform
// reads.  src may alias pose.  Nothing is written to the tables when f >= cap.
int tloam_gmc_pose(const double* src, double* pose, double* O, double* P, const unsigned long long* frames,
                   unsigned long long cap, const tloam_gmc_mat* M, int device, cudaStream_t stream);

typedef struct tloam_gmc_args {
  const long long* node;              // frames: the pose-graph node of every map frame, -1: none
  const double* node_O;               // the nodes' odometry poses
  const double* node_T;               // the last optimisation's poses of nodes [0, n_opt) (unused when n_opt is 0)
  unsigned long long n_opt;
  tloam_gmc_mat delta_new;            // Delta of nodes >= n_opt: the map -> odom correction (host value)
  const double* O;                    // frames x 16: the frames' odometry poses
  double* P;                          // frames x 16: the poses the blocks are expressed at, updated in place
  double* M;                          // frames x 16 scratch: C_f P_f^-1 of every moved frame
  unsigned* moved;                    // frames scratch
  unsigned long long frames, points;
  const unsigned long long* offsets;  // frames + 1: the map's frame table
  double* map;                        // points x 3
  int device;
  cudaStream_t stream;
} tloam_gmc_args;

// k_gmc_frames (one thread per frame) -> k_gmc_points (one thread per map point).  *launches (host) receives the kernel
// count.
int tloam_gmc_correct(const tloam_gmc_args* a, int* launches);

typedef int (*tloam_gmc_pose_fn)(const double*, double*, double*, double*, const unsigned long long*, unsigned long long,
                                 const tloam_gmc_mat*, int, cudaStream_t);
typedef int (*tloam_gmc_correct_fn)(const tloam_gmc_args*, int*);

#ifdef __cplusplus
}
#endif
