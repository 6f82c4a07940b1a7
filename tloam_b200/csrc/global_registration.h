// global_registration.h -- the C launchers of libtloam_b200_greg.so (global_registration.cu): registration of two clouds
// with no initial guess by FPFH features, mutual matches, a RANSAC search and a truncated-least-squares refinement
// (include/tloam_b200.h, "Global registration").
//
// libtloam_b200.so loads that library with dlopen on tloam_b200_global_registration_enable and resolves these symbols;
// nothing here defines a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Each side's grid
// index and normals come from tloam_loc_index (libtloam_b200_loc.so) in buffers of this feature.  Every pointer is a device
// pointer, the launchers enqueue their work on `stream` of `device`, and nothing synchronises.  The return value is a
// cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "localize.h"

#ifdef __cplusplus
extern "C" {
#endif

#define TLOAM_GR_BINS 33              // FPFH: 11 bins each of alpha, phi and theta
#define TLOAM_GR_THREADS 256          // hypotheses per block of k_gr_hyp, threads of k_gr_best and k_gr_refine

// one cloud: its keypoints, its index and normals (tloam_loc_index), and what the features write
typedef struct tloam_gr_side {
  tloam_loc_grid grid;
  const double* xyz;                  // n x 3 keypoints, row order
  double* normal;                     // n x 3, oriented in place by k_gr_orient
  const unsigned char* valid;         // n
  unsigned long long n;
  int* spfh;                          // n x 33 integer counts
  int* pairs;                         // n: the pairs behind the counts
  double* feature;                    // n x 33 (0 where the row has no feature)
  unsigned char* has_feature;         // n
  int* nn;                            // n: the nearest feature row of the other side (-1: none)
  unsigned long long* n_features;     // the rows with a feature (counted by k_gr_fpfh; zero on entry)
} tloam_gr_side;

// the run's device-side result
typedef struct tloam_gr_state {
  unsigned long long n_corr;          // mutual pairs (k_gr_mutual)
  int n_valid, best, best_inliers;    // valid hypotheses, the best one and its inliers (k_gr_best; best -1: none)
  int inliers, iterations, term;      // k_gr_refine
  int pad;
  double R[9], t[3];                  // the best hypothesis's T, then the refined T (R row-major)
  double rmse;
  unsigned long long fit_count;       // source keypoints with a target keypoint within tau under T (k_gr_fitness)
  unsigned long long n_features[2];   // source, target
} tloam_gr_state;

typedef struct tloam_gr_args {
  tloam_gr_side src, tgt;
  double feature_radius, tau;
  double theta_cs[20];                // (cos, sin) of the theta bin boundaries -pi + 2 pi k / 11, k = 1 .. 10
  int n_hypotheses;
  unsigned long long seed;
  double edge_similarity, min_triangle_area;
  int max_refine_iterations;
  int* corr;                          // n_src x 2: the mutual pairs (source row, target row), in source order
  int* hyp_inliers;                   // n_hypotheses: inlier count (-1: rejected)
  unsigned char* in_set;              // 2 x n_src: the refinement's current and next inlier sets
  tloam_gr_state* state;
  int device;
  cudaStream_t stream;
} tloam_gr_args;

// with both sides indexed: *state cleared, then per side k_gr_orient, k_gr_spfh, k_gr_fpfh; k_gr_match both ways,
// k_gr_mutual, k_gr_hyp, k_gr_best, k_gr_refine, k_gr_fitness
int tloam_gr_run(const tloam_gr_args* a, int* launches);

typedef int (*tloam_gr_run_fn)(const tloam_gr_args*, int*);

#ifdef __cplusplus
}
#endif
