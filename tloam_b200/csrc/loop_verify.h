// loop_verify.h -- the C launchers of libtloam_b200_loopv.so (loop_verify.cu): the keyframe store's commit and the
// scan-to-scan ICP that verifies a loop candidate (include/tloam_b200.h, "Loop verification").
//
// libtloam_b200.so loads that library with dlopen on the first verification call and resolves these symbols; nothing here
// defines a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer is a device pointer
// unless marked, each launcher enqueues its work on `stream` of `device`, and nothing synchronises.  The return value is a
// cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TLOAM_LV_THREADS 256          // queries per block of the correspondence search
#define TLOAM_LV_SUMS 32              // per-block partials: H (21, packed upper triangle), g (6), inliers, sum d2 of the
                                      // inliers, sum d2 of every query, two unused

// the device-side state of one verification: the current T (R row-major, t), the radius, the iteration count and the
// termination; then the result of the final pass
typedef struct tloam_lv_state {
  double R[9], t[3];
  double r;
  int iter, done, term, pad;
  double fitness, rmse;
  unsigned long long inliers;
} tloam_lv_state;

// the nearest candidate row of a query row over one slice of the candidate keyframe
typedef struct tloam_lv_best {
  double d2;
  long long index;
} tloam_lv_best;

typedef struct tloam_lv_args {
  const double* pts;                  // the keyframe store (FP64 xyz)
  unsigned long long q0, nq;          // the query keyframe Q: rows q0 .. q0 + nq - 1
  unsigned long long m0, nm;          // the candidate keyframe M
  double corr_dist_coarse, corr_dist_fine, eps_translation, eps_rotation;
  int max_iterations;
  unsigned splits;                    // M is searched in this many slices (grid y)
  tloam_lv_state* state;              // initialised by the caller (T = guess, r = coarse, the rest 0)
  tloam_lv_best* part;                // splits x nq
  double* sums;                       // ceil(nq / TLOAM_LV_THREADS) x TLOAM_LV_SUMS
  int* match_index;                   // (max_iterations + 1) x nq: pass k's nearest candidate row (-1: none)
  double* match_d2;                   // the same passes' d2
  int device;
  cudaStream_t stream;
} tloam_lv_args;

// max_iterations rounds of k_lv_match -> k_lv_reduce -> k_lv_step (a round after termination does nothing), then the final
// pass at r = corr_dist_fine (k_lv_match -> k_lv_reduce -> k_lv_final).  *launches (host) receives the kernel count.
int tloam_lv_verify(const tloam_lv_args* a, int* launches);

// k_lv_commit: closes keyframe slot *frames: offsets[*frames + 1] = *count + (the frame's voxels unless it was refused or
// would pass cap), *count and *frames advance.  A frame past cap gets an empty slot and sets bit 2 of *flags.  Every call
// advances by exactly one slot.
int tloam_lv_commit(const unsigned* n_vox, const unsigned* refused, unsigned long long* count, unsigned long long* frames,
                    unsigned* flags, unsigned long long* offsets, unsigned long long cap, int device, cudaStream_t stream);

typedef int (*tloam_lv_verify_fn)(const tloam_lv_args*, int*);
typedef int (*tloam_lv_commit_fn)(const unsigned*, const unsigned*, unsigned long long*, unsigned long long*, unsigned*,
                                  unsigned long long*, unsigned long long, int, cudaStream_t);

#ifdef __cplusplus
}
#endif
