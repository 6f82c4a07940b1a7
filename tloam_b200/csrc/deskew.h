// deskew.h -- the C launchers of libtloam_b200_deskew.so (deskew.cu): the motion correction of a raw scan from per-point
// times and the constant-velocity increment of the handle's pose history.
//
// libtloam_b200.so loads that library with dlopen on the first timed call and resolves these symbols; nothing here defines
// a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer in tloam_deskew_args is a
// device pointer, each launcher enqueues one kernel on `stream` of `device`, and nothing synchronises.  The three run in
// the order motion, tend, apply on the same args.  The return value is a cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct tloam_deskew_args {
  const double* last_pose;        // 4 x 4 column-major: FrameState::last_pose / curr_pose
  const double* curr_pose;
  const double* time;             // n FP64 times, or null: read from the packed records
  const unsigned char* records;   // n records of point_step bytes (little-endian), the time field at `offset`
  unsigned long long point_step;
  int offset, datatype;           // sensor_msgs/PointField: 6 UINT32, 7 FLOAT32, 8 FLOAT64
  double unit;                    // a record's time is its field's value times unit
  unsigned long long n;
  double period;                  // the frame period, in the unit of the times
  const double* xyz;              // n x 3 FP64, the raw scan
  double* out;                    // n x 3 FP64, the corrected scan
  double* scratch;                // TLOAM_DESKEW_SCRATCH_DOUBLES: xi (6), then the encoded t_end
  int device;
  cudaStream_t stream;
} tloam_deskew_args;

#define TLOAM_DESKEW_SCRATCH_DOUBLES 8

// k_deskew_motion: xi = log(last^-1 . curr) and t_end cleared
int tloam_deskew_motion(const tloam_deskew_args* a);
// k_deskew_tend: t_end = the largest finite time
int tloam_deskew_tend(const tloam_deskew_args* a);
// k_deskew: out_i = exp(s_i . xi) . xyz_i, s_i = (t_i - t_end) / period (0 for a non-finite t_i or no finite time)
int tloam_deskew_apply(const tloam_deskew_args* a);

typedef int (*tloam_deskew_fn)(const tloam_deskew_args*);

#ifdef __cplusplus
}
#endif
