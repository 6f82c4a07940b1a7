// unpack_scan.h -- the C launcher of libtloam_b200_unpack.so (unpack_scan.cu): a sensor's packed float32 records to the
// FP64 arrays the raw-scan chain and the global map read.
//
// libtloam_b200.so loads that library with dlopen on the first packed-scan call and resolves this symbol; nothing here
// defines a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer is a device pointer,
// the launch is enqueued on `stream` of `device`, and nothing synchronises.  The return value is a cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

// bytes: n records of point_step bytes (little-endian), in a buffer of at least round_up(n * point_step, 16) bytes starting
// 16-byte aligned.  off[0..2]: the FLOAT32 x / y / z fields, off[3]: intensity or -1; every field lies inside the record
// (0 <= off, off + 4 <= point_step).  xyz (n x 3 FP64) and, when off[3] >= 0 and intensity is not null, intensity (n FP64)
// receive (double)float of every record.
int tloam_unpack_scan(const unsigned char* bytes, unsigned long long n, unsigned long long point_step, const int off[4], double* xyz,
                      double* intensity, int device, cudaStream_t stream);

typedef int (*tloam_unpack_scan_fn)(const unsigned char*, unsigned long long, unsigned long long, const int*, double*, double*, int,
                                    cudaStream_t);

#ifdef __cplusplus
}
#endif
