// unpack_scan.cu -- libtloam_b200_unpack.so: a sensor's packed float32 records to FP64 AoS xyz and an FP64 intensity array
// (hand-written CUDA for sm_90a).  The device form of the reference's RosToOpen3d (ref: src/open3d/open3d_to_ros.cpp:344-374)
// and readVelodyneToO3d (include/tloam/models/io/read_file.hpp:307-327), which copy every float into a double on the host.
//
// Records are point_step bytes with no alignment guarantee (velodyne_pointcloud's XYZIRT: 22 bytes, record i's x at byte
// 22 i), so a field cannot be loaded as a float from global memory.  k_unpack_scan instead gives each block a run of
// consecutive records, stages the bytes they span in shared memory with aligned 16-byte loads, and lets each thread assemble
// its record's fields from those bytes.  The staging window is a fixed kUnpackWindow (+ 16) bytes: a block whose records
// span more (only possible when point_step exceeds the window) walks its span window by window, and every field is taken
// from the window its first byte lies in -- its last byte is then at most 3 bytes past that window, inside the 16 staged
// beyond it.  One code path for every point_step and field offset.
//
// (double)float is exact: every float, subnormals included, is a double (the build has no fast-math flags, so nothing
// flushes to zero).  A NaN stays a NaN; its payload is not specified.
//
// A separate library so that the kernels of libtloam_b200.so keep their SASS.
#include <cuda_runtime.h>

#include "unpack_scan.h"

namespace tloam {

constexpr unsigned kUnpackThreads = 256;
constexpr unsigned kUnpackWindow = 16384;                   // bytes staged per step (+ 16)
constexpr unsigned kUnpackMaxRecords = 1024;                // records per block

__device__ __forceinline__ unsigned long long unpack_ceil_div(long long a, unsigned long long b) {   // ceil(a / b), 0 for a <= 0
  return a <= 0 ? 0ull : ((unsigned long long)a + b - 1ull) / b;
}

__global__ void __launch_bounds__(kUnpackThreads) k_unpack_scan(const unsigned char* __restrict__ bytes, unsigned long long n,
                                                                unsigned long long ps, unsigned long long alloc, int4 off, int nf,
                                                                int lo, int hi, unsigned long long per_block, double* __restrict__ xyz,
                                                                double* __restrict__ inten) {
  __shared__ uint4 s[kUnpackWindow / 16 + 1];
  const unsigned char* sb = reinterpret_cast<const unsigned char*>(s);
  const unsigned long long r0 = blockIdx.x * per_block, r1 = r0 + per_block < n ? r0 + per_block : n;
  const unsigned long long b0 = r0 * ps + (unsigned)lo, b1 = (r1 - 1ull) * ps + (unsigned)hi;   // bytes the fields span
  const int f[4] = {off.x, off.y, off.z, off.w};
  for (unsigned long long base = b0 & ~15ull; base < b1; base += kUnpackWindow) {
    __syncthreads();                                        // the previous window has been read
    for (unsigned q = threadIdx.x; q < kUnpackWindow / 16 + 1; q += kUnpackThreads)
      if (base + 16ull * q < alloc) s[q] = __ldg(reinterpret_cast<const uint4*>(bytes + base) + q);
    __syncthreads();
    const unsigned long long c0 = base > b0 ? base : b0, c1 = base + kUnpackWindow < b1 ? base + kUnpackWindow : b1;
    unsigned long long i0 = unpack_ceil_div((long long)c0 - (hi - 4), ps);   // the records with a field whose first byte
    unsigned long long i1 = unpack_ceil_div((long long)c1 - lo, ps);         // lies in [c0, c1)
    i0 = i0 > r0 ? i0 : r0;
    i1 = i1 < r1 ? i1 : r1;
    for (unsigned long long i = i0 + threadIdx.x; i < i1; i += kUnpackThreads) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (k >= nf) break;
        const unsigned long long p = i * ps + (unsigned)f[k];
        if (p < c0 || p >= c1) continue;
        const unsigned q = (unsigned)(p - base);
        const unsigned u = (unsigned)sb[q] | ((unsigned)sb[q + 1] << 8) | ((unsigned)sb[q + 2] << 16) | ((unsigned)sb[q + 3] << 24);
        const double v = (double)__uint_as_float(u);
        if (k < 3) xyz[3ull * i + k] = v; else inten[i] = v;
      }
    }
  }
}

}  // namespace tloam

using namespace tloam;

extern "C" __attribute__((visibility("default"))) int tloam_unpack_scan(const unsigned char* bytes, unsigned long long n,
                                                                        unsigned long long point_step, const int off[4], double* xyz,
                                                                        double* intensity, int device, cudaStream_t stream) {
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess || n == 0) return (int)e;
  const int nf = off[3] >= 0 && intensity ? 4 : 3;
  int lo = off[0], hi = off[0];
  for (int k = 0; k < nf; ++k) {
    lo = off[k] < lo ? off[k] : lo;
    hi = off[k] > hi ? off[k] : hi;
  }
  const unsigned long long fit = kUnpackWindow / point_step;
  const unsigned long long per_block = fit < 1ull ? 1ull : fit > kUnpackMaxRecords ? kUnpackMaxRecords : fit;
  const unsigned long long blocks = (n + per_block - 1ull) / per_block;
  k_unpack_scan<<<(unsigned)blocks, kUnpackThreads, 0, stream>>>(bytes, n, point_step, (n * point_step + 15ull) & ~15ull,
                                                                  make_int4(off[0], off[1], off[2], off[3]), nf, lo, hi + 4, per_block,
                                                                  xyz, intensity);
  return (int)cudaGetLastError();
}
