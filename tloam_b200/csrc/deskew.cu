// deskew.cu -- libtloam_b200_deskew.so: motion correction of a raw scan on the device (hand-written CUDA for sm_90a).
//
// A spinning sensor takes a whole sweep to build one scan.  With per-point times t_i, t_end the largest finite t_i, the
// frame period P and xi = log(last^-1 . curr) (the constant-velocity increment of the pose history, the one
// scan_match_predicted predicts with), every row becomes
//     p'_i = exp(s_i . xi) . p_i,   s_i = (t_i - t_end) / P,
// the point expressed in the sensor frame at the end of the sweep (LOAM's TransformToEnd).  A non-finite t_i, or a scan
// without a finite time, gives s_i = 0: the row is copied.  exp / log are se3.cuh's, the solver's own.  All FP64; the build
// has no fast-math flags.
//
// A separate library so that the kernels of libtloam_b200.so keep their SASS.
#include <cuda_runtime.h>
#include <math.h>

#include "deskew.h"
#include "se3.cuh"

namespace tloam {

constexpr unsigned kDeskewThreads = 256;
constexpr unsigned kDeskewMaxBlocks = 1056;                 // 8 per SM of an H100 SXM: the grid-stride max

// order-preserving map of a double onto an unsigned 64-bit integer (a > b <=> enc(a) > enc(b)); 0 is below every
// encoded value and stands for "no finite time"
__device__ __forceinline__ unsigned long long deskew_enc(double v) {
  const unsigned long long u = (unsigned long long)__double_as_longlong(v);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double deskew_dec(unsigned long long e) {
  return __longlong_as_double((long long)((e >> 63) ? (e & 0x7fffffffffffffffull) : ~e));
}

// row i's time: the FP64 array, or the packed record's field assembled from single bytes (no alignment is guaranteed:
// velodyne_pointcloud's XYZIRT records are 22 bytes) and scaled by unit
__device__ __forceinline__ double deskew_time(const tloam_deskew_args& a, unsigned long long i) {
  if (a.time) return a.time[i];
  const unsigned char* p = a.records + i * a.point_step + (unsigned)a.offset;
  unsigned long long u = 0;
  const int bytes = a.datatype == 8 ? 8 : 4;
  for (int k = 0; k < bytes; ++k) u |= (unsigned long long)__ldg(p + k) << (8 * k);
  if (a.datatype == 8) return __longlong_as_double((long long)u) * a.unit;
  if (a.datatype == 7) return (double)__uint_as_float((unsigned)u) * a.unit;
  return (double)(unsigned)u * a.unit;                     // 6: UINT32
}

// one warp: xi from the pose history (lane 0), t_end cleared for k_deskew_tend
__global__ void __launch_bounds__(32) k_deskew_motion(tloam_deskew_args a) {
  if (threadIdx.x != 0) return;
  const double* L = a.last_pose;
  const double* Cp = a.curr_pose;
  double step[16];                                          // last^-1 . curr = [Rl^T Rc, Rl^T (tc - tl)], column-major
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r) step[c * 4 + r] = L[r * 4 + 0] * Cp[c * 4 + 0] + L[r * 4 + 1] * Cp[c * 4 + 1] + L[r * 4 + 2] * Cp[c * 4 + 2];
  const double d[3] = {Cp[12] - L[12], Cp[13] - L[13], Cp[14] - L[14]};
  for (int r = 0; r < 3; ++r) step[12 + r] = L[r * 4 + 0] * d[0] + L[r * 4 + 1] * d[1] + L[r * 4 + 2] * d[2];
  step[3] = step[7] = step[11] = 0.0; step[15] = 1.0;
  Pose7 p;
  double xi[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (pose_from_matrix(step, p)) {
    se3_log(p, xi);
    bool finite = true;
    for (int k = 0; k < 6; ++k) finite = finite && isfinite(xi[k]);
    if (!finite)                                            // no usable increment: the scan is not corrected
      for (int k = 0; k < 6; ++k) xi[k] = 0.0;
  }
  for (int k = 0; k < 6; ++k) a.scratch[k] = xi[k];
  reinterpret_cast<unsigned long long*>(a.scratch)[6] = 0ull;
}

// t_end = max of the finite times: grid-stride, a warp max, one atomicMax per warp on the order-preserving encoding
__global__ void __launch_bounds__(kDeskewThreads) k_deskew_tend(tloam_deskew_args a) {
  unsigned long long best = 0ull;
  for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < a.n;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const double t = deskew_time(a, i);
    if (isfinite(t)) {
      const unsigned long long e = deskew_enc(t);
      best = e > best ? e : best;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long v = __shfl_xor_sync(0xffffffffu, best, o);
    best = v > best ? v : best;
  }
  if ((threadIdx.x & 31) == 0 && best) atomicMax(reinterpret_cast<unsigned long long*>(a.scratch) + 6, best);
}

// one thread per row
__global__ void __launch_bounds__(kDeskewThreads) k_deskew(tloam_deskew_args a) {
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const double x = a.xyz[3 * i], y = a.xyz[3 * i + 1], z = a.xyz[3 * i + 2];
  const unsigned long long e = reinterpret_cast<const unsigned long long*>(a.scratch)[6];
  const double t = deskew_time(a, i);
  double s = 0.0;
  if (e && isfinite(t)) s = (t - deskew_dec(e)) / a.period;
  double v[6];
  bool moves = false;
  for (int k = 0; k < 6; ++k) {
    v[k] = s * a.scratch[k];
    moves = moves || v[k] != 0.0;
  }
  double* o = a.out + 3 * i;
  if (!moves) {                                             // s = 0 or xi = 0: the row itself, bit for bit
    o[0] = x; o[1] = y; o[2] = z;
    return;
  }
  const Rt T = pose_to_rt(se3_exp(v));
  rt_apply(T, x, y, z, o[0], o[1], o[2]);
}

}  // namespace tloam

using namespace tloam;

#define TLOAM_DESKEW_API extern "C" __attribute__((visibility("default")))

TLOAM_DESKEW_API int tloam_deskew_motion(const tloam_deskew_args* a) {
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  k_deskew_motion<<<1, 32, 0, a->stream>>>(*a);
  return (int)cudaGetLastError();
}

TLOAM_DESKEW_API int tloam_deskew_tend(const tloam_deskew_args* a) {
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess || a->n == 0) return (int)e;
  const unsigned long long blocks = (a->n + kDeskewThreads - 1) / kDeskewThreads;
  k_deskew_tend<<<(unsigned)(blocks < kDeskewMaxBlocks ? blocks : kDeskewMaxBlocks), kDeskewThreads, 0, a->stream>>>(*a);
  return (int)cudaGetLastError();
}

TLOAM_DESKEW_API int tloam_deskew_apply(const tloam_deskew_args* a) {
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess || a->n == 0) return (int)e;
  k_deskew<<<(unsigned)((a->n + kDeskewThreads - 1) / kDeskewThreads), kDeskewThreads, 0, a->stream>>>(*a);
  return (int)cudaGetLastError();
}
