// map_correct.cu -- libtloam_b200_gmc.so: the global map's per-frame pose tables and its loop-closure correction on the
// device (hand-written CUDA for sm_90a).  The full definition is in include/tloam_b200.h ("Loop-corrected global map");
// tests/map_correct_oracle.py restates it in numpy bit for bit.
//
// Every product and sum is a separately rounded __dmul_rn / __dadd_rn / __dsub_rn in the order written, so that nothing
// is contracted into an FMA and a numpy restatement reproduces every bit.  Poses are column-major 4 x 4.
//
// A separate library so that the kernels of libtloam_b200.so keep their SASS.
#include <cuda_runtime.h>

#include "map_correct.h"

namespace tloam {

constexpr unsigned kGmcT = 256;

__device__ __forceinline__ double gmc_dot3(double a0, double b0, double a1, double b1, double a2, double b2) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a0, b0), __dmul_rn(a1, b1)), __dmul_rn(a2, b2));
}

__device__ __forceinline__ bool gmc_same_bits(const double* a, const double* b) {
  bool same = true;
#pragma unroll
  for (int k = 0; k < 16; ++k) same &= __double_as_longlong(a[k]) == __double_as_longlong(b[k]);
  return same;
}

__device__ __forceinline__ bool gmc_is_identity(const double* a) {
  bool same = true;
#pragma unroll
  for (int k = 0; k < 16; ++k) same &= __double_as_longlong(a[k]) == __double_as_longlong(k % 5 == 0 ? 1.0 : 0.0);
  return same;
}

// C = A B of rigid poses: R_A R_B, R_A t_B + t_A; bottom row (0, 0, 0, 1)
__device__ void gmc_compose(const double* A, const double* B, double* C) {
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) C[4 * c + r] = gmc_dot3(A[r], B[4 * c], A[4 + r], B[4 * c + 1], A[8 + r], B[4 * c + 2]);
    C[12 + r] = __dadd_rn(gmc_dot3(A[r], B[12], A[4 + r], B[13], A[8 + r], B[14]), A[12 + r]);
    C[4 * r + 3] = 0.0;
  }
  C[15] = 1.0;
}

// C = A B^-1 in the operation order of tloam_b200_pose_graph_correction: R = R_A R_B^T, t = t_A - R t_B
__device__ void gmc_mul_inv(const double* A, const double* B, double* C) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) C[4 * c + r] = gmc_dot3(A[r], B[c], A[4 + r], B[4 + c], A[8 + r], B[8 + c]);
  for (int r = 0; r < 3; ++r) C[12 + r] = __dsub_rn(A[12 + r], gmc_dot3(C[r], B[12], C[4 + r], B[13], C[8 + r], B[14]));
  for (int r = 0; r < 3; ++r) C[4 * r + 3] = 0.0;
  C[15] = 1.0;
}

// one warp: lanes 0..15 hold the 16 entries; every source entry is read before any write, so src may alias pose
__global__ void k_gmc_pose(const double* src, double* pose, double* O, double* P, const unsigned long long* frames,
                           unsigned long long cap, tloam_gmc_mat M, int multiply) {
  const int lane = threadIdx.x & 31;
  const double o = lane < 16 ? src[lane] : 0.0;
  double e[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) e[k] = __shfl_sync(0xffffffffu, o, k);
  double p = o;
  if (multiply) {
    double c[16];
    gmc_compose(M.m, e, c);
#pragma unroll
    for (int k = 0; k < 16; ++k)
      if (lane == k) p = c[k];
  }
  if (lane < 16) {
    const unsigned long long f = *frames;
    if (f < cap) { O[16ull * f + lane] = o; P[16ull * f + lane] = p; }
    pose[lane] = p;
  }
}

// per frame f: Delta of its node, C_f = Delta O_f (O_f itself when Delta is the identity), moved = C_f != P_f bitwise;
// a moved frame gets M_f = C_f P_f^-1 and P_f = C_f
__global__ void __launch_bounds__(kGmcT) k_gmc_frames(tloam_gmc_args a) {
  const unsigned long long f = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= a.frames) return;
  const long long k = a.node[f];
  double D[16], O[16], Pf[16], C[16];
  for (int i = 0; i < 16; ++i) { O[i] = a.O[16 * f + i]; Pf[i] = a.P[16 * f + i]; }
  bool ident = k < 0;
  if (k >= 0 && (unsigned long long)k < a.n_opt) {
    double T[16], Ok[16];
    for (int i = 0; i < 16; ++i) { T[i] = a.node_T[16 * k + i]; Ok[i] = a.node_O[16 * k + i]; }
    gmc_mul_inv(T, Ok, D);
    ident = gmc_is_identity(D);
  } else if (k >= 0) {
    for (int i = 0; i < 16; ++i) D[i] = a.delta_new.m[i];
    ident = gmc_is_identity(D);
  }
  if (ident) for (int i = 0; i < 16; ++i) C[i] = O[i];
  else gmc_compose(D, O, C);
  const bool moved = !gmc_same_bits(C, Pf);
  a.moved[f] = moved ? 1u : 0u;
  if (!moved) return;
  double Mf[16];
  gmc_mul_inv(C, Pf, Mf);
  for (int i = 0; i < 16; ++i) { a.M[16 * f + i] = Mf[i]; a.P[16 * f + i] = C[i]; }
}

// map point i: its frame by binary search over the frame table (the last f with offsets[f] <= i), moved by M_f
__global__ void __launch_bounds__(kGmcT) k_gmc_points(tloam_gmc_args a) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.points) return;
  unsigned long long lo = 0, hi = a.frames - 1;
  while (lo < hi) {
    const unsigned long long mid = (lo + hi + 1) / 2;
    if (a.offsets[mid] <= i) lo = mid;
    else hi = mid - 1;
  }
  if (!a.moved[lo]) return;
  const double* M = a.M + 16 * lo;
  double* p = a.map + 3 * i;
  const double x = p[0], y = p[1], z = p[2];
  for (int r = 0; r < 3; ++r) p[r] = __dadd_rn(gmc_dot3(M[r], x, M[4 + r], y, M[8 + r], z), M[12 + r]);
}

}  // namespace tloam

using namespace tloam;

#define TLOAM_GMC_API extern "C" __attribute__((visibility("default")))

TLOAM_GMC_API int tloam_gmc_pose(const double* src, double* pose, double* O, double* P, const unsigned long long* frames,
                                 unsigned long long cap, const tloam_gmc_mat* M, int device, cudaStream_t stream) {
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) return (int)e;
  tloam_gmc_mat m = {};
  if (M) m = *M;
  k_gmc_pose<<<1, 32, 0, stream>>>(src, pose, O, P, frames, cap, m, M ? 1 : 0);
  return (int)cudaGetLastError();
}

TLOAM_GMC_API int tloam_gmc_correct(const tloam_gmc_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  if (!a->frames) return (int)cudaSuccess;
  const tloam_gmc_args args = *a;
  k_gmc_frames<<<(unsigned)((a->frames + kGmcT - 1) / kGmcT), kGmcT, 0, a->stream>>>(args);
  *launches += 1;
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  if (!a->points) return (int)cudaSuccess;
  k_gmc_points<<<(unsigned)((a->points + kGmcT - 1) / kGmcT), kGmcT, 0, a->stream>>>(args);
  *launches += 1;
  return (int)cudaGetLastError();
}
