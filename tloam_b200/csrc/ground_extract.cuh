// ground_extract.cuh -- "next" row (f)-4, first part: multi-region ground extraction of the segmentation nodelet on the
// device.  Replaces Segmentation::groundRemove (ref: src/models/segmentation/segmentation.cpp:738-770) and what it calls:
// estimateRingsAndTimes2 / HDL_64E (:341-384) and VLP_16 (:386-429), filterByHeight (:454-470), fillSectionIndex with
// cv::fastAtan2 (:507-541), getSection (:230-238), segmentGroundThread (:626-730), findBestPlane (:551-616); and, for the
// raw-scan chain, RemoveClosedNonFinitePoints (:472-499, k_rm_* at the end of this file).
//
// Pipeline (7 launches, no host round trip until the index lists are fetched):
//   k_ge_pre      per 256-point chunk: quadrant 4 -> 1 transition count (HDL-64E) / first half-pass index (VLP-16),
//                 chunk sum of z
//   k_ge_scan1    prefix of the transition counts (HDL-64E) / first half pass, startOri, scanOri, halfOri (VLP-16);
//                 mean height -> height threshold
//   k_ge_region   per point: the intensity channel (HDL-64E: beam = min(prefix, 63); VLP-16: beamId + correctTime),
//                 key = region (quadrant x section) | above-threshold | dropped; per-chunk key histogram
//   k_ge_scan2    prefix of the histograms per key over the chunks (stable 14-way partition)
//   k_ge_scatter  order[] = point ids grouped by key, index order inside a key (= the reference's regionIndex lists)
//   k_ge_fit      one block per region: 20 lowest seeds of every 10th point, seed set, 3 x (findBestPlane + classify),
//                 region-local ground / leftover lists
//   k_ge_emit     lists in the reference's output order
// Bit-exact against oracle/segmentation_oracle.cpp: every floating-point operation is spelled with round-to-nearest
// intrinsics in the oracle's order (the oracle is compiled with -ffp-contract=off), sums that the reference forms
// sequentially are formed sequentially here too (one lane per accumulator), and the orders the reference leaves
// unspecified are fixed identically on both sides (see the oracle's header).
#pragma once
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>

namespace tloam {

constexpr int kGeChunk = 256;          // points per chunk (k_ge_pre / k_ge_region / k_ge_scatter block size)
constexpr int kGeKeys = 14;            // 12 regions + above the height threshold (12) + dropped (13)
constexpr int kGeFitThreads = 512;
constexpr int kGeMaxIter = 8;
constexpr int kGeSeedCache = 4096;     // seed candidates whose height is cached in shared memory (regions up to 40 960 points)

struct GeArgs {
  const double* pts;                   // AoS xyz
  unsigned n, nchunk;
  int sensor_model, num_sec, max_iter, seed_num;   // sensor_model 64: HDL-64E branch, 16: VLP-16 branch
  double sensor_height, min_range, max_range, plane_dis;
  double ang_bot, vertical_res;        // VLP-16 branch: |initAngle| + 0.1, verticalRes
  float bounds[4];
  int nbounds;
  unsigned* chunk_trans;               // [nchunk] HDL-64E: transitions in the chunk -> exclusive prefix;
                                       //          VLP-16: first half-pass index in the chunk (0xFFFFFFFF: none)
  double* chunk_sum;                   // [nchunk]
  double* scal;                        // [0] height threshold; VLP-16: [1] startOri, [2] scanOri, [3] halfOri
  unsigned* first_trans;               // VLP-16: first half-pass index of the scan (0xFFFFFFFF: none)
  int* beam;                           // [n] (int) of the channel
  double* intensity;                   // [n] the reference's intensity channel (FP64)
  unsigned char* key;                  // [n]
  unsigned* chunk_cnt;                 // [nchunk][kGeKeys] -> exclusive prefix per key
  unsigned* key_base;                  // [kGeKeys + 1]
  unsigned* order;                     // [n]
  unsigned char* flag;                 // [n] by position in `order`: 1 = in the current ground set / ground, 2 = leftover
  unsigned* lists;                     // [2][n] region-local ground / leftover lists at the region's base
  unsigned* reg_cnt;                   // [12][2]
  double* planes;                      // [12][kGeMaxIter][4] (NaN = skipped)
  unsigned* out_ground;                // [n]
  unsigned* out_object;                // [n]
  unsigned* out_counts;                // [2]
};

__device__ __forceinline__ double ge_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ge_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ge_sub(double a, double b) { return __dsub_rn(a, b); }

// cv::fastAtan2 (OpenCV mathfuncs_core), degrees
__device__ __forceinline__ float ge_fast_atan2(float y, float x) {
  const float p1 = 0.9997878412794807f * (float)(180 / M_PI);
  const float p3 = -0.3258083974640975f * (float)(180 / M_PI);
  const float p5 = 0.1555786518463281f * (float)(180 / M_PI);
  const float p7 = -0.04432655554792128f * (float)(180 / M_PI);
  const float eps = (float)DBL_EPSILON;
  const float ax = fabsf(x), ay = fabsf(y);
  float a, c, c2;
  if (ax >= ay) {
    c = __fdiv_rn(ay, __fadd_rn(ax, eps));
    c2 = __fmul_rn(c, c);
    a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
  } else {
    c = __fdiv_rn(ax, __fadd_rn(ay, eps));
    c2 = __fmul_rn(c, c);
    a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
  }
  if (x < 0) a = __fsub_rn(180.f, a);
  if (y < 0) a = __fsub_rn(360.f, a);
  return a;
}

__device__ __forceinline__ int ge_quadrant(double x, double y) {        // get_quadrant, ref: :346-361
  if (x > 0 && y >= 0) return 1;
  if (x <= 0 && y > 0) return 2;
  if (x < 0 && y <= 0) return 3;
  return 4;
}

__device__ __forceinline__ bool ge_transition(const GeArgs& a, unsigned i) {
  if (i == 0u || i >= a.n) return false;                                 // prev_q starts at 0
  const int q = ge_quadrant(a.pts[3ull * i], a.pts[3ull * i + 1]);
  const int pq = ge_quadrant(a.pts[3ull * (i - 1)], a.pts[3ull * (i - 1) + 1]);
  return q == 1 && pq == 4;
}

// Sign of atan2(y, x) without rounding: atan2(+-0, x < 0 or x = -0) = +-pi, atan2(+-0, +0 or x > 0) = +-0.
__device__ __forceinline__ bool ge_ori_negative(double x, double y) {
  return !isnan(x) && (y < 0.0 || (y == 0.0 && signbit(y) && signbit(x)));
}
__device__ __forceinline__ bool ge_ori_positive(double x, double y) {
  return !isnan(x) && (y > 0.0 || (y == 0.0 && !signbit(y) && signbit(x)));
}

// VLP-16 branch (ref: :386-429): the half pass starts at the first i >= 1 with ori[i-1] < 0 < ori[i] (prevOri = 0.0 before
// point 0; after the half pass prevOri = pi - ori >= 0, so the transition fires at most once)
__device__ __forceinline__ bool ge_vlp_transition(const GeArgs& a, unsigned i) {
  if (i == 0u || i >= a.n) return false;
  return ge_ori_positive(a.pts[3ull * i], a.pts[3ull * i + 1]) && ge_ori_negative(a.pts[3ull * (i - 1)], a.pts[3ull * (i - 1) + 1]);
}

__global__ void __launch_bounds__(kGeChunk) k_ge_pre(const __grid_constant__ GeArgs a) {
  const unsigned i = blockIdx.x * kGeChunk + threadIdx.x;
  const bool vlp = a.sensor_model == 16;
  __shared__ double s_z[kGeChunk];
  __shared__ unsigned s_first;
  if (threadIdx.x == 0) s_first = 0xFFFFFFFFu;
  s_z[threadIdx.x] = i < a.n ? a.pts[3ull * i + 2] : 0.0;
  const bool tr = vlp ? ge_vlp_transition(a, i) : ge_transition(a, i);
  const int cnt = __syncthreads_count(tr);                                 // also orders s_first's initialisation
  if (vlp) {
    if (tr) atomicMin(&s_first, i);
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    a.chunk_trans[blockIdx.x] = vlp ? s_first : (unsigned)cnt;
    const unsigned m = min((unsigned)kGeChunk, a.n - blockIdx.x * kGeChunk);
    double s = 0.0;
    for (unsigned k = 0; k < m; ++k) s = ge_add(s, s_z[k]);            // chunk sum in index order (see the oracle)
    a.chunk_sum[blockIdx.x] = s;
  }
}

// exclusive prefix of per-chunk values, in place (one block)
__device__ __forceinline__ void ge_block_exclusive_scan(unsigned* v, unsigned n, unsigned stride, unsigned* total_out) {
  __shared__ unsigned s_warp[32];
  __shared__ unsigned s_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (threadIdx.x == 0) s_carry = 0u;
  __syncthreads();
  for (unsigned base = 0; base < n; base += blockDim.x) {
    const unsigned i = base + threadIdx.x;
    const unsigned x = i < n ? v[(size_t)i * stride] : 0u;
    unsigned incl = x;
    for (int o = 1; o < 32; o <<= 1) { const unsigned t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    unsigned off = s_carry;
    for (int w = 0; w < warp; ++w) off += s_warp[w];
    if (i < n) v[(size_t)i * stride] = off + incl - x;
    __syncthreads();
    if (threadIdx.x == 0) { unsigned t = 0; for (int w = 0; w < nw; ++w) t += s_warp[w]; s_carry += t; }
    __syncthreads();
  }
  if (total_out && threadIdx.x == 0) *total_out = s_carry;
  __syncthreads();
}

__global__ void __launch_bounds__(1024) k_ge_scan1(const __grid_constant__ GeArgs a) {
  const bool vlp = a.sensor_model == 16;
  if (!vlp) ge_block_exclusive_scan(a.chunk_trans, a.nchunk, 1u, nullptr);
  if (threadIdx.x == 0) {
    double total = 0.0;
    unsigned first = 0xFFFFFFFFu;
    for (unsigned c = 0; c < a.nchunk; ++c) {
      total = ge_add(total, a.chunk_sum[c]);
      if (vlp) first = min(first, a.chunk_trans[c]);
    }
    a.scal[0] = ge_add(__ddiv_rn(total, (double)a.n), 0.5);              // mean height + 0.5, ref: :743
    if (vlp) {                                                             // ref: :391-400, :413-416
      const double* p = a.pts;
      const double start = atan2(p[1], p[0]);
      double end = atan2(p[3ull * (a.n - 1) + 1], p[3ull * (a.n - 1)]);
      if (ge_sub(end, start) > 3 * M_PI) end = ge_sub(end, 2 * M_PI);
      else if (ge_sub(end, start) < M_PI) end = ge_add(end, 2 * M_PI);
      a.scal[1] = start;
      a.scal[2] = ge_sub(end, start);
      a.scal[3] = first != 0xFFFFFFFFu ? fabs(ge_sub(atan2(p[3ull * (first - 1) + 1], p[3ull * (first - 1)]), start)) : 0.0;
      *a.first_trans = first;
    }
  }
}

// the VLP-16 channel of point i (ref: :404-425): beamId + correctTime, in the reference's operation order
__device__ __forceinline__ double ge_vlp_channel(const GeArgs& a, unsigned i, double x, double y, double z) {
  const double pitch = __ddiv_rn(ge_mul(atan2(z, __dsqrt_rn(ge_add(ge_mul(x, x), ge_mul(y, y)))), 180.0), M_PI);
  const double beam_id = __ddiv_rn((double)(int)ge_add(pitch, a.ang_bot), a.vertical_res);
  const double ori = atan2(y, x);
  double t;
  if (i >= *a.first_trans) {
    t = __ddiv_rn(ge_add(ge_sub(M_PI, ori), a.scal[3]), a.scal[2]);
    if (t > 1.0) t = 0.99999;
  } else {
    t = __ddiv_rn(fabs(ge_sub(ori, a.scal[1])), a.scal[2]);
  }
  return ge_add(beam_id, t);
}

__device__ __forceinline__ int ge_section(const GeArgs& a, double radius) {   // getSection, ref: :230-238 (see the oracle)
  for (int i = 0; i < a.num_sec; ++i) {
    if (i >= a.nbounds) return a.num_sec - 1;
    if (radius < (double)a.bounds[i]) return i;
  }
  return a.num_sec - 1;
}

__device__ __forceinline__ int ge_key_of(const GeArgs& a, double x, double y, double z, double thr) {
  if (z > thr) return 12;                                                  // filterByHeight, :460-464
  const double r = __dsqrt_rn(ge_add(ge_mul(x, x), ge_mul(y, y)));
  const float theta = ge_fast_atan2((float)(-y), (float)x);                // :522
  const int s = ge_section(a, r);
  int q = -1;
  if (theta >= 0.0f && theta < 90.0f) q = 0;
  else if (theta >= 90.0f && theta < 180.0f) q = 1;
  else if (theta >= 180.0f && theta < 270.0f) q = 2;
  else if (theta >= 270.0f && theta < 360.0f) q = 3;
  return q < 0 ? 13 : q * a.num_sec + s;
}

// rank of this thread among the threads of the block that hold the same key (index order) + per-key block totals
__device__ __forceinline__ unsigned ge_rank_in_block(int key, unsigned (*s_cnt)[kGeKeys], unsigned* totals /*[kGeKeys] or null*/) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned rank = 0u;
#pragma unroll
  for (int k = 0; k < kGeKeys; ++k) {
    const unsigned b = __ballot_sync(0xffffffffu, key == k);
    if (key == k) rank = __popc(b & ((1u << lane) - 1u));
    if (lane == 0) s_cnt[warp][k] = __popc(b);
  }
  __syncthreads();
  if (key >= 0)
    for (int w = 0; w < warp; ++w) rank += s_cnt[w][key];
  if (totals && threadIdx.x < kGeKeys) {
    unsigned t = 0;
    for (int w = 0; w < kGeChunk / 32; ++w) t += s_cnt[w][threadIdx.x];
    totals[threadIdx.x] = t;
  }
  return rank;
}

__global__ void __launch_bounds__(kGeChunk) k_ge_region(const __grid_constant__ GeArgs a) {
  const unsigned i = blockIdx.x * kGeChunk + threadIdx.x;
  __shared__ unsigned s_cnt[kGeChunk / 32][kGeKeys];
  __shared__ unsigned s_w[kGeChunk / 32];
  // HDL-64E: beam = transitions up to and including this point, saturating (ref: :367-374)
  const bool vlp = a.sensor_model == 16;
  const bool tr = !vlp && ge_transition(a, i);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned b = __ballot_sync(0xffffffffu, tr);
  if (lane == 0) s_w[warp] = __popc(b);
  __syncthreads();
  unsigned pre = a.chunk_trans[blockIdx.x] + __popc(b & ((2u << lane) - 1u));
  for (int w = 0; w < warp; ++w) pre += s_w[w];
  int key = -1;
  if (i < a.n) {
    if (vlp) {
      const double c = ge_vlp_channel(a, i, a.pts[3ull * i], a.pts[3ull * i + 1], a.pts[3ull * i + 2]);
      a.intensity[i] = c;
      a.beam[i] = (int)c;
    } else {
      const int bm = (int)pre < a.sensor_model - 1 ? (int)pre : a.sensor_model - 1;
      a.beam[i] = bm;
      a.intensity[i] = (double)bm;
    }
    key = ge_key_of(a, a.pts[3ull * i], a.pts[3ull * i + 1], a.pts[3ull * i + 2], a.scal[0]);
    a.key[i] = (unsigned char)key;
  }
  __syncthreads();
  ge_rank_in_block(key, s_cnt, a.chunk_cnt + (size_t)blockIdx.x * kGeKeys);
}

__global__ void __launch_bounds__(1024) k_ge_scan2(const __grid_constant__ GeArgs a) {
  __shared__ unsigned s_tot[kGeKeys];
  for (int k = 0; k < kGeKeys; ++k) ge_block_exclusive_scan(a.chunk_cnt + k, a.nchunk, (unsigned)kGeKeys, &s_tot[k]);
  if (threadIdx.x == 0) {
    unsigned off = 0u;
    for (int k = 0; k < kGeKeys; ++k) { a.key_base[k] = off; off += s_tot[k]; }
    a.key_base[kGeKeys] = off;
  }
}

__global__ void __launch_bounds__(kGeChunk) k_ge_scatter(const __grid_constant__ GeArgs a) {
  const unsigned i = blockIdx.x * kGeChunk + threadIdx.x;
  __shared__ unsigned s_cnt[kGeChunk / 32][kGeKeys];
  const int key = i < a.n ? (int)a.key[i] : -1;
  const unsigned rank = ge_rank_in_block(key, s_cnt, nullptr);
  if (key >= 0) a.order[a.key_base[key] + a.chunk_cnt[(size_t)blockIdx.x * kGeKeys + key] + rank] = i;
}

// findBestPlane (ref: :551-616) over the positions pos = 0, step, 2 step, ... of the region whose flag is 1, in that
// order.  The reference's sums are sequential (left to right), and so are these: ONE lane per accumulator adds the terms in
// order.  Everything around the additions is parallel: the whole block gathers a tile of candidates into shared memory
// (coordinates for the centroid, the six centred products for the second moments; a candidate that is not selected
// contributes +0.0, which leaves a running sum unchanged -- it can never be -0.0), then lanes 0..2 / 0..5 of warp 0 run
// their chains over the tile out of shared memory.  (Round 2, first version: the lanes read pts[order[..]] behind the flag
// test inside the chain, ~600 cycles of exposed latency per term, 2.5 ms per scan.)
constexpr int kGeTile = 1024;

__device__ __forceinline__ void ge_plane_from_moments(double cx, double cy, double cz, double xx, double xy, double xz, double yy, double yz,
                                                      double zz, double plane[4]);

__device__ __forceinline__ void ge_fit_plane(const GeArgs& a, unsigned base, unsigned cnt, unsigned step, double nsel, double* s_tile,
                                             double* s_bc, double plane[4]) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned ncand = (cnt + step - 1u) / step;
  double acc = 0.0;
  for (unsigned c0 = 0; c0 < ncand; c0 += kGeTile) {
    const unsigned m = min((unsigned)kGeTile, ncand - c0);
    for (unsigned c = tid; c < m; c += kGeFitThreads) {
      const unsigned k = (c0 + c) * step;
      double v0 = 0.0, v1 = 0.0, v2 = 0.0;
      if (a.flag[base + k] == 1) { const double* p = a.pts + 3ull * a.order[base + k]; v0 = p[0]; v1 = p[1]; v2 = p[2]; }
      s_tile[c] = v0; s_tile[kGeTile + c] = v1; s_tile[2 * kGeTile + c] = v2;
    }
    __syncthreads();
    if (warp == 0 && lane < 3) {
      const double* t = s_tile + lane * kGeTile;
#pragma unroll 8
      for (unsigned c = 0; c < m; ++c) acc = ge_add(acc, t[c]);
    }
    __syncthreads();
  }
  if (warp == 0 && lane < 3) s_bc[lane] = __ddiv_rn(acc, nsel);
  __syncthreads();
  const double cx = s_bc[0], cy = s_bc[1], cz = s_bc[2];
  acc = 0.0;
  for (unsigned c0 = 0; c0 < ncand; c0 += kGeTile) {
    const unsigned m = min((unsigned)kGeTile, ncand - c0);
    for (unsigned c = tid; c < m; c += kGeFitThreads) {
      const unsigned k = (c0 + c) * step;
      double q[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      if (a.flag[base + k] == 1) {
        const double* p = a.pts + 3ull * a.order[base + k];
        const double rx = ge_sub(p[0], cx), ry = ge_sub(p[1], cy), rz = ge_sub(p[2], cz);
        q[0] = ge_mul(rx, rx); q[1] = ge_mul(rx, ry); q[2] = ge_mul(rx, rz); q[3] = ge_mul(ry, ry); q[4] = ge_mul(ry, rz); q[5] = ge_mul(rz, rz);
      }
#pragma unroll
      for (int j = 0; j < 6; ++j) s_tile[j * kGeTile + c] = q[j];
    }
    __syncthreads();
    if (warp == 0 && lane < 6) {
      const double* t = s_tile + lane * kGeTile;
#pragma unroll 8
      for (unsigned c = 0; c < m; ++c) acc = ge_add(acc, t[c]);
    }
    __syncthreads();
  }
  if (warp == 0 && lane < 6) s_bc[3 + lane] = __ddiv_rn(acc, nsel);
  __syncthreads();
  if (tid == 0) ge_plane_from_moments(cx, cy, cz, s_bc[3], s_bc[4], s_bc[5], s_bc[6], s_bc[7], s_bc[8], plane);
}

__device__ __forceinline__ void ge_plane_from_moments(double cx, double cy, double cz, double xx, double xy, double xz, double yy, double yz,
                                                      double zz, double plane[4]) {
  double wx = 0.0, wy = 0.0, wz = 0.0;
  auto dot3 = [](double ax, double ay, double az, double bx, double by, double bz) {
    return ge_add(ge_add(ge_mul(ax, bx), ge_mul(ay, by)), ge_mul(az, bz));
  };
  {
    const double det = ge_sub(ge_mul(yy, zz), ge_mul(yz, yz));
    const double ax = det, ay = ge_sub(ge_mul(xz, yz), ge_mul(xy, zz)), az = ge_sub(ge_mul(xy, yz), ge_mul(xz, yy));
    double w = ge_mul(det, det);
    if (dot3(wx, wy, wz, ax, ay, az) < 0.0) w = -w;
    wx = ge_add(wx, ge_mul(ax, w)); wy = ge_add(wy, ge_mul(ay, w)); wz = ge_add(wz, ge_mul(az, w));
  }
  {
    const double det = ge_sub(ge_mul(xx, zz), ge_mul(xz, xz));
    const double ax = ge_sub(ge_mul(xz, yz), ge_mul(xy, zz)), ay = det, az = ge_sub(ge_mul(xy, xz), ge_mul(yz, xx));
    double w = ge_mul(det, det);
    if (dot3(wx, wy, wz, ax, ay, az) < 0.0) w = -w;
    wx = ge_add(wx, ge_mul(ax, w)); wy = ge_add(wy, ge_mul(ay, w)); wz = ge_add(wz, ge_mul(az, w));
  }
  {
    const double det = ge_sub(ge_mul(xx, yy), ge_mul(xy, xy));
    const double ax = ge_sub(ge_mul(xy, yz), ge_mul(xz, yy)), ay = ge_sub(ge_mul(xy, xz), ge_mul(yz, xx)), az = det;
    double w = ge_mul(det, det);
    if (dot3(wx, wy, wz, ax, ay, az) < 0.0) w = -w;
    wx = ge_add(wx, ge_mul(ax, w)); wy = ge_add(wy, ge_mul(ay, w)); wz = ge_add(wz, ge_mul(az, w));
  }
  const double n2 = dot3(wx, wy, wz, wx, wy, wz);
  if (n2 > 0.0) { const double nn = __dsqrt_rn(n2); wx = __ddiv_rn(wx, nn); wy = __ddiv_rn(wy, nn); wz = __ddiv_rn(wz, nn); }   // Eigen 3.3 normalize()
  plane[0] = wx; plane[1] = wy; plane[2] = wz; plane[3] = -dot3(wx, wy, wz, cx, cy, cz);
}

__device__ __forceinline__ unsigned ge_block_sum(unsigned v, unsigned* s_red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned t = 0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_red[w];
  __syncthreads();
  return t;
}

// one block per region, ref: segmentGroundThread :626-730
__global__ void __launch_bounds__(kGeFitThreads) k_ge_fit(const __grid_constant__ GeArgs a) {
  const int rg = blockIdx.x;
  const unsigned base = a.key_base[rg], cnt = a.key_base[rg + 1] - base;
  __shared__ unsigned s_red[kGeFitThreads / 32];
  __shared__ double s_zmin[kGeFitThreads / 32];
  __shared__ unsigned s_kmin[kGeFitThreads / 32];
  __shared__ double s_plane[4], s_lastz, s_sum, s_bc[9];
  __shared__ unsigned s_lastk, s_found;
  extern __shared__ __align__(16) unsigned char ge_raw[];
  double* s_tile = reinterpret_cast<double*>(ge_raw);                      // [6][kGeTile]
  double* s_cz = s_tile + 6 * kGeTile;                                     // [kGeSeedCache] candidate heights (DBL_MAX = not a candidate)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int it = tid; it < kGeMaxIter * 4; it += kGeFitThreads) a.planes[(size_t)rg * kGeMaxIter * 4 + it] = __longlong_as_double(0x7FF8000000000000ll);
  if (tid == 0) { a.reg_cnt[2 * rg] = 0u; a.reg_cnt[2 * rg + 1] = 0u; }
  // ---- seed candidates: every 10th point of the region inside the height / range gates (:641-647) ----
  auto cand_z = [&](unsigned k, double& z) {
    const double* p = a.pts + 3ull * a.order[base + k];
    z = p[2];
    const double r = __dsqrt_rn(ge_add(ge_add(ge_mul(p[0], p[0]), ge_mul(p[1], p[1])), ge_mul(p[2], p[2])));
    return z >= ge_mul(-1.5, a.sensor_height) && r >= a.min_range && r <= a.max_range;
  };
  // heights of the first kGeSeedCache candidates are computed once (the 20 argmin rounds below re-read them)
  for (unsigned j = tid; j < (unsigned)kGeSeedCache && j * 10u < cnt; j += kGeFitThreads) {
    double z;
    s_cz[j] = cand_z(j * 10u, z) ? z : DBL_MAX;
  }
  // ---- the ground_seed_num lowest candidates, ascending (z, k); their sum in that order (:649-657) ----
  if (tid == 0) { s_sum = 0.0; s_lastz = -DBL_MAX; s_lastk = 0u; s_found = 0u; }
  __syncthreads();
  int count = 0;
  for (int round = 0; round < a.seed_num; ++round) {
    double bz = DBL_MAX;
    unsigned bk = 0xFFFFFFFFu;
    const double lz = s_lastz;
    const unsigned lk = s_lastk;
    const bool first = round == 0;
    for (unsigned k = (unsigned)tid * 10u; k < cnt; k += (unsigned)kGeFitThreads * 10u) {
      double z;
      if (k < (unsigned)kGeSeedCache * 10u) { z = s_cz[k / 10u]; if (z == DBL_MAX) continue; }
      else if (!cand_z(k, z)) continue;
      if (!first && !(z > lz || (z == lz && k > lk))) continue;            // already taken
      if (z < bz || (z == bz && k < bk)) { bz = z; bk = k; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const double oz = __shfl_xor_sync(0xffffffffu, bz, o);
      const unsigned ok = __shfl_xor_sync(0xffffffffu, bk, o);
      if (oz < bz || (oz == bz && ok < bk)) { bz = oz; bk = ok; }
    }
    if (lane == 0) { s_zmin[warp] = bz; s_kmin[warp] = bk; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < kGeFitThreads / 32; ++w)
        if (s_zmin[w] < bz || (s_zmin[w] == bz && s_kmin[w] < bk)) { bz = s_zmin[w]; bk = s_kmin[w]; }
      if (bk != 0xFFFFFFFFu) { s_sum = ge_add(s_sum, bz); s_lastz = bz; s_lastk = bk; s_found = 1u; }
      else s_found = 0u;
    }
    __syncthreads();
    if (!s_found) break;
    ++count;
  }
  const double av = count != 0 ? __ddiv_rn(s_sum, (double)count) : 0.0;
  const double zlim = ge_add(av, a.plane_dis);
  // ---- seed set (:659-663), as flags over the region's positions ----
  unsigned nsel = 0u;
  for (unsigned k = tid; k < cnt; k += kGeFitThreads) {
    unsigned char f = 0;
    if (k % 10u == 0u) {
      double z;
      if (k < (unsigned)kGeSeedCache * 10u) { z = s_cz[k / 10u]; if (z != DBL_MAX && z < zlim) f = 1; }
      else if (cand_z(k, z) && z < zlim) f = 1;
    }
    a.flag[base + k] = f;
    nsel += f;
  }
  __syncthreads();
  nsel = ge_block_sum(nsel, s_red);
  if (nsel <= 3u) return;                                                  // :665-666: region skipped entirely
  unsigned step = 10u;
  for (int iter = 0; iter < a.max_iter; ++iter) {
    if (nsel <= 3u) continue;                                              // :670-672
    {
      double plane[4];
      ge_fit_plane(a, base, cnt, step, (double)nsel, s_tile, s_bc, plane);
      if (tid == 0) {
        for (int j = 0; j < 4; ++j) { s_plane[j] = plane[j]; a.planes[((size_t)rg * kGeMaxIter + iter) * 4 + j] = plane[j]; }
      }
    }
    __syncthreads();
    const double p0 = s_plane[0], p1 = s_plane[1], p2 = s_plane[2], p3 = s_plane[3];
    const bool last = iter == a.max_iter - 1;
    unsigned sel = 0u;
    for (unsigned k = tid; k < cnt; k += kGeFitThreads) {
      const double* p = a.pts + 3ull * a.order[base + k];
      const double dis = fabs(ge_add(ge_add(ge_add(ge_mul(p0, p[0]), ge_mul(p1, p[1])), ge_mul(p2, p[2])), ge_mul(p3, 1.0)));
      unsigned char f;
      if (dis < a.plane_dis) f = (last || k % 5u == 0u) ? 1 : 0;           // :685-690
      else f = last ? 2 : 0;                                                // :704-706
      a.flag[base + k] = f;
      sel += f == 1 ? 1u : 0u;
    }
    __syncthreads();
    nsel = ge_block_sum(sel, s_red);
    step = 5u;
  }
  // ---- region-local lists in index order: ground (flag 1), leftover (flag 2) ----
  unsigned run_g = 0u, run_v = 0u;
  for (unsigned k0 = 0; k0 < cnt; k0 += kGeFitThreads) {
    const unsigned k = k0 + tid;
    const unsigned char f = k < cnt ? a.flag[base + k] : 0;
    const unsigned bg = __ballot_sync(0xffffffffu, f == 1), bv = __ballot_sync(0xffffffffu, f == 2);
    __shared__ unsigned s_g[kGeFitThreads / 32], s_v[kGeFitThreads / 32];
    if (lane == 0) { s_g[warp] = __popc(bg); s_v[warp] = __popc(bv); }
    __syncthreads();
    unsigned og = run_g, ov = run_v, tg = 0u, tv = 0u;
    for (int w = 0; w < kGeFitThreads / 32; ++w) { if (w < warp) { og += s_g[w]; ov += s_v[w]; } tg += s_g[w]; tv += s_v[w]; }
    if (f == 1) a.lists[base + og + __popc(bg & ((1u << lane) - 1u))] = a.order[base + k];
    if (f == 2) a.lists[a.n + base + ov + __popc(bv & ((1u << lane) - 1u))] = a.order[base + k];
    run_g += tg; run_v += tv;
    __syncthreads();
  }
  if (tid == 0) { a.reg_cnt[2 * rg] = run_g; a.reg_cnt[2 * rg + 1] = run_v; }
}

// ground_scan = regions' ground lists in (quadrant, section) order; object_scan = regions' leftovers in that order, then
// the points above the height threshold in index order (ref: :722-724, :762).  blockIdx.y = job.
__global__ void __launch_bounds__(256) k_ge_emit(const __grid_constant__ GeArgs a) {
  const int job = blockIdx.y;                       // 0..11 ground of region, 12..23 leftover of region, 24 above-threshold
  const int nreg = 4 * a.num_sec;
  unsigned off = 0u, cnt;
  const unsigned* src;
  unsigned* dst;
  if (job < 12) {
    if (job >= nreg) return;
    for (int r = 0; r < job; ++r) off += a.reg_cnt[2 * r];
    cnt = a.reg_cnt[2 * job]; src = a.lists + a.key_base[job]; dst = a.out_ground;
  } else if (job < 24) {
    const int rg = job - 12;
    if (rg >= nreg) return;
    for (int r = 0; r < rg; ++r) off += a.reg_cnt[2 * r + 1];
    cnt = a.reg_cnt[2 * rg + 1]; src = a.lists + a.n + a.key_base[rg]; dst = a.out_object;
  } else {
    for (int r = 0; r < nreg; ++r) off += a.reg_cnt[2 * r + 1];
    cnt = a.key_base[13] - a.key_base[12]; src = a.order + a.key_base[12]; dst = a.out_object;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      unsigned g = 0u;
      for (int r = 0; r < nreg; ++r) g += a.reg_cnt[2 * r];
      a.out_counts[0] = g; a.out_counts[1] = off + cnt;
    }
  }
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += gridDim.x * blockDim.x) dst[off + i] = src[i];
}

// ---- Segmentation::RemoveClosedNonFinitePoints (ref: :472-499) on the uploaded raw scan: a stable compaction that keeps
// a point iff it has no NaN / Inf coordinate and pt.norm() >= dis_th * dis_th (a norm against a SQUARED threshold:
// near_dis 3.0 removes every point closer than 9 m).  kept[] = the surviving points, map[k] = raw index of kept point k.
struct RmArgs {
  const double* raw;                   // AoS xyz
  unsigned n, nchunk;
  double norm_min;                     // dis_th * dis_th
  unsigned* chunk_cnt;                 // [nchunk] kept points in the chunk -> exclusive prefix
  unsigned* total;                     // [1]
  double* kept;                        // [n] AoS xyz
  unsigned* map;                       // [n]
};

__device__ __forceinline__ bool rm_keep(const RmArgs& a, unsigned i) {
  if (i >= a.n) return false;
  const double x = a.raw[3ull * i], y = a.raw[3ull * i + 1], z = a.raw[3ull * i + 2];
  if (!isfinite(x) || !isfinite(y) || !isfinite(z)) return false;
  return __dsqrt_rn(ge_add(ge_add(ge_mul(x, x), ge_mul(y, y)), ge_mul(z, z))) >= a.norm_min;   // Eigen norm(): (x^2 + y^2) + z^2
}

__global__ void __launch_bounds__(kGeChunk) k_rm_count(const __grid_constant__ RmArgs a) {
  const int cnt = __syncthreads_count(rm_keep(a, blockIdx.x * kGeChunk + threadIdx.x));
  if (threadIdx.x == 0) a.chunk_cnt[blockIdx.x] = (unsigned)cnt;
}

__global__ void __launch_bounds__(1024) k_rm_scan(const __grid_constant__ RmArgs a) {
  ge_block_exclusive_scan(a.chunk_cnt, a.nchunk, 1u, a.total);
}

__global__ void __launch_bounds__(kGeChunk) k_rm_scatter(const __grid_constant__ RmArgs a) {
  const unsigned i = blockIdx.x * kGeChunk + threadIdx.x;
  __shared__ unsigned s_w[kGeChunk / 32];
  const bool keep = rm_keep(a, i);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned b = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) s_w[warp] = __popc(b);
  __syncthreads();
  if (!keep) return;
  unsigned k = a.chunk_cnt[blockIdx.x] + __popc(b & ((1u << lane) - 1u));
  for (int w = 0; w < warp; ++w) k += s_w[w];
  a.kept[3ull * k] = a.raw[3ull * i]; a.kept[3ull * k + 1] = a.raw[3ull * i + 1]; a.kept[3ull * k + 2] = a.raw[3ull * i + 2];
  a.map[k] = i;
}

}  // namespace tloam
