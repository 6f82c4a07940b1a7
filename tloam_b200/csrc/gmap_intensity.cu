// gmap_intensity.cu -- libtloam_b200_gmi.so: the intensity channel of the global map (hand-written CUDA for sm_90a).
//
// The reference's map is XYZI: VoxelDownSample averages intensity_ per voxel (ref: src/open3d/PointCloud2.cpp:253-286,
// :396-397) and operator+= keeps the channel under its own rule (:118-124).  AccumulatedPoint starts from intensity_ = 0.0
// and adds the voxel's rows in ascending row order, then divides by the count: a SEQUENTIAL FP64 sum in raw-row order.
// Restated bit for bit, per frame:
//   k_gmi_rank     every finite row of the registered scan -> its voxel's rank j in the frame's emission order (the key
//                  k_vox_accum computes, looked up in the sorted key list); non-finite rows get j = n_vox (left out)
//   k_gmi_hist     \  stable LSD partition of (j, intensity) on 8-bit digits of j, 1-4 passes from the bound n >= n_vox
//   k_gmi_scatter  /  (those above n_vox's top digit skipped on the device): a voxel's rows become contiguous, in raw order
//   k_gmi_sum      one warp per voxel: +0.0, then __dadd_rn row by row, then / count, at map_intensity[count + j] (the
//                  offset k_gmap_emit writes the xyz at, with its refusal and capacity conditions); thread 0 applies the +=
//                  rule to the channel flag
// k_gmi_plain applies the rule for a frame appended without intensity.
//
// A separate library so that the kernels of libtloam_b200.so keep their SASS: this TU includes map_grid.cuh (no kernels)
// and nothing that defines one.
#include <cuda_runtime.h>
#include <string.h>

#include "gmap_intensity.h"
#include "map_grid.cuh"

namespace tloam {

constexpr unsigned kGmiThreads = 256;
constexpr unsigned kGmiItems = 8;                          // rows per thread of a tile
constexpr unsigned kGmiTile = kGmiThreads * kGmiItems;     // rows per block of the partition
constexpr unsigned kGmiBatch = 16;                         // loads in flight per thread of the last block's scan

static unsigned gmi_tiles(unsigned n) { return (n + kGmiTile - 1) / kGmiTile; }
static int gmi_passes(unsigned n) {                        // 8-bit digits that cover every key (<= n_vox <= n)
  int bits = 0;
  while (bits < 32 && (n >> bits)) ++bits;
  return bits <= 8 ? 1 : (bits + 7) / 8;
}
static size_t gmi_align(size_t v) { return (v + 255) & ~(size_t)255; }

struct GmiScratch {
  unsigned* key[2];
  double* val[2];
  unsigned* hist;                                          // [256][tiles], digit-major
  unsigned* ticket;
};
static GmiScratch gmi_carve(void* base, unsigned n) {
  char* p = static_cast<char*>(base);
  GmiScratch s;
  for (int b = 0; b < 2; ++b) { s.key[b] = reinterpret_cast<unsigned*>(p); p += gmi_align((size_t)n * 4); }
  for (int b = 0; b < 2; ++b) { s.val[b] = reinterpret_cast<double*>(p); p += gmi_align((size_t)n * 8); }
  s.hist = reinterpret_cast<unsigned*>(p); p += gmi_align((size_t)gmi_tiles(n) * 256 * 4);
  s.ticket = reinterpret_cast<unsigned*>(p);
  return s;
}

// j of every row: the voxel index of k_vox_accum (same expression: mb = min_bound - voxel/2, floor((p - mb) / voxel)),
// packed as cell_key and found in the sorted list; a finite row without a voxel is a bug: state[1] is raised
__global__ void __launch_bounds__(kGmiThreads) k_gmi_rank(const double* reg, const double* inten, unsigned n,
                                                          const unsigned long long* minenc, double voxel,
                                                          const unsigned long long* keys_sorted, const unsigned* n_vox,
                                                          const unsigned* refused, unsigned* key_out, double* val_out,
                                                          unsigned* state, unsigned* ticket) {
  if (blockIdx.x == 0 && threadIdx.x == 0) *ticket = 0u;
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (*refused || i >= n) return;
  const unsigned nv = *n_vox;
  const double p[3] = {reg[3ull * i], reg[3ull * i + 1], reg[3ull * i + 2]};
  unsigned j = nv;
  if (isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2])) {
    int idx[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const double mb = dec_ordered(~minenc[d]) - voxel * 0.5;
      idx[d] = (int)floor((p[d] - mb) / voxel);
    }
    const unsigned long long ck = ~cell_key(idx[0] - (1 << 20), idx[1] - (1 << 20), idx[2] - (1 << 20));
    unsigned lo = 0u, hi = nv;                             // first position with keys_sorted[pos] <= ck (descending list)
    while (lo < hi) {
      const unsigned mid = (lo + hi) >> 1;
      if (keys_sorted[mid] > ck) lo = mid + 1u; else hi = mid;
    }
    if (lo < nv && keys_sorted[lo] == ck) j = lo;
    else atomicOr(&state[1], 1u);
  }
  key_out[i] = j;
  val_out[i] = inten[i];
}

// keys are <= n_vox (the sentinel of the non-finite rows): a pass whose digit is 0 for every key would leave the order as it
// is, so it is skipped on the device (the passes that run are a prefix; k_gmi_sum reads the buffer the last one wrote)
__device__ __forceinline__ bool gmi_pass_live(unsigned nv, int sh) { return sh == 0 || (nv >> sh) != 0u; }

// per-tile counts of digit (key >> sh) & 255 at hist[digit * tiles + tile]; the last block to finish turns them into
// exclusive offsets in (digit, tile) order
__global__ void __launch_bounds__(kGmiThreads) k_gmi_hist(const unsigned* key, unsigned n, int sh, unsigned* hist, unsigned tiles,
                                                          unsigned* ticket, const unsigned* refused, const unsigned* n_vox) {
  if (*refused || !gmi_pass_live(*n_vox, sh)) return;
  __shared__ unsigned s_h[256], s_scan[256];
  __shared__ bool s_last;
  const unsigned t = threadIdx.x, lane = t & 31u;
  s_h[t] = 0u;
  __syncthreads();
  const unsigned base = blockIdx.x * kGmiTile;
  for (unsigned q = 0; q < kGmiItems; ++q) {
    const unsigned i = base + q * kGmiThreads + t;
    const unsigned d = i < n ? (key[i] >> sh) & 255u : 256u;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    if (d < 256u && (peers & ((1u << lane) - 1u)) == 0u) atomicAdd(&s_h[d], (unsigned)__popc(peers));
  }
  __syncthreads();
  hist[(size_t)t * tiles + blockIdx.x] = s_h[t];
  __threadfence();
  __syncthreads();
  if (t == 0) s_last = atomicAdd(ticket, 1u) == tiles - 1u;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  unsigned* row = hist + (size_t)t * tiles;                // thread t owns digit t; its loads go out kGmiBatch at a time
  unsigned tot = 0u;
  for (unsigned b0 = 0; b0 < tiles; b0 += kGmiBatch) {
    unsigned c[kGmiBatch];
#pragma unroll
    for (unsigned q = 0; q < kGmiBatch; ++q) c[q] = b0 + q < tiles ? __ldcg(&row[b0 + q]) : 0u;
#pragma unroll
    for (unsigned q = 0; q < kGmiBatch; ++q) tot += c[q];
  }
  s_scan[t] = tot;
  __syncthreads();
  for (unsigned o = 1; o < 256u; o <<= 1) {
    const unsigned v = t >= o ? s_scan[t - o] : 0u;
    __syncthreads();
    s_scan[t] += v;
    __syncthreads();
  }
  unsigned run = s_scan[t] - tot;
  for (unsigned b0 = 0; b0 < tiles; b0 += kGmiBatch) {
    unsigned c[kGmiBatch];
#pragma unroll
    for (unsigned q = 0; q < kGmiBatch; ++q) c[q] = b0 + q < tiles ? __ldcg(&row[b0 + q]) : 0u;
#pragma unroll
    for (unsigned q = 0; q < kGmiBatch; ++q)
      if (b0 + q < tiles) { row[b0 + q] = run; run += c[q]; }
  }
  if (t == 0) *ticket = 0u;
}

// stable scatter by digit: a tile's rows go in row order to the offsets of k_gmi_hist (within a warp by lane, across warps
// by a per-digit prefix, across the tile's sub-tiles by a running offset)
__global__ void __launch_bounds__(kGmiThreads) k_gmi_scatter(const unsigned* key_in, const double* val_in, unsigned n, int sh,
                                                             const unsigned* hist, unsigned tiles, unsigned* key_out,
                                                             double* val_out, const unsigned* refused, const unsigned* n_vox) {
  if (*refused || !gmi_pass_live(*n_vox, sh)) return;
  __shared__ unsigned s_off[256];
  __shared__ unsigned s_w[kGmiThreads / 32][256];
  const unsigned t = threadIdx.x, lane = t & 31u, warp = t >> 5;
  s_off[t] = hist[(size_t)t * tiles + blockIdx.x];
  const unsigned base = blockIdx.x * kGmiTile;
  for (unsigned q = 0; q < kGmiItems; ++q) {
#pragma unroll
    for (unsigned w = 0; w < kGmiThreads / 32; ++w) s_w[w][t] = 0u;
    __syncthreads();
    const unsigned i = base + q * kGmiThreads + t;
    const bool ok = i < n;
    unsigned k = 0u, d = 256u;
    double v = 0.0;
    if (ok) { k = key_in[i]; v = val_in[i]; d = (k >> sh) & 255u; }
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const unsigned r = __popc(peers & ((1u << lane) - 1u));
    if (ok && r == 0u) s_w[warp][d] = __popc(peers);
    __syncthreads();
    unsigned run = s_off[t];
#pragma unroll
    for (unsigned w = 0; w < kGmiThreads / 32; ++w) { const unsigned c = s_w[w][t]; s_w[w][t] = run; run += c; }
    s_off[t] = run;
    __syncthreads();
    if (ok) {
      const unsigned pos = s_w[warp][d] + r;
      key_out[pos] = k;
      val_out[pos] = v;
    }
    __syncthreads();
  }
}

__device__ __forceinline__ unsigned gmi_lower_bound(const unsigned* key, unsigned lo, unsigned hi, unsigned j) {
  while (lo < hi) {
    const unsigned mid = (lo + hi) >> 1;
    if (key[mid] < j) lo = mid + 1u; else hi = mid;
  }
  return lo;
}

// the += rule (ref: PointCloud2.cpp:99-100, :118-124) for a frame that adds voxels: the map keeps its channel iff
// (map empty || map has intensity) && frame has intensity.  A fresh state (no intensity frame since the map was emptied)
// has seen plain frames only: it has a channel iff it is still empty.
__device__ __forceinline__ bool gmi_adds(unsigned nv, unsigned long long cnt, unsigned long long frames, unsigned long long cap,
                                         unsigned long long frame_cap) {
  return nv > 0u && cnt + nv <= cap && frames + 1ull < frame_cap;        // k_gmap_commit appends it
}

// voxel j (one warp): sequential FP64 sum of its rows from +0.0, in raw-row order, / count -> map_intensity[count + j].
// The warp loads 32 consecutive values at a time (the next 32 are in flight) and every lane runs the same chain of adds over
// them by shuffles, so the chain's only wait is the add latency.
__global__ void __launch_bounds__(kGmiThreads) k_gmi_sum(const unsigned* key0, const double* val0, const unsigned* key1,
                                                         const double* val1, int passes, unsigned n, const unsigned* n_vox,
                                                         const unsigned* refused, const unsigned long long* count,
                                                         const unsigned long long* frames, unsigned long long cap,
                                                         unsigned long long frame_cap, double* out, unsigned* state, int fresh) {
  const unsigned long long cnt = *count;
  const unsigned nv = *n_vox;
  const bool ref = *refused != 0u, bad = state[1] != 0u;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    bool has = fresh ? cnt == 0ull : state[0] != 0u;
    if (!ref && gmi_adds(nv, cnt, *frames, cap, frame_cap)) has = (cnt == 0ull || has) && !bad;
    state[0] = has ? 1u : 0u;
  }
  if (ref || bad || cnt + nv > cap) return;
  int live = 0;
  for (int p = 0; p < passes; ++p) live += gmi_pass_live(nv, 8 * p) ? 1 : 0;
  const unsigned* key = (live & 1) ? key1 : key0;
  const double* val = (live & 1) ? val1 : val0;
  const unsigned lane = threadIdx.x & 31u, warps = gridDim.x * blockDim.x / 32u;
  for (unsigned j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < nv; j += warps) {   // warp-uniform
    const unsigned lo = gmi_lower_bound(key, 0u, n, j), hi = gmi_lower_bound(key, lo, n, j + 1u);
    double s = 0.0;
    double v = lo + lane < hi ? val[lo + lane] : 0.0;
    for (unsigned k = lo; k < hi; k += 32u) {
      const double next = k + 32u + lane < hi ? val[k + 32u + lane] : 0.0;
      const unsigned m = hi - k < 32u ? hi - k : 32u;
      if (m == 32u) {                                      // unrolled: the shuffles go out ahead of the adds
#pragma unroll
        for (unsigned q = 0; q < 32u; ++q) s = __dadd_rn(s, __shfl_sync(0xffffffffu, v, q));
      } else {
        for (unsigned q = 0; q < m; ++q) s = __dadd_rn(s, __shfl_sync(0xffffffffu, v, q));
      }
      v = next;
    }
    if (lane == 0) out[cnt + j] = __ddiv_rn(s, (double)(hi - lo));
  }
}

__global__ void k_gmi_plain(unsigned* state, const unsigned* n_vox, const unsigned* refused, const unsigned long long* count,
                            const unsigned long long* frames, unsigned long long cap, unsigned long long frame_cap) {
  if (threadIdx.x != 0 || *refused) return;
  if (gmi_adds(*n_vox, *count, *frames, cap, frame_cap)) state[0] = 0u;
}

}  // namespace tloam

using namespace tloam;

extern "C" __attribute__((visibility("default"))) size_t tloam_gmi_scratch_bytes(unsigned n) {
  return 2 * gmi_align((size_t)n * 4) + 2 * gmi_align((size_t)n * 8) + gmi_align((size_t)gmi_tiles(n) * 256 * 4) + 256;
}

extern "C" __attribute__((visibility("default"))) int tloam_gmi_append(const tloam_gmi_frame* f, int device, cudaStream_t stream,
                                                                       int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess || f->n == 0) return (int)e;
  const unsigned n = f->n, tiles = gmi_tiles(n), gb = (n + kGmiThreads - 1) / kGmiThreads;
  const GmiScratch s = gmi_carve(f->scratch, n);
  k_gmi_rank<<<gb, kGmiThreads, 0, stream>>>(f->reg, f->intensity, n, f->minenc, f->voxel, f->keys_sorted, f->n_vox, f->refused,
                                            s.key[0], s.val[0], f->state, s.ticket);
  int cur = 0, nl = 1;
  const int passes = gmi_passes(n);
  for (int p = 0; p < passes; ++p, cur ^= 1) {
    k_gmi_hist<<<tiles, kGmiThreads, 0, stream>>>(s.key[cur], n, 8 * p, s.hist, tiles, s.ticket, f->refused, f->n_vox);
    k_gmi_scatter<<<tiles, kGmiThreads, 0, stream>>>(s.key[cur], s.val[cur], n, 8 * p, s.hist, tiles, s.key[cur ^ 1], s.val[cur ^ 1],
                                                    f->refused, f->n_vox);
    nl += 2;
  }
  const unsigned warps_per_block = kGmiThreads / 32, need = (n + warps_per_block - 1) / warps_per_block;   // n >= n_vox
  const unsigned sb = need < 2048u ? need : 2048u;                                                           // grid-stride beyond
  k_gmi_sum<<<sb, kGmiThreads, 0, stream>>>(s.key[0], s.val[0], s.key[1], s.val[1], passes, n, f->n_vox, f->refused, f->count,
                                           f->frames, f->cap, f->frame_cap, f->map_intensity, f->state, f->fresh);
  *launches = nl + 1;
  return (int)cudaGetLastError();
}

extern "C" __attribute__((visibility("default"))) int tloam_gmi_plain(unsigned* state, const unsigned* n_vox, const unsigned* refused,
                                                                      const unsigned long long* count, const unsigned long long* frames,
                                                                      unsigned long long cap, unsigned long long frame_cap, int device,
                                                                      cudaStream_t stream) {
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) return (int)e;
  k_gmi_plain<<<1, 32, 0, stream>>>(state, n_vox, refused, count, frames, cap, frame_cap);
  return (int)cudaGetLastError();
}
