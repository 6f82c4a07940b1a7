// submap.cuh -- device-side local-map maintenance ("next" row (f)-1 of SURVEY.md section 8).
//
// Restates FrontEnd::updateSubmap (ref: src/front_end/front_end.cpp:201-267) and the first-frame seeding
// (ref: front_end.cpp:285-305) with the PointCloud2 operations they use (ref: src/open3d/PointCloud2.cpp):
//   Transform (:71-75) + operator+= (:96-132)  -> k_transform_append
//   Crop(AxisAlignedBoundingBox) (:551-559)     -> folded into the voxel kernels (inclusive bounds)
//   VoxelDownSample (:358-403)                  -> k_vox_min / k_vox_accum / k_vox_emit (k_vox_keys + sort +
//                                                  k_vox_emit_sorted for the scan features of processCloud)
// so that the map never leaves the GPU between frames: per frame only the new scan's submap selection crosses
// PCIe, instead of the whole 12 MB map (set_target).
//
// VoxelDownSample on the device: voxel index = floor((p - (min_bound - voxel/2)) / voxel) like the reference;
// the per-voxel average is accumulated in 64-bit FIXED POINT (offsets inside the voxel, 2^-40 m resolution), so the VALUES
// do not depend on the order of the atomics (bit-reproducible); each is within 2^-41 + 2^-51 voxel + 1.5 ulp(max |p|) of the
// voxel's EXACT mean (tests/voxel_edges_oracle.py).  The output ORDER is not reproducible: slots are claimed by CAS and k_vox_emit takes
// its output base with one atomicAdd per block, so it follows block scheduling (the reference's own order is
// std::unordered_map iteration order -- implementation-defined).  Downstream, point order only enters the kNN
// tie-break (d2, original index): it can matter for EXACT distance ties between two averaged voxel centres, nowhere else
// (tests compare maps as sets and registration results for equality).
#pragma once
#include <cuda_runtime.h>

#include "map_grid.cuh"

namespace tloam {

struct VoxArgs {
  const double* in;            // AoS xyz
  unsigned n;
  double lo[3], hi[3];         // crop box, inclusive (+-DBL_MAX = no crop)
  double voxel;
  unsigned long long* minenc;  // [3] COMPLEMENTED ordered-uint encodings of the min bound of the cropped cloud (0 = none yet:
                               //     the whole scratch area is cleared by ONE memset; updated with atomicMax)
  unsigned long long* keys;    // [mask+1] 0 = empty
  long long* sums;             // [3*(mask+1)] fixed-point offset sums
  unsigned* cnt;               // [mask+1]
  unsigned mask;
  double* out;                 // AoS xyz of the voxel averages
  unsigned* out_count;
  // sync-free chain: the input count lives on the device (n = *n_dev + n_add; `n` is then only the host's bound) and the
  // crop box is centred on a pose held in device memory (the result of the frame that was just enqueued)
  const unsigned* n_dev;
  unsigned n_add;
  const double* box_pose;      // 4x4 column-major, or nullptr: lo / hi above
  double box_len;
};

__device__ __forceinline__ unsigned vox_n(const VoxArgs& a) { return a.n_dev ? *a.n_dev + a.n_add : a.n; }

__device__ __forceinline__ bool vox_in_box(const VoxArgs& a, double x, double y, double z) {
  if (a.box_pose) {            // inclusive box pose.t +- len (ref: front_end.cpp:248-264)
    const double cx = a.box_pose[12], cy = a.box_pose[13], cz = a.box_pose[14], L = a.box_len;
    return x >= cx - L && x <= cx + L && y >= cy - L && y <= cy + L && z >= cz - L && z <= cz + L;
  }
  return x >= a.lo[0] && x <= a.hi[0] && y >= a.lo[1] && y <= a.hi[1] && z >= a.lo[2] && z <= a.hi[2];
}

// out_off: device-side number of points already in `out` (nullptr = 0)
__global__ void k_transform_append(const double* in, unsigned n, double* out, const double* pose /*device, 16 col-major*/,
                                   const unsigned* out_off) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (out_off) out += 3ull * *out_off;
  const double x = in[3ull * i], y = in[3ull * i + 1], z = in[3ull * i + 2];
  out[3ull * i] = pose[0] * x + pose[4] * y + pose[8] * z + pose[12];
  out[3ull * i + 1] = pose[1] * x + pose[5] * y + pose[9] * z + pose[13];
  out[3ull * i + 2] = pose[2] * x + pose[6] * y + pose[10] * z + pose[14];
}

__global__ void __launch_bounds__(256) k_vox_min(VoxArgs a) {
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.out_count = 0u;              // k_vox_emit (two launches later) counts into it
  double mn[3] = {DBL_MAX, DBL_MAX, DBL_MAX};
  const unsigned n = vox_n(a);
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double x = a.in[3ull * i], y = a.in[3ull * i + 1], z = a.in[3ull * i + 2];
    if (vox_in_box(a, x, y, z)) { mn[0] = fmin(mn[0], x); mn[1] = fmin(mn[1], y); mn[2] = fmin(mn[2], z); }
  }
#pragma unroll
  for (int d = 0; d < 3; ++d)
    for (int o = 16; o > 0; o >>= 1) mn[d] = fmin(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o));
  __shared__ double s_mn[8][3];
  if ((threadIdx.x & 31) == 0)
    for (int d = 0; d < 3; ++d) s_mn[threadIdx.x >> 5][d] = mn[d];
  __syncthreads();
  if (threadIdx.x < 3) {
    double lo = s_mn[0][threadIdx.x];
    for (int wi = 1; wi < 8; ++wi) lo = fmin(lo, s_mn[wi][threadIdx.x]);
    atomicMax(&a.minenc[threadIdx.x], ~enc_ordered(lo));
  }
}

constexpr double kVoxFix = 1099511627776.0;   // 2^40

__global__ void __launch_bounds__(256) k_vox_accum(VoxArgs a) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= vox_n(a)) return;
  const double p[3] = {a.in[3ull * i], a.in[3ull * i + 1], a.in[3ull * i + 2]};
  if (!vox_in_box(a, p[0], p[1], p[2])) return;
  int idx[3];
  long long q[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const double mb = dec_ordered(~a.minenc[d]) - a.voxel * 0.5;            // voxel_min_bound (:367)
    const double ref = (p[d] - mb) / a.voxel;                              // :381
    idx[d] = (int)floor(ref);
    q[d] = llrint((p[d] - (mb + (double)idx[d] * a.voxel)) * kVoxFix);
  }
  const unsigned long long key = cell_key(idx[0] - (1 << 20), idx[1] - (1 << 20), idx[2] - (1 << 20));   // indices are >= 0
  unsigned s = hash_key(key) & a.mask;
  while (true) {
    const unsigned long long prev = atomicCAS(&a.keys[s], 0ull, key);
    if (prev == 0ull || prev == key) break;
    s = (s + 1u) & a.mask;
  }
#pragma unroll
  for (int d = 0; d < 3; ++d) atomicAdd(reinterpret_cast<unsigned long long*>(&a.sums[3ull * s + d]), (unsigned long long)q[d]);
  atomicAdd(&a.cnt[s], 1u);
}

// GetAveragePoint of the occupied slot s (c points) into out[0..2]; both emission orders below write it, so their values
// are the same bits
__device__ __forceinline__ void vox_average(const VoxArgs& a, unsigned s, unsigned c, double* out) {
  const unsigned long long key = a.keys[s];
  const int idx[3] = {(int)((key >> 42) & 0x1FFFFFu), (int)((key >> 21) & 0x1FFFFFu), (int)(key & 0x1FFFFFu)};
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const double mb = dec_ordered(~a.minenc[d]) - a.voxel * 0.5;
    out[d] = mb + (double)idx[d] * a.voxel + ((double)a.sums[3ull * s + d] / kVoxFix) / (double)c;
  }
}

__global__ void __launch_bounds__(256) k_vox_emit(VoxArgs a) {
  const unsigned s = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned c = (s <= a.mask) ? a.cnt[s] : 0u;
  const unsigned has = c > 0u ? 1u : 0u;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned incl = has;
  for (int o = 1; o < 32; o <<= 1) { const unsigned v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  __shared__ unsigned s_w[8];
  __shared__ unsigned s_base;
  if (lane == 31) s_w[warp] = incl;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned tot = 0;
    for (int wi = 0; wi < 8; ++wi) { const unsigned v = s_w[wi]; s_w[wi] = tot; tot += v; }
    s_base = tot ? atomicAdd(a.out_count, tot) : 0u;
  }
  __syncthreads();
  if (!has) return;
  const unsigned j = s_base + s_w[warp] + incl - 1u;
  vox_average(a, s, c, a.out + 3ull * j);
}

// ---- ordered emission (the scan features of tloam_b200_process_cloud): the occupied voxels come out in ascending packed
// key ix<<42 | iy<<21 | iz, i.e. ascending (ix, iy, iz) -- the order of the oracle's VoxelDownSample.  The registration caps
// (*_maxnum) take source features in feature-index order, so a scan cloud must not be ordered by block scheduling.
// k_vox_keys compacts the occupied slots as (~key, slot) pairs; the rank sort / bitonic network of the PCA selection
// (feature_extract.cuh: key descending, index ascending) then orders them by ascending key (keys are distinct); k_vox_emit_sorted
// writes the averages in that order.  The count of occupied voxels lands in *a.out_count (zeroed by k_vox_min).
__global__ void __launch_bounds__(256) k_vox_keys(VoxArgs a, unsigned long long* key_raw, unsigned* slot_raw) {
  const unsigned s = blockIdx.x * blockDim.x + threadIdx.x;
  const bool has = s <= a.mask && a.cnt[s] > 0u;
  __shared__ unsigned s_w[8], s_base;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned b = __ballot_sync(0xffffffffu, has);
  if (lane == 0) s_w[warp] = __popc(b);
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned tot = 0;
    for (int wi = 0; wi < 8; ++wi) { const unsigned v = s_w[wi]; s_w[wi] = tot; tot += v; }
    s_base = tot ? atomicAdd(a.out_count, tot) : 0u;
  }
  __syncthreads();
  if (!has) return;
  const unsigned j = s_base + s_w[warp] + __popc(b & ((1u << lane) - 1u));
  key_raw[j] = ~a.keys[s];
  slot_raw[j] = s;
}

// out[j] = the average of the j-th voxel in key order (slot_sorted: the slots after the sort), j < *a.out_count
__global__ void __launch_bounds__(256) k_vox_emit_sorted(VoxArgs a, const unsigned* slot_sorted, double* out) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= *a.out_count) return;
  const unsigned s = slot_sorted[j];
  vox_average(a, s, a.cnt[s], out + 3ull * j);
}

// SelectByIndex (ref: src/open3d/PointCloud2.cpp:198) on the device: out[j] = in[idx[j]] (idx == nullptr: in[j]), j < n
template <class Index>
__global__ void __launch_bounds__(256) k_select_by_index(const double* in, const Index* idx, unsigned n, double* out) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const size_t i = idx ? (size_t)idx[j] : j;
  out[3ull * j] = in[3ull * i]; out[3ull * j + 1] = in[3ull * i + 1]; out[3ull * j + 2] = in[3ull * i + 2];
}

// host-known counts of the planar / sphere map clouds -> the device-side count array (cnt[c] = n)
__global__ void k_set_counts(unsigned* cnt, int c0, unsigned n0, int c1, unsigned n1) {
  if (threadIdx.x == 0) { if (c0 >= 0) cnt[c0] = n0; if (c1 >= 0) cnt[c1] = n1; }
}

// ---- global map (FrontEnd::updateSubmap with mapping_flag, ref: front_end.cpp:269-274):
//        curr_map = raw.Transform(pose); global_map += curr_map->VoxelDownSample(voxel)
// per frame on the handle's stream: k_gmap_transform (T.p of every raw row + the finite rows compacted + their bounds) ->
// k_gmap_guard (key range) -> voxel_pipeline(sorted) over the finite rows -> k_gmap_emit (ascending key, at the map's
// device-side end) -> k_gmap_commit (count, frame table).  No host round trip: the map's size lives in GMapState.
struct GMapState {
  unsigned long long count;       // points in the map
  unsigned long long frames;      // frames in the map (offsets[0 .. frames] are valid)
  unsigned flags;                 // sticky until the host reads it: kGMapKeyRange | kGMapOverflow
  // ---- per frame (cleared by one memset before k_gmap_transform) ----
  unsigned n_fin;                 // finite rows compacted into the voxel input (0 when the frame is refused)
  unsigned n_vox;                 // voxels of the frame (voxel_pipeline's out_count)
  unsigned refused;
  unsigned long long lo[3];       // complemented ordered encodings of the finite rows' min (0 = none yet)
  unsigned long long hi[3];       // ordered encodings of their max (0 = none yet)
};
constexpr unsigned kGMapKeyRange = 1u, kGMapOverflow = 2u;
constexpr unsigned kGMapKeyBits = 21;   // per axis of the packed voxel key (cell_key)

// reg[i] = T.p_i for every row (non-finite rows stay non-finite, like Transform); the finite rows also go to fin[] (order
// irrelevant: the voxel sums are fixed point and the emission is sorted), with their count and bounds in st.
// Same expression as k_transform_append, so both transforms round alike.  in may alias reg (each thread reads its row first).
__global__ void __launch_bounds__(256) k_gmap_transform(const double* in, unsigned n, const double* pose, double* reg, double* fin,
                                                        GMapState* st) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  double p[3] = {0.0, 0.0, 0.0};
  bool ok = false;
  if (i < n) {
    const double x = in[3ull * i], y = in[3ull * i + 1], z = in[3ull * i + 2];
    p[0] = pose[0] * x + pose[4] * y + pose[8] * z + pose[12];
    p[1] = pose[1] * x + pose[5] * y + pose[9] * z + pose[13];
    p[2] = pose[2] * x + pose[6] * y + pose[10] * z + pose[14];
    reg[3ull * i] = p[0]; reg[3ull * i + 1] = p[1]; reg[3ull * i + 2] = p[2];
    ok = isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned b = __ballot_sync(0xffffffffu, ok);
  unsigned base = 0u;
  if (lane == 0 && b) base = atomicAdd(&st->n_fin, (unsigned)__popc(b));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (ok) {
    const unsigned j = base + __popc(b & ((1u << lane) - 1u));
    fin[3ull * j] = p[0]; fin[3ull * j + 1] = p[1]; fin[3ull * j + 2] = p[2];
  }
  double mn[3], mx[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) { mn[d] = ok ? p[d] : DBL_MAX; mx[d] = ok ? p[d] : -DBL_MAX; }
#pragma unroll
  for (int d = 0; d < 3; ++d)
    for (int o = 16; o > 0; o >>= 1) {
      mn[d] = fmin(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o));
      mx[d] = fmax(mx[d], __shfl_xor_sync(0xffffffffu, mx[d], o));
    }
  __shared__ double s_b[8][6];
  __shared__ unsigned s_any;
  if (threadIdx.x == 0) s_any = 0u;
  __syncthreads();
  if (lane == 0) {
    for (int d = 0; d < 3; ++d) { s_b[warp][d] = mn[d]; s_b[warp][3 + d] = mx[d]; }
    if (b) atomicOr(&s_any, 1u);
  }
  __syncthreads();
  if (threadIdx.x < 6 && s_any) {
    const int d = threadIdx.x;
    double v = s_b[0][d];
    for (int wi = 1; wi < 8; ++wi) v = d < 3 ? fmin(v, s_b[wi][d]) : fmax(v, s_b[wi][d]);
    if (d < 3) atomicMax(&st->lo[d], ~enc_ordered(v));
    else atomicMax(&st->hi[d - 3], enc_ordered(v));
  }
}

// a frame whose finite extent reaches 2^21 voxels on an axis cannot be keyed (the reference's "voxel_size is too small"):
// it is refused -- no voxel input, no append -- and the sticky flag reports it.  floor((p - min_bound) / voxel) as in
// k_vox_accum is monotone in p, so the max row gives the largest index.
__global__ void k_gmap_guard(GMapState* st, double voxel) {
  if (threadIdx.x != 0 || st->n_fin == 0u) return;
  bool bad = false;
  for (int d = 0; d < 3; ++d) {
    const double mb = dec_ordered(~st->lo[d]) - voxel * 0.5;
    const double ref = (dec_ordered(st->hi[d]) - mb) / voxel;
    bad |= !(ref < (double)(1u << kGMapKeyBits));
  }
  if (bad) { st->refused = 1u; st->n_fin = 0u; st->flags |= kGMapKeyRange; }
}

// map[count + j] = the average of the j-th voxel in key order (k_vox_emit_sorted with the output base read on the device);
// nothing is written unless the whole frame fits below cap (k_gmap_commit then flags the overflow)
__global__ void __launch_bounds__(256) k_gmap_emit(VoxArgs a, const unsigned* slot_sorted, double* map, const GMapState* st,
                                                   unsigned long long cap) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned nv = *a.out_count;
  if (j >= nv || st->refused || st->count + nv > cap) return;
  const unsigned s = slot_sorted[j];
  vox_average(a, s, a.cnt[s], map + 3ull * (st->count + j));
}

// offsets[f] = first point of frame f; offsets[frames] = count
__global__ void k_gmap_commit(GMapState* st, unsigned long long* offsets, unsigned long long cap, unsigned long long frame_cap) {
  if (threadIdx.x != 0 || st->refused) return;
  const unsigned long long end = st->count + st->n_vox;
  if (end > cap || st->frames + 1ull >= frame_cap) { st->flags |= kGMapOverflow; return; }
  st->count = end;
  st->frames += 1ull;
  offsets[st->frames] = end;
}

}  // namespace tloam
