// map_dynamic.cu -- libtloam_b200_gmd.so: dynamic-point removal for the global map on the device (hand-written CUDA for
// sm_90a).  The full definition is in include/tloam_b200.h ("Dynamic-point removal"); tests/map_dynamic_oracle.py restates
// it in numpy bit for bit.
//
// Per append: the scan's range image (the minimum range per pixel, by atomicMin on the ordered bits of r > 0), its window
// image, then one thread per earlier map point casts that point's vote.  The static map is a count, a block scan and a
// scatter in row order, so it is deterministic.  Every product, sum, quotient and square root is a separately rounded
// __dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn / __dsqrt_rn in the order written, so that nothing is contracted into an
// FMA and a numpy restatement reproduces every counter.
//
// A separate library so that the kernels of libtloam_b200.so keep their SASS.
#include <cuda_runtime.h>

#include "map_dynamic.h"

namespace tloam {

constexpr unsigned kGmdT = 256;
constexpr unsigned kGmdMaxBlocks = 1024;
constexpr unsigned long long kGmdEmpty = 0x7FF0000000000000ull;   // the bits of +inf: an empty pixel

__device__ __forceinline__ double gmd_range(double x, double y, double z) {
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
}

// Scan Context's sector of (x, y): the half-plane split, then the number of boundaries k of that half with
// c_k y - s_k x > 0.  The sign sequence is true then false within a half-plane, so a binary search counts it.
__device__ __forceinline__ int gmd_column(double x, double y, const double* D, int n_cols) {
  const int n_up = (n_cols - 1) / 2;
  const bool upper = y > 0.0 || (y == 0.0 && x >= 0.0);
  const int base = upper ? 0 : n_up;
  int lo = 0, hi = upper ? n_up : n_cols - 1 - n_up;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    const int k = base + mid - 1;
    if (__dsub_rn(__dmul_rn(D[2 * k], y), __dmul_rn(D[2 * k + 1], x)) > 0.0) lo = mid;
    else hi = mid - 1;
  }
  return base + lo;
}

// the pixel of a sensor-frame point and its range; false: outside [min_range, max_range] or outside the image
__device__ __forceinline__ bool gmd_pixel(double x, double y, double z, const tloam_gmd_params& p, int* pix, double* r_out) {
  const double r = gmd_range(x, y, z);
  *r_out = r;
  if (!(r >= p.min_range && r <= p.max_range)) return false;
  const double s = __ddiv_rn(z, r);
  const double* b = p.row_bounds;
  if (!(s >= b[0] && s <= b[p.n_rows])) return false;
  int lo = 0, hi = p.n_rows - 1;                   // the number of k in 1 .. n_rows - 1 with s > b_k
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (s > b[mid]) lo = mid;
    else hi = mid - 1;
  }
  *pix = lo * p.n_cols + gmd_column(x, y, p.col_bounds, p.n_cols);
  return true;
}

__global__ void __launch_bounds__(kGmdT) k_gmd_clear(unsigned long long* image, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) image[i] = kGmdEmpty;
}

__global__ void __launch_bounds__(kGmdT) k_gmd_bin(const double* scan, unsigned n, tloam_gmd_params p,
                                                   unsigned long long* image) {
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int pix;
    double r;
    if (gmd_pixel(scan[3ull * i], scan[3ull * i + 1], scan[3ull * i + 2], p, &pix, &r))
      atomicMin(image + pix, (unsigned long long)__double_as_longlong(r));   // r > 0: the bits order as the values
  }
}

// the minimum over rows i - wr .. i + wr (clipped) and columns j - wc .. j + wc (wrapped); NaN if a pixel there is empty
__global__ void __launch_bounds__(kGmdT) k_gmd_window(const unsigned long long* image, tloam_gmd_params p, double* window) {
  const int n = p.n_rows * p.n_cols;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int row = i / p.n_cols, col = i - row * p.n_cols;
    const int r0 = row - p.wr < 0 ? 0 : row - p.wr, r1 = row + p.wr > p.n_rows - 1 ? p.n_rows - 1 : row + p.wr;
    double m = __longlong_as_double((long long)kGmdEmpty);
    bool known = true;
    for (int rr = r0; rr <= r1; ++rr)
      for (int dc = -p.wc; dc <= p.wc; ++dc) {
        int c = (col + dc) % p.n_cols;
        if (c < 0) c += p.n_cols;
        const unsigned long long v = image[rr * p.n_cols + c];
        known &= v != kGmdEmpty;
        m = fmin(m, __longlong_as_double((long long)v));
      }
    window[i] = known ? m : __longlong_as_double(0x7FF8000000000000ll);
  }
}

// one thread per map row [0, *count): into the sensor frame of the pose, then the vote against its pixel
__global__ void __launch_bounds__(kGmdT) k_gmd_vote(tloam_gmd_params p, const double* pose, const double* map,
                                                    const unsigned long long* count, const unsigned long long* image,
                                                    const double* window, unsigned* through, unsigned* hits) {
  __shared__ double T[16];
  if (threadIdx.x < 16) T[threadIdx.x] = pose[threadIdx.x];
  __syncthreads();
  const unsigned long long n = *count;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const double d0 = __dsub_rn(map[3 * i], T[12]), d1 = __dsub_rn(map[3 * i + 1], T[13]);
    const double d2 = __dsub_rn(map[3 * i + 2], T[14]);
    double q[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)                    // R(k, r) = T[4r + k]: q = R^T d
      q[r] = __dadd_rn(__dadd_rn(__dmul_rn(T[4 * r], d0), __dmul_rn(T[4 * r + 1], d1)), __dmul_rn(T[4 * r + 2], d2));
    int pix;
    double r;
    if (!gmd_pixel(q[0], q[1], q[2], p, &pix, &r)) continue;
    const double mg = fmax(p.margin_abs, __dmul_rn(p.margin_rel, r));
    const unsigned long long c = image[pix];
    if (window[pix] > __dadd_rn(r, mg)) through[i] += 1u;
    if (c != kGmdEmpty && fabs(__dsub_rn(__longlong_as_double((long long)c), r)) <= mg) hits[i] += 1u;
  }
}

__device__ __forceinline__ bool gmd_static(const tloam_gmd_static_args& a, unsigned long long i) {
  const unsigned t = a.through[i];
  return !(t >= a.min_through && t > a.hits[i]);
}

// the sum of one value per thread, the same for every thread of the block
__device__ unsigned gmd_block_sum(unsigned v) {
  __shared__ unsigned part[kGmdT / 32];
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned s = 0;
  for (unsigned w = 0; w < kGmdT / 32; ++w) s += part[w];
  return s;
}

// block b: the static rows of its chunk [b chunk, (b + 1) chunk)
__global__ void __launch_bounds__(kGmdT) k_gmd_count(tloam_gmd_static_args a, unsigned long long chunk) {
  const unsigned long long lo = blockIdx.x * chunk, hi = lo + chunk < a.count ? lo + chunk : a.count;
  unsigned c = 0;
  for (unsigned long long i = lo + threadIdx.x; i < hi; i += kGmdT) c += gmd_static(a, i) ? 1u : 0u;
  c = gmd_block_sum(c);
  if (threadIdx.x == 0) a.block_counts[blockIdx.x] = c;
}

// block b: its base = the static rows of blocks 0 .. b - 1, then its chunk tile by tile, each row at base + the static
// rows before it (a ballot per warp and a scan over the warps), so the output keeps the map's row order
__global__ void __launch_bounds__(kGmdT) k_gmd_scatter(tloam_gmd_static_args a, unsigned long long chunk) {
  __shared__ unsigned warp_n[kGmdT / 32];
  unsigned before = 0;
  for (unsigned k = threadIdx.x; k < blockIdx.x; k += kGmdT) before += a.block_counts[k];
  unsigned long long base = gmd_block_sum(before);
  const unsigned long long lo = blockIdx.x * chunk, hi = lo + chunk < a.count ? lo + chunk : a.count;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (unsigned long long t = lo; t < hi; t += kGmdT) {
    const unsigned long long i = t + threadIdx.x;
    const bool keep = i < hi && gmd_static(a, i);
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_n[warp] = __popc(ballot);
    __syncthreads();
    unsigned off = 0, tile = 0;
    for (unsigned w = 0; w < kGmdT / 32; ++w) {
      off += w < warp ? warp_n[w] : 0u;
      tile += warp_n[w];
    }
    if (keep) {
      const unsigned long long o = base + off + __popc(ballot & ((1u << lane) - 1u));
      a.out_xyz[3 * o] = a.map[3 * i];
      a.out_xyz[3 * o + 1] = a.map[3 * i + 1];
      a.out_xyz[3 * o + 2] = a.map[3 * i + 2];
      if (a.out_intensity) a.out_intensity[o] = a.intensity[i];
    }
    base += tile;
    __syncthreads();
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) *a.total = base;
}

static int gmd_sms(int device) {
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0) sms = 132;
  return sms;
}

}  // namespace tloam

using namespace tloam;

#define TLOAM_GMD_API extern "C" __attribute__((visibility("default")))

TLOAM_GMD_API int tloam_gmd_vote(const tloam_gmd_vote_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  const int n_pix = a->p.n_rows * a->p.n_cols;
  const unsigned gp = (unsigned)((n_pix + kGmdT - 1) / kGmdT);
  k_gmd_clear<<<gp, kGmdT, 0, a->stream>>>(a->image, n_pix);
  *launches += 1;
  if (a->n) {
    k_gmd_bin<<<(a->n + kGmdT - 1) / kGmdT, kGmdT, 0, a->stream>>>(a->scan, a->n, a->p, a->image);
    *launches += 1;
  }
  k_gmd_window<<<gp, kGmdT, 0, a->stream>>>(a->image, a->p, a->window);
  *launches += 1;
  const int sms = gmd_sms(a->device);             // the count is on the device: a grid that fills the GPU, grid-stride
  k_gmd_vote<<<(unsigned)sms * 8u, kGmdT, 0, a->stream>>>(a->p, a->pose, a->map, a->count, a->image, a->window, a->through,
                                                            a->hits);
  *launches += 1;
  return (int)cudaGetLastError();
}

static unsigned long long gmd_chunk(unsigned long long count, unsigned blocks) {
  const unsigned long long c = (count + blocks - 1) / blocks;
  return (c + kGmdT - 1) / kGmdT * kGmdT;
}

TLOAM_GMD_API unsigned tloam_gmd_static_blocks(unsigned long long count) {
  if (!count) return 0;
  unsigned long long b = (count + kGmdT - 1) / kGmdT;
  if (b > kGmdMaxBlocks) b = kGmdMaxBlocks;
  const unsigned long long chunk = gmd_chunk(count, (unsigned)b);
  return (unsigned)((count + chunk - 1) / chunk);
}

TLOAM_GMD_API int tloam_gmd_static(const tloam_gmd_static_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  if (!a->count) return (int)cudaMemsetAsync(a->total, 0, sizeof(unsigned long long), a->stream);
  unsigned long long b = (a->count + kGmdT - 1) / kGmdT;
  if (b > kGmdMaxBlocks) b = kGmdMaxBlocks;
  const unsigned long long chunk = gmd_chunk(a->count, (unsigned)b);
  const unsigned blocks = tloam_gmd_static_blocks(a->count);
  const tloam_gmd_static_args args = *a;
  k_gmd_count<<<blocks, kGmdT, 0, a->stream>>>(args, chunk);
  *launches += 1;
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  k_gmd_scatter<<<blocks, kGmdT, 0, a->stream>>>(args, chunk);
  *launches += 1;
  return (int)cudaGetLastError();
}
