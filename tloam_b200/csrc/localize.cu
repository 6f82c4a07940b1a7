// localize.cu -- libtloam_b200_loc.so: localization of a scan in a prior map (hand-written CUDA for sm_90a).  The map is
// indexed once per load by a grid of `cell`-metre cells: the rows sorted by cell key with the merge's stable radix sort
// (radix_sort.cuh), the occupied cells' keys and starts, and a normal per row by the rule of "Loop verification against a
// submap" (normal_fit.cuh).  Each frame is then the point-to-plane ICP of that verification with the grid search in place
// of the exhaustive one.  The full definition is in include/tloam_b200.h ("Localization in a prior map");
// tests/localize_oracle.py restates it in numpy.
//
// The search is exact: the cells it visits per axis run from the cell of p - rr (rounded down) to the cell of p + rr
// (rounded up), rr = r (1 + 1e-7) rounded up, and the cell index floor((x - min) / cell) is monotone in x, so every row
// with d2 <= r * r lies in a visited cell.  Within that set the nearest row is taken by (d2, row index).
//
// A separate library so that the kernels of libtloam_b200.so keep their SASS.
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>

#include "localize.h"
#include "localize_icp.cuh"
#include "map_grid.cuh"
#include "normal_fit.cuh"
#include "radix_sort.cuh"

namespace tloam {

constexpr unsigned kLocW = TLOAM_LOC_NORMAL_WARPS;
constexpr unsigned kLocCols = TLOAM_LOC_MAX_SPAN * TLOAM_LOC_MAX_SPAN;
constexpr unsigned kLocNb = 256;                           // neighbours a warp sorts in shared memory

static size_t loc_align(size_t v) { return (v + 255) & ~(size_t)255; }

struct LocScratch {
  unsigned long long* key[2];
  unsigned* row[2];
  unsigned* hist;
  unsigned* totals;
  unsigned* block_counts;
};
static LocScratch loc_carve(void* base, unsigned long long n) {
  char* p = static_cast<char*>(base);
  LocScratch s;
  for (int b = 0; b < 2; ++b) { s.key[b] = reinterpret_cast<unsigned long long*>(p); p += loc_align((size_t)n * 8); }
  for (int b = 0; b < 2; ++b) { s.row[b] = reinterpret_cast<unsigned*>(p); p += loc_align((size_t)n * 4); }
  s.hist = reinterpret_cast<unsigned*>(p); p += loc_align((size_t)gmm_tiles(n) * 256 * 4);
  s.totals = reinterpret_cast<unsigned*>(p); p += loc_align(256 * 4);
  s.block_counts = reinterpret_cast<unsigned*>(p);
  return s;
}

// ---- index --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kGmmT) k_loc_bounds(tloam_loc_index_args a) {
  double mn[3] = {DBL_MAX, DBL_MAX, DBL_MAX}, mx[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX};
  unsigned bad = 0u, any = 0u;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const double p[3] = {a.map[3 * i], a.map[3 * i + 1], a.map[3 * i + 2]};
    if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]))) { bad = 1u; continue; }
    any = 1u;
#pragma unroll
    for (int d = 0; d < 3; ++d) { mn[d] = fmin(mn[d], p[d]); mx[d] = fmax(mx[d], p[d]); }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      mn[d] = fmin(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o));
      mx[d] = fmax(mx[d], __shfl_xor_sync(0xffffffffu, mx[d], o));
    }
    bad |= __shfl_xor_sync(0xffffffffu, bad, o);
    any |= __shfl_xor_sync(0xffffffffu, any, o);
  }
  if ((threadIdx.x & 31u) != 0u) return;
  if (bad) atomicOr(&a.st->nonfinite, 1u);
  if (any) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      atomicMax(&a.st->lo[d], ~enc_ordered(mn[d]));
      atomicMax(&a.st->hi[d], enc_ordered(mx[d]));
    }
  }
}

// key = ix << (by + bz) | iy << bz | iz with i = floor((x - min) / cell), each operation rounded on its own
__global__ void __launch_bounds__(kGmmT) k_loc_keys(tloam_loc_index_args a, unsigned long long* key, unsigned* row) {
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    long long idx[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) idx[d] = (long long)floor(__ddiv_rn(__dsub_rn(a.map[3 * i + d], a.grid.mb[d]), a.grid.cell));
    key[i] = loc_key(a.grid, idx[0], idx[1], idx[2]);
    row[i] = (unsigned)i;
  }
}

// sorted position p: its row's xyz; cell j: its key
__global__ void __launch_bounds__(kGmmT) k_loc_cells(tloam_loc_index_args a, const unsigned long long* key) {
  const unsigned n_cells = (unsigned)a.st->n_vox;
  for (unsigned long long p = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; p < a.n;
       p += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long r = a.srow[p];
    a.sxyz[3 * p] = a.map[3 * r]; a.sxyz[3 * p + 1] = a.map[3 * r + 1]; a.sxyz[3 * p + 2] = a.map[3 * r + 2];
    if (p < n_cells) a.ckey[p] = key[a.cstart[p]];
  }
}

// one warp per map row i: the cells within normal_radius, the rows among them with d2 <= normal_radius^2 collected in
// shared memory and put in ascending row order by rank (row indices are distinct), then lane 0 sums the mean and the
// covariance in that order (normal_fit.cuh).  A neighbourhood of more than kLocNb rows is walked in ascending row order
// by a warp minimum per neighbour instead: the same order, so the same bits.
__global__ void __launch_bounds__(kLocW * 32) k_loc_normals(tloam_loc_index_args a) {
  __shared__ unsigned s_lo[kLocW][kLocCols], s_hi[kLocW][kLocCols], s_nb[kLocW][kLocNb];
  __shared__ double s_p[kLocW][kLocNb][3];
  const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  const unsigned long long i = (unsigned long long)blockIdx.x * kLocW + warp;
  if (i >= a.n) return;
  const tloam_loc_grid& g = a.grid;
  const unsigned n_cells = (unsigned)a.st->n_vox;
  const double px = a.map[3 * i], py = a.map[3 * i + 1], pz = a.map[3 * i + 2];
  const double r2 = __dmul_rn(a.normal_radius, a.normal_radius), rr = __dmul_ru(a.normal_radius, kLocInflate);
  long long lx, hx, ly, hy, lz, hz;
  loc_range(g, 0, px, rr, lx, hx);
  loc_range(g, 1, py, rr, ly, hy);
  loc_range(g, 2, pz, rr, lz, hz);
  // the row's own cell: >= 1 each; at most TLOAM_LOC_MAX_SPAN each, since the radius is <= 3 cells and the load refuses a
  // map whose coordinates round by 1e-6 cell or more
  const unsigned ny = (unsigned)(hy - ly + 1), ncol = (unsigned)(hx - lx + 1) * ny;
  for (unsigned c = lane; c < ncol; c += 32) loc_column(g, n_cells, lx + c / ny, ly + c % ny, lz, hz, s_lo[warp][c], s_hi[warp][c]);
  __syncwarp();
  unsigned cnt = 0;
  for (unsigned c = 0; c < ncol; ++c)
    for (unsigned base = s_lo[warp][c]; base < s_hi[warp][c]; base += 32) {
      const unsigned j = base + lane;
      const bool ok = j < s_hi[warp][c] && nf_d2(px, py, pz, g.sxyz[3ull * j], g.sxyz[3ull * j + 1], g.sxyz[3ull * j + 2]) <= r2;
      const unsigned b = __ballot_sync(0xffffffffu, ok);
      const unsigned pos = cnt + __popc(b & ((1u << lane) - 1u));
      if (ok && pos < kLocNb) s_nb[warp][pos] = g.srow[j];
      cnt += __popc(b);
    }
  __syncwarp();
  double c6[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  double mx = 0.0, my = 0.0, mz = 0.0;
  if (cnt <= kLocNb) {
    for (unsigned e = lane; e < cnt; e += 32) {
      const unsigned v = s_nb[warp][e];
      unsigned rank = 0;
      for (unsigned k = 0; k < cnt; ++k) rank += s_nb[warp][k] < v ? 1u : 0u;
      s_p[warp][rank][0] = a.map[3ull * v]; s_p[warp][rank][1] = a.map[3ull * v + 1]; s_p[warp][rank][2] = a.map[3ull * v + 2];
    }
    __syncwarp();
    if (lane != 0) return;
    for (unsigned k = 0; k < cnt; ++k) { mx = __dadd_rn(mx, s_p[warp][k][0]); my = __dadd_rn(my, s_p[warp][k][1]); mz = __dadd_rn(mz, s_p[warp][k][2]); }
    const double n = (double)cnt;
    mx = __ddiv_rn(mx, n); my = __ddiv_rn(my, n); mz = __ddiv_rn(mz, n);
    for (unsigned k = 0; k < cnt; ++k) nf_cov_add(c6, s_p[warp][k][0], s_p[warp][k][1], s_p[warp][k][2], mx, my, mz);
  } else {
    for (int sweep = 0; sweep < 2; ++sweep) {
      long long cur = -1;
      for (;;) {
        unsigned best = 0xffffffffu;
        for (unsigned c = 0; c < ncol; ++c)
          for (unsigned j = s_lo[warp][c] + lane; j < s_hi[warp][c]; j += 32) {
            const unsigned v = g.srow[j];
            if ((long long)v > cur && v < best &&
                nf_d2(px, py, pz, g.sxyz[3ull * j], g.sxyz[3ull * j + 1], g.sxyz[3ull * j + 2]) <= r2)
              best = v;
          }
        best = __reduce_min_sync(0xffffffffu, best);
        if (best == 0xffffffffu) break;
        const double x = a.map[3ull * best], y = a.map[3ull * best + 1], z = a.map[3ull * best + 2];
        if (sweep == 0) { mx = __dadd_rn(mx, x); my = __dadd_rn(my, y); mz = __dadd_rn(mz, z); }
        else nf_cov_add(c6, x, y, z, mx, my, mz);
        cur = best;
      }
      if (sweep == 0) {
        const double n = (double)cnt;
        mx = __ddiv_rn(mx, n); my = __ddiv_rn(my, n); mz = __ddiv_rn(mz, n);
      }
    }
    if (lane != 0) return;
  }
  double nv[3];
  const unsigned char ok = nf_finish((int)cnt, c6, a.min_normal_neighbours, a.max_planarity, nv);
  a.normal[3 * i] = nv[0]; a.normal[3 * i + 1] = nv[1]; a.normal[3 * i + 2] = nv[2];
  a.neighbours[i] = (int)cnt;
  a.valid[i] = ok;
}

// ---- per frame ----------------------------------------------------------------------------------------------------------
// one thread: O_now copied; with predict, G = L . D, D = O_prev^-1 O_now (each product and sum rounded on its own):
//   R_D(r, c) = (R_p(0, r) R_n(0, c) + R_p(1, r) R_n(1, c)) + R_p(2, r) R_n(2, c)
//   t_D(r)    = (R_p(0, r) e0 + R_p(1, r) e1) + R_p(2, r) e2,  e = t_n - t_p
//   R_G(r, c) = (R_L(r, 0) R_D(0, c) + R_L(r, 1) R_D(1, c)) + R_L(r, 2) R_D(2, c)
//   t_G(r)    = ((R_L(r, 0) t_D(0) + R_L(r, 1) t_D(1)) + R_L(r, 2) t_D(2)) + t_L(r)
// then T = G
__global__ void k_loc_predict(tloam_loc_args a) {
  if (threadIdx.x != 0) return;
  tloam_loc_state* s = a.state;
  const double* On = a.odom;
  for (int k = 0; k < 16; ++k) s->odom[k] = On[k];
  if (a.predict) {
    const double* Op = a.memory->O;
    const double* L = a.memory->L;
    double D[16], G[16];
    const double e[3] = {__dsub_rn(On[12], Op[12]), __dsub_rn(On[13], Op[13]), __dsub_rn(On[14], Op[14])};
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c)
        D[4 * c + r] = nf_dot3(Op[4 * r], On[4 * c], Op[4 * r + 1], On[4 * c + 1], Op[4 * r + 2], On[4 * c + 2]);
      D[12 + r] = nf_dot3(Op[4 * r], e[0], Op[4 * r + 1], e[1], Op[4 * r + 2], e[2]);
    }
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) G[4 * c + r] = nf_dot3(L[r], D[4 * c], L[4 + r], D[4 * c + 1], L[8 + r], D[4 * c + 2]);
      G[12 + r] = __dadd_rn(nf_dot3(L[r], D[12], L[4 + r], D[13], L[8 + r], D[14]), L[12 + r]);
      G[4 * r + 3] = 0.0;
    }
    G[15] = 1.0;
    for (int k = 0; k < 16; ++k) s->guess[k] = G[k];
  }
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) s->R[3 * r + c] = s->guess[4 * c + r];
    s->t[r] = s->guess[12 + r];
  }
}

// the bodies are in localize_icp.cuh, shared with the batched runs of relocalization
__global__ void __launch_bounds__(kLocT) k_loc_match(tloam_loc_args a, int pass, int final_pass) {
  loc_match_run(a, LocRun{a}, pass, final_pass);
}

__global__ void __launch_bounds__(kLocT) k_loc_reduce(tloam_loc_args a, int pass, int final_pass) {
  loc_reduce_run(a, LocRun{a}, pass, final_pass);
}

// one warp: the run's totals, then the step (thread 0)
__global__ void k_loc_step(tloam_loc_args a) {
  tloam_loc_state* s = a.state;
  if (s->done) return;
  __shared__ double tot[TLOAM_LOC_SUMS];
  loc_total(a, a.sums, tot);
  if (threadIdx.x != 0) return;
  loc_step_solve(s, tot, a.eps_translation, a.eps_rotation, a.corr_dist_fine, a.max_iterations);
}

__global__ void k_loc_final(tloam_loc_args a) { loc_final_run<true>(a, LocRun{a}); }

static unsigned loc_grid(unsigned long long n, int device) {
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0) sms = 132;
  const unsigned long long need = (n + kGmmT - 1) / kGmmT, cap = (unsigned long long)sms * 8u;
  return (unsigned)(need < cap ? (need ? need : 1ull) : cap);
}

}  // namespace tloam

using namespace tloam;

#define TLOAM_LOC_API extern "C" __attribute__((visibility("default")))

TLOAM_LOC_API size_t tloam_loc_scratch_bytes(unsigned long long n) {
  return 2 * loc_align((size_t)n * 8) + 2 * loc_align((size_t)n * 4) + loc_align((size_t)gmm_tiles(n) * 256 * 4) +
         loc_align(256 * 4) + loc_align(kGmmMaxBlocks * 4);
}

TLOAM_LOC_API int tloam_loc_bounds(const tloam_loc_index_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  if ((e = cudaMemsetAsync(a->st, 0, sizeof(tloam_gmm_state), a->stream)) != cudaSuccess) return (int)e;
  if (!a->n) return (int)cudaSuccess;
  k_loc_bounds<<<loc_grid(a->n, a->device), kGmmT, 0, a->stream>>>(*a);
  *launches = 1;
  return (int)cudaGetLastError();
}

TLOAM_LOC_API int tloam_loc_index(const tloam_loc_index_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  if (!a->n) return (int)cudaSuccess;
  const LocScratch s = loc_carve(a->scratch, a->n);
  const unsigned long long n = a->n;
  const unsigned grid = loc_grid(n, a->device);
  k_loc_keys<<<grid, kGmmT, 0, a->stream>>>(*a, s.key[0], s.row[0]);
  const int passes = (a->grid.bits[0] + a->grid.bits[1] + a->grid.bits[2] + 7) / 8, cur = passes & 1;
  int nl = 1 + gmm_radix_sort(s.key, s.row, n, passes, s.hist, s.totals, a->stream);
  if ((e = cudaMemcpyAsync(a->srow, s.row[cur], n * sizeof(unsigned), cudaMemcpyDeviceToDevice, a->stream)) != cudaSuccess) return (int)e;
  nl += gmm_heads(s.key[cur], n, s.block_counts, a->cstart, a->st, a->stream);
  k_loc_cells<<<grid, kGmmT, 0, a->stream>>>(*a, s.key[cur]);
  k_loc_normals<<<(unsigned)((n + kLocW - 1) / kLocW), kLocW * 32, 0, a->stream>>>(*a);
  *launches = nl + 2;
  return (int)cudaGetLastError();
}

TLOAM_LOC_API int tloam_loc_run(const tloam_loc_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  k_loc_predict<<<1, 32, 0, a->stream>>>(*a);
  *launches = 1;
  if (a->nq) {
    const unsigned qb = (unsigned)((a->nq + kLocT - 1) / kLocT);
    for (int k = 0; k <= a->max_iterations; ++k) {
      const int fin = k == a->max_iterations;
      k_loc_match<<<qb, kLocT, 0, a->stream>>>(*a, k, fin);
      k_loc_reduce<<<qb, kLocT, 0, a->stream>>>(*a, k, fin);
      if (!fin) k_loc_step<<<1, 32, 0, a->stream>>>(*a);
      *launches += fin ? 2 : 3;
      if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    }
  }
  k_loc_final<<<1, 32, 0, a->stream>>>(*a);
  *launches += 1;
  return (int)cudaGetLastError();
}
