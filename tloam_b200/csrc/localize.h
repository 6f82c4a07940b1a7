// localize.h -- the C launchers of libtloam_b200_loc.so (localize.cu): localization of a scan in a prior map, with a grid
// index of the map and a normal per map row (include/tloam_b200.h, "Localization in a prior map").
//
// libtloam_b200.so loads that library with dlopen on tloam_b200_localize_enable and resolves these symbols; nothing here
// defines a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer is a device
// pointer unless marked, each launcher enqueues its work on `stream` of `device`, and nothing synchronises.  The return
// value is a cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "map_merge.h"

#ifdef __cplusplus
extern "C" {
#endif

#define TLOAM_LOC_THREADS 256         // queries per block of the search and the reduction
#define TLOAM_LOC_NORMAL_WARPS 4      // map rows (one per warp) per block of the normal estimation
#define TLOAM_LOC_SUMS 32             // per-block partials: H (21), g (6), contributing rows, sum e^2 over them, sum of
                                      // min(d2, coarse^2) over every query row, two unused
#define TLOAM_LOC_MAX_SPAN 8          // cells per axis a search visits at most (radius <= 3 cells)

// the device-side state of one localization: the current T (R row-major, t), the radius, the iteration count and the
// termination; then the final pass's result, the poses the run started from and its map <- odom correction
typedef struct tloam_loc_state {
  double R[9], t[3];
  double r;
  int iter, done, term, accepted;
  double fitness, rmse;
  unsigned long long inliers;
  double guess[16];                   // G, column-major
  double odom[16];                    // O_now, column-major
  double map_odom[16];                // T . O_now^-1, column-major
} tloam_loc_state;

// what the prediction of the next localization reads (kept on the device across calls)
typedef struct tloam_loc_memory {
  double L[16];                       // the previous result if accepted, else the previous guess
  double O[16];                       // the previous O_now
} tloam_loc_memory;

// the prior map's index: map rows sorted by cell key (stable, so a cell's rows stay in row order)
typedef struct tloam_loc_grid {
  const double* sxyz;                 // n x 3, the map rows in sorted order
  const unsigned* srow;               // n: the map row at each sorted position
  const unsigned long long* ckey;     // n_cells: the occupied cells' keys, ascending
  const unsigned* cstart;             // n_cells + 1: cell j's sorted positions [cstart[j], cstart[j + 1])
  const tloam_gmm_state* st;          // st->n_vox = n_cells (written on the device by the index build)
  double mb[3];                       // the map's min per axis
  double cell;
  long long top[3];                   // the largest cell index per axis
  int bits[3];                        // bits of ix, iy, iz in the key
} tloam_loc_grid;

typedef struct tloam_loc_index_args {
  const double* map;                  // n x 3 (FP64 xyz), n < 2^32
  unsigned long long n;
  tloam_loc_grid grid;                // sxyz, srow, ckey, cstart and st point into the buffers below
  double* sxyz;
  unsigned* srow;
  unsigned long long* ckey;
  unsigned* cstart;
  void* scratch;                      // tloam_loc_scratch_bytes(n)
  tloam_gmm_state* st;                // the bounds and the cell count
  double normal_radius, max_planarity;
  int min_normal_neighbours;
  double* normal;                     // n x 3, map row order
  unsigned char* valid;               // n
  int* neighbours;                    // n
  int device;
  cudaStream_t stream;
} tloam_loc_index_args;

typedef struct tloam_loc_args {
  tloam_loc_grid grid;
  const double* map;                  // n x 3, map row order
  const double* normal;
  const unsigned char* valid;
  const double* query;                // nq x 3
  unsigned long long nq;
  const double* odom;                 // O_now (column-major 4 x 4)
  int predict;                        // 1: G = L . O_prev^-1 . O_now from *memory; 0: G = state->guess (set by the host)
  tloam_loc_memory* memory;
  double corr_dist_coarse, corr_dist_fine, eps_translation, eps_rotation, max_fitness;
  int max_iterations;
  tloam_loc_state* state;
  double* sums;                       // ceil(nq / TLOAM_LOC_THREADS) x TLOAM_LOC_SUMS
  int* match_index;                   // (max_iterations + 1) x nq: pass k's map row (-1: none within the pass's radius)
  double* match_d2;                   // the same passes' d2 (+inf: none)
  int device;
  cudaStream_t stream;
} tloam_loc_args;

// the scratch of an index over n map rows: two key / row buffers and the radix histograms
size_t tloam_loc_scratch_bytes(unsigned long long n);
// clears *st, then k_loc_bounds: the rows' bounds and non-finite flag (st->lo / hi / nonfinite, st->n_sel = n)
int tloam_loc_bounds(const tloam_loc_index_args* a, int* launches);
// with a->grid's mb, cell, top and bits set by the host: k_loc_keys, the shared radix sort, the heads (the cell starts
// and st->n_vox), k_loc_cells (sorted xyz and cell keys), then k_loc_normals
int tloam_loc_index(const tloam_loc_index_args* a, int* launches);
// k_loc_predict, max_iterations rounds of k_loc_match -> k_loc_reduce -> k_loc_step (a round after termination does
// nothing), then the final pass (k_loc_match -> k_loc_reduce -> k_loc_final)
int tloam_loc_run(const tloam_loc_args* a, int* launches);

typedef size_t (*tloam_loc_scratch_bytes_fn)(unsigned long long);
typedef int (*tloam_loc_index_fn)(const tloam_loc_index_args*, int*);
typedef int (*tloam_loc_run_fn)(const tloam_loc_args*, int*);

#ifdef __cplusplus
}
#endif
