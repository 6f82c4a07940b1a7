// frontier.h -- the C launchers of libtloam_b200_frontier.so (frontier.cu): the frontier cells of a costmap, their
// 8-connected components and each component's statistics and approach cell (include/tloam_b200.h, "Frontiers").
//
// libtloam_b200.so loads that library with dlopen on the first frontier call and resolves these symbols; nothing here
// defines a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer is a device pointer,
// each launcher enqueues its work on `stream` of `device`, and nothing synchronises.  The return value is a cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "map_merge.h"

#ifdef __cplusplus
extern "C" {
#endif

#define TLOAM_FR_TILE 32                            // cells per side of a labelling tile
#define TLOAM_FR_NONE 0xFFFFFFFFu                   // the label of a cell that is not a frontier cell
#define TLOAM_FR_BLOCKS 1024                        // the most blocks of the ordered compaction (its block counts)

// what the launchers leave for the host: the frontier cells (tloam_fr_label) and the components (the head scan's n_vox)
typedef struct tloam_fr_state {
  tloam_gmm_state gmm;
  unsigned long long cells;
} tloam_fr_state;

// one component (k_fr_stats), 64 B
typedef struct tloam_fr_stat {
  unsigned long long sum_i, sum_j;    // the integer sums of the cells' i and j
  unsigned long long approach_p;      // P at the approach cell
  unsigned n;                         // cells
  unsigned approach;                  // the approach cell's linear index j width + i
  unsigned min_i, min_j, max_i, max_j;
  unsigned first;                     // where its cells begin in the sorted cells
  unsigned pad[3];
} tloam_fr_stat;

typedef struct tloam_fr_args {
  const unsigned char* costs;         // width x height, costmap_2d's codes
  const unsigned long long* P;        // width x height, the plan's potential on those costs
  unsigned width, height;             // >= 1 each, width x height < 2^32 - 1
  unsigned free_max;                  // <= 252
  unsigned* labels;                   // width x height: the root, then the component's id; TLOAM_FR_NONE elsewhere
  unsigned char* tile_any;            // tiles: the tile holds a frontier cell
  unsigned* block_counts;             // TLOAM_FR_BLOCKS
  tloam_fr_state* state;              // 1
  // the grouping (tloam_fr_group), over the state's `cells` frontier cells
  unsigned long long cells;           // the host's copy of state->cells
  unsigned long long* key[2];         // cells each: the root
  unsigned* row[2];                   // cells each: the cell's linear index
  unsigned* hist;                     // 256 x gmm_tiles(cells)
  unsigned* totals;                   // 256
  unsigned* start;                    // cells + 1: where component j's cells begin in the sorted order
  tloam_fr_stat* stats;               // cells (components <= cells)
  int device;
  cudaStream_t stream;
} tloam_fr_args;

// k_fr_tile, k_fr_border and k_fr_flatten: every cell's label (its root) and the frontier cells' count in state->cells
int tloam_fr_label(const tloam_fr_args* a, int* launches);
// over the `cells` frontier cells (buffers laid out by tloam_fr_sort_layout): k_fr_compact (the cells in index order in
// key[0] / row[0]), the radix sort of (root, cell), the head scan and k_fr_stats: the components in state->gmm.n_vox,
// each one's record in stats and its cells' labels set to its id; the sorted cells end in
// row[tloam_fr_passes(width x height) & 1]
int tloam_fr_group(const tloam_fr_args* a, int* launches);
// the bytes of the grouping's buffers for `cells` frontier cells, and their layout in `scratch` (key, row, hist, totals,
// start and stats of *a)
size_t tloam_fr_sort_bytes(unsigned long long cells);
void tloam_fr_sort_layout(void* scratch, unsigned long long cells, tloam_fr_args* a);
// the radix passes of a grid of n cells (the bytes of its largest index)
static inline int tloam_fr_passes(unsigned long long n) {
  int p = 1;
  while (p < 4 && (n - 1) >> (8 * p)) ++p;
  return p;
}

typedef int (*tloam_fr_fn)(const tloam_fr_args*, int*);
typedef size_t (*tloam_fr_sort_bytes_fn)(unsigned long long);
typedef void (*tloam_fr_sort_layout_fn)(void*, unsigned long long, tloam_fr_args*);

#ifdef __cplusplus
}
#endif
