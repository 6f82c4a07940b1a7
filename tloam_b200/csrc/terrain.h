// terrain.h -- the C launchers of libtloam_b200_terrain.so (terrain.cu): the terrain map of a cloud, per cell its ground
// reference, elevation, step, slope, roughness and traversability value (include/tloam_b200.h, "Terrain").
//
// libtloam_b200.so loads that library with dlopen on the first terrain call and resolves these symbols; nothing here
// defines a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer is a device pointer,
// each launcher enqueues its work on `stream` of `device`, and nothing synchronises.  The return value is a cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TLOAM_TER_TILE 32                           // cells per side of a layers tile
#define TLOAM_TER_HALO_MAX 16                       // the largest step / slope radius in cells

// what the launchers leave for the host (one copy home each)
typedef struct tloam_ter_state {
  unsigned long long lo[2];           // complemented ordered encodings of the selected finite rows' least x, y (0 = none)
  unsigned long long hi[2];           // ordered encodings of their largest x, y (0 = none)
  unsigned long long used, skipped, dropped, overhang, known, lethal;
} tloam_ter_state;

typedef struct tloam_ter_args {
  const double* rows;                 // count x 3
  const unsigned* through;            // with hits: the removal's counters (static_only), or null (every row)
  const unsigned* hits;
  unsigned min_through;
  unsigned long long count;
  // the grid (set by the host after tloam_ter_bounds)
  double origin_x, origin_y, resolution;
  unsigned width, height;             // width x height <= 2^28
  unsigned rg, rs, rp;                // the radii in cells; rs, rp <= TLOAM_TER_HALO_MAX
  double clearance, max_step, tan_max_slope, max_roughness;
  unsigned min_points, min_fit;
  const signed char* occupancy;       // width x height: the occupancy build's values to combine with, or null
  // per cell (width x height each)
  unsigned long long* lo;             // complemented ordered encoding of the least z (0: no row)
  unsigned long long* gx;             // the ground filter's row pass
  unsigned long long* g;              // complemented ordered encoding of G (0: +inf)
  unsigned long long* e;              // ordered encoding of the elevation (0: no ground-side row)
  unsigned* n;                        // rows
  unsigned* m;                        // ground-side rows
  double* step;
  double* slope;
  double* roughness;
  signed char* values;
  tloam_ter_state* state;
  int device;
  cudaStream_t stream;
} tloam_ter_args;

// clears the state, then k_ter_bounds: the selected finite rows' x / y extent
int tloam_ter_bounds(const tloam_ter_args* a, int* launches);
// clears the cells, then k_ter_low, k_ter_ground (rows, then columns), k_ter_high and k_ter_layers: every layer, value and
// count of the grid
int tloam_ter_build(const tloam_ter_args* a, int* launches);

typedef int (*tloam_ter_fn)(const tloam_ter_args*, int*);

#ifdef __cplusplus
}
#endif
