// scan_context.h -- the C launchers of libtloam_b200_loop.so (scan_context.cu): Scan Context descriptors (Kim & Kim, IROS
// 2018) of raw scans kept in a database on the device, and an exact search of that database for the best earlier frame.
//
// libtloam_b200.so loads that library with dlopen on the first loop call and resolves these symbols; nothing here defines a
// kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer in tloam_sc_args is a device
// pointer, each launcher enqueues its work on `stream` of `device`, and nothing synchronises.  Per added frame they run in
// the order bin, finish, search on the same args.  The return value is a cudaError_t.
//
// A descriptor slot holds n_ring * n_sector bins (row-major: ring r, sector s at r * n_sector + s), then the n_ring ring
// key values, then the n_sector column norms: TLOAM_SC_SLOT_DOUBLES(n_ring, n_sector) doubles.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TLOAM_SC_SLOT_DOUBLES(n_ring, n_sector) ((unsigned long long)(n_ring) * (n_sector) + (n_ring) + (n_sector))
#define TLOAM_SC_MAX_BLOCKS 1056          // search grid cap: 8 blocks per SM of an H100 SXM

// the best (distance, candidate, shift) of a search, lexicographic; candidate -1: no eligible frame
typedef struct tloam_sc_best {
  double distance;
  long long candidate;
  long long shift;
} tloam_sc_best;

typedef struct tloam_sc_args {
  int n_ring, n_sector;
  double lidar_height, max_radius;
  const double* dirs;               // (n_sector - 1) x 2: (cos, sin) of the sector boundary 2 pi k / n_sector, k = 1 ..
  const double* xyz;                // n x 3 FP64, the scan (sensor frame)
  unsigned long long n;
  double* db;                       // the database: slot f at db + f * TLOAM_SC_SLOT_DOUBLES
  unsigned long long frame;         // the slot the scan is binned into, and the query of the search
  unsigned long long n_candidates;  // the search runs over slots 0 .. n_candidates - 1
  tloam_sc_best* partial;           // TLOAM_SC_MAX_BLOCKS entries
  tloam_sc_best* best;              // the result
  int device;
  cudaStream_t stream;
} tloam_sc_args;

// clears the frame's slot, then k_sc_bin: every finite row within max_radius raises its bin to z + lidar_height
int tloam_sc_bin(const tloam_sc_args* a);
// k_sc_finish: bins decoded (an empty bin is 0), ring key and column norms written
int tloam_sc_finish(const tloam_sc_args* a);
// k_sc_search over every (candidate, shift), then k_sc_reduce into *best
int tloam_sc_search(const tloam_sc_args* a);

typedef int (*tloam_sc_fn)(const tloam_sc_args*);

#ifdef __cplusplus
}
#endif
