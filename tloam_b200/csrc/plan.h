// plan.h -- the C launchers of libtloam_b200_plan.so (plan.cu): the cost-to-go of every cell of a costmap to a goal and
// the paths down it (include/tloam_b200.h, "Path planning").
//
// libtloam_b200.so loads that library with dlopen on the first plan call and resolves these symbols; nothing here
// defines a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer is a device pointer,
// each launcher enqueues its work on `stream` of `device`, and nothing synchronises.  The return value is a cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TLOAM_PLAN_TILE 32                          // cells per side of a relaxation tile
#define TLOAM_PLAN_INF 0xFFFFFFFFFFFFFFFFull        // impassable, or the goal cannot be reached
#define TLOAM_PLAN_SIDE 70                          // a move to a side neighbour costs 70 t, to a diagonal one 99 t
#define TLOAM_PLAN_DIAG 99

// the worklists' state (plan_state, zeroed and seeded by tloam_plan_init): the three rotating counts (round r reads
// count[r % 3] and appends to count[(r + 1) % 3]), the rounds that had work and the tiles they processed
typedef struct tloam_plan_state {
  unsigned count[3];
  unsigned rounds;
  unsigned long long tiles;
  unsigned long long reachable;
} tloam_plan_state;

typedef struct tloam_plan_args {
  const unsigned char* costs;         // width x height, costmap_2d's codes (the source; read by tloam_plan_init only)
  unsigned width, height;             // >= 1 each
  unsigned neutral_cost, cost_factor; // t = neutral_cost + cost_factor c
  int allow_unknown;
  unsigned goal_i, goal_j;            // a passable cell
  unsigned short* t;                  // width x height: the traversal cost, 0 = impassable
  unsigned long long* P;              // width x height: the potential
  unsigned* stamp;                    // tiles: the last round a tile was queued for
  unsigned* list;                     // 2 x tiles: the two worklists of tile indices
  tloam_plan_state* state;            // 1
  int device;
  cudaStream_t stream;
} tloam_plan_args;

// k_plan_init (one thread per cell: t, P = INF, P(goal) = 0) and the worklists seeded with the goal's tile
int tloam_plan_init(const tloam_plan_args* a, int* launches);
// `rounds` launches of k_plan_round from round `first` (>= 1) on; a round with no work exits at once
int tloam_plan_rounds(const tloam_plan_args* a, unsigned first, unsigned rounds, int* launches);
// k_plan_count: the cells with a finite potential into state->reachable
int tloam_plan_count(const tloam_plan_args* a, int* launches);

typedef struct tloam_plan_path_args {
  const unsigned short* t;            // the plan's
  const unsigned long long* P;
  unsigned width, height;
  const int* start;                   // n x 2: the start cells (i, j), i < 0 when the start is not finite or outside
  unsigned n;
  int* status;                        // n (k_plan_length)
  unsigned long long* cost;           // n (k_plan_length): P(start), INF unless the status is 0
  unsigned* length;                   // n (k_plan_length): the cells of the path, 0 unless the status is 0
  const unsigned long long* offset;   // n (k_plan_walk): where each path's cells begin
  int* cells;                         // sum of length x 2 (k_plan_walk): (i, j) from the start to the goal
  int device;
  cudaStream_t stream;
} tloam_plan_path_args;

// k_plan_length: one thread per start, walks the path rule and counts its cells
int tloam_plan_length(const tloam_plan_path_args* a, int* launches);
// k_plan_walk: one thread per start, walks again and writes the cells at the start's offset
int tloam_plan_walk(const tloam_plan_path_args* a, int* launches);

typedef int (*tloam_plan_init_fn)(const tloam_plan_args*, int*);
typedef int (*tloam_plan_rounds_fn)(const tloam_plan_args*, unsigned, unsigned, int*);
typedef int (*tloam_plan_count_fn)(const tloam_plan_args*, int*);
typedef int (*tloam_plan_path_fn)(const tloam_plan_path_args*, int*);

#ifdef __cplusplus
}
#endif
