// plan.cu -- libtloam_b200_plan.so: the cost-to-go of every cell of a costmap to a goal, and the paths down it, on the
// device (hand-written CUDA for sm_90a).  The full definition is in include/tloam_b200.h ("Path planning");
// tests/plan_oracle.py restates it in numpy bit for bit.
//
// The potential P is the unique fixed point of P(v) = min over allowed moves v -> u of (k t(u) + P(u)), P(goal) = 0.  It
// is reached by tiled relaxation over a worklist of TLOAM_PLAN_TILE^2-cell tiles:
//   - k_plan_init: t per cell, P = INF but at the goal, and the goal's tile and the tiles around it as the first
//     round's work.
//   - k_plan_round, a fixed grid per round: each block takes tiles of the round's list, stages a tile's P and t with a
//     one-cell halo in shared memory, and relaxes it in place until a pass lowers nothing (__syncthreads_or).  Lowered
//     cells go back with a 64-bit atomicMin; halo cells are read with relaxed loads, so a value a neighbouring block is
//     lowering at that moment is never read torn.  When an edge or corner cell fell, every tile that has it in its halo
//     is appended to the next round's list, once per round (the tile's stamp holds the round it was queued for).
//     P only falls and every value is the length of a real path; a tile is queued again whenever a cell of its halo fell
//     after it was staged, so when a round has no work every cell satisfies its equation, and the fixed point is unique.
//   - k_plan_count: the cells with a finite P.
// Paths: k_plan_length walks each start's path and counts its cells, k_plan_walk walks it again and writes them.
//
// A separate library so that the kernels of libtloam_b200.so and of the other side libraries keep their SASS.
#include <cuda_runtime.h>

#include "plan.h"

namespace tloam {

constexpr unsigned kPlanT = 256;                   // a round's block: 32 x 8 threads, 4 rows each of a 32 x 32 tile
constexpr unsigned kPlanRows = TLOAM_PLAN_TILE * TLOAM_PLAN_TILE / kPlanT;
constexpr unsigned kPlanS = TLOAM_PLAN_TILE + 2;   // the staged tile's side, halo included
static_assert(TLOAM_PLAN_TILE == 32 && kPlanRows * 8 == TLOAM_PLAN_TILE, "a warp is one row of a tile");

// the moves in the path rule's order: 4 sides, then 4 diagonals
__constant__ int kPlanDi[8] = {1, 0, -1, 0, 1, -1, -1, 1};
__constant__ int kPlanDj[8] = {0, 1, 0, -1, 1, 1, -1, -1};

__device__ __forceinline__ unsigned long long lds_relaxed(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.cta.shared.u64 %0, [%1];" : "=l"(v) : "r"((unsigned)__cvta_generic_to_shared(p)) : "memory");
  return v;
}
__device__ __forceinline__ void sts_relaxed(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.cta.shared.u64 [%0], %1;" :: "r"((unsigned)__cvta_generic_to_shared(p)), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ldg_relaxed(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// one thread per cell: the traversal cost and the initial potential; thread 0 seeds round 1
__global__ void __launch_bounds__(kPlanT) k_plan_init(tloam_plan_args a) {
  const unsigned long long n = (unsigned long long)a.width * a.height;
  const unsigned long long goal = (unsigned long long)a.goal_j * a.width + a.goal_i;
  for (unsigned long long c = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; c < n;
       c += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned code = a.costs[c];
    const bool pass = code <= 252u || (code == 255u && a.allow_unknown);
    a.t[c] = pass ? (unsigned short)(a.neutral_cost + a.cost_factor * (code == 255u ? 252u : code)) : (unsigned short)0;
    a.P[c] = c == goal ? 0ull : TLOAM_PLAN_INF;
  }
  // the goal never falls, so no round would queue a tile for it: round 1 takes its tile and the 8 around it, which hold
  // every cell whose halo the goal can be in
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const unsigned ntx = (a.width + TLOAM_PLAN_TILE - 1) / TLOAM_PLAN_TILE;
    const unsigned nty = (a.height + TLOAM_PLAN_TILE - 1) / TLOAM_PLAN_TILE;
    const long long gi = a.goal_i / TLOAM_PLAN_TILE, gj = a.goal_j / TLOAM_PLAN_TILE;
    unsigned k = 0;
    for (long long nj = gj - 1; nj <= gj + 1; ++nj)
      for (long long ni = gi - 1; ni <= gi + 1; ++ni) {
        if (ni < 0 || nj < 0 || ni >= (long long)ntx || nj >= (long long)nty) continue;
        const unsigned tile = (unsigned)nj * ntx + (unsigned)ni;
        a.list[ntx * nty + k++] = tile;            // round 1 reads list 1 % 2
        a.stamp[tile] = 1;
      }
    a.state->count[0] = 0; a.state->count[1] = k; a.state->count[2] = 0;
    a.state->rounds = 0; a.state->tiles = 0; a.state->reachable = 0;
  }
}

// round r: the tiles of list r % 2 (count[r % 3]) relaxed to local convergence; tiles to redo go to list (r + 1) % 2
__global__ void __launch_bounds__(kPlanT) k_plan_round(tloam_plan_args a, unsigned r) {
  __shared__ unsigned long long sP[kPlanS * kPlanS];
  __shared__ unsigned short sT[kPlanS * kPlanS];
  __shared__ unsigned s_dirs;
  const unsigned count = a.state->count[r % 3];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    if (count) { a.state->rounds += 1; a.state->tiles += count; }
    a.state->count[(r + 2) % 3] = 0;               // the output count of round r + 1, last read by round r - 1
  }
  if (!count) return;
  const unsigned ntx = (a.width + TLOAM_PLAN_TILE - 1) / TLOAM_PLAN_TILE;
  const unsigned nty = (a.height + TLOAM_PLAN_TILE - 1) / TLOAM_PLAN_TILE;
  const unsigned ntiles = ntx * nty;
  const unsigned* in = a.list + (r % 2) * ntiles;
  unsigned* out = a.list + ((r + 1) % 2) * ntiles;
  unsigned* out_count = &a.state->count[(r + 1) % 3];
  const unsigned tx = threadIdx.x % TLOAM_PLAN_TILE, ty = threadIdx.x / TLOAM_PLAN_TILE;
  const unsigned long long goal = (unsigned long long)a.goal_j * a.width + a.goal_i;
  for (unsigned w = blockIdx.x; w < count; w += gridDim.x) {
    const unsigned tile = in[w];
    const unsigned ti = tile % ntx, tj = tile / ntx;
    const long long x0 = (long long)ti * TLOAM_PLAN_TILE - 1, y0 = (long long)tj * TLOAM_PLAN_TILE - 1;
    if (threadIdx.x == 0) s_dirs = 0;
    for (unsigned k = threadIdx.x; k < kPlanS * kPlanS; k += kPlanT) {
      const long long x = x0 + (long long)(k % kPlanS), y = y0 + (long long)(k / kPlanS);
      unsigned short t = 0;
      unsigned long long p = TLOAM_PLAN_INF;
      if (x >= 0 && y >= 0 && x < (long long)a.width && y < (long long)a.height) {
        const unsigned long long c = (unsigned long long)y * a.width + (unsigned long long)x;
        t = a.t[c];
        if (t) p = ldg_relaxed(a.P + c);
      }
      sT[k] = t;
      sP[k] = p;
    }
    __syncthreads();
    // this thread's cells (tx, ty + 8 q) and their allowed moves (bit d: move d of kPlanDi / kPlanDj)
    unsigned mask[kPlanRows];
    unsigned long long p0[kPlanRows];
    for (unsigned q = 0; q < kPlanRows; ++q) {
      const unsigned lx = tx + 1, ly = ty + 8 * q + 1, s = ly * kPlanS + lx;
      const unsigned long long gx = (unsigned long long)(x0 + lx), gy = (unsigned long long)(y0 + ly);
      unsigned m = 0;
      if (sT[s] && gy * a.width + gx != goal) {
        for (int d = 0; d < 8; ++d) {
          const int di = kPlanDi[d], dj = kPlanDj[d];
          if (!sT[s + dj * (int)kPlanS + di]) continue;
          if (d >= 4 && (!sT[s + di] || !sT[s + dj * (int)kPlanS])) continue;
          m |= 1u << d;
        }
      }
      mask[q] = m;
      p0[q] = sP[s];
    }
    bool changed;
    do {
      changed = false;
      for (unsigned q = 0; q < kPlanRows; ++q) {
        if (!mask[q]) continue;
        const unsigned s = (ty + 8 * q + 1) * kPlanS + tx + 1;
        const unsigned long long cur = lds_relaxed(&sP[s]);
        unsigned long long best = cur;
        for (int d = 0; d < 8; ++d) {
          if (!((mask[q] >> d) & 1u)) continue;
          const unsigned u = s + kPlanDj[d] * (int)kPlanS + kPlanDi[d];
          const unsigned long long pu = lds_relaxed(&sP[u]);
          if (pu == TLOAM_PLAN_INF) continue;
          const unsigned long long c = pu + (unsigned long long)(d < 4 ? TLOAM_PLAN_SIDE : TLOAM_PLAN_DIAG) * sT[u];
          if (c < best) best = c;
        }
        if (best < cur) { sts_relaxed(&sP[s], best); changed = true; }
      }
    } while (__syncthreads_or(changed));
    // write back what fell; an edge cell that fell queues the tiles that hold it in their halo
    unsigned dirs = 0;
    for (unsigned q = 0; q < kPlanRows; ++q) {
      const unsigned lx = tx + 1, ly = ty + 8 * q + 1;
      const unsigned long long p = sP[ly * kPlanS + lx];
      if (p >= p0[q]) continue;
      atomicMin(a.P + (unsigned long long)(y0 + ly) * a.width + (unsigned long long)(x0 + lx), p);
      const int ex = lx == 1 ? -1 : lx == TLOAM_PLAN_TILE ? 1 : 0;
      const int ey = ly == 1 ? -1 : ly == TLOAM_PLAN_TILE ? 1 : 0;
      if (ex) dirs |= 1u << ((ex + 1) + 3 * 1);
      if (ey) dirs |= 1u << (1 + 3 * (ey + 1));
      if (ex && ey) dirs |= 1u << ((ex + 1) + 3 * (ey + 1));
    }
    if (dirs) atomicOr(&s_dirs, dirs);
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int b = 0; b < 9; ++b) {
        if (!((s_dirs >> b) & 1u)) continue;
        const long long ni = (long long)ti + (b % 3) - 1, nj = (long long)tj + (b / 3) - 1;
        if (ni < 0 || nj < 0 || ni >= (long long)ntx || nj >= (long long)nty) continue;
        const unsigned nt = (unsigned)nj * ntx + (unsigned)ni;
        if (atomicExch(&a.stamp[nt], r + 1) == r + 1) continue;
        out[atomicAdd(out_count, 1u)] = nt;
      }
    }
    __syncthreads();                               // s_dirs and the staged tile are reused by the next tile
  }
}

// one thread per cell: the cells with a finite potential, counted by warp
__global__ void __launch_bounds__(kPlanT) k_plan_count(tloam_plan_args a) {
  const unsigned long long n = (unsigned long long)a.width * a.height;
  for (unsigned long long base = (unsigned long long)blockIdx.x * blockDim.x; base < n;
       base += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long c = base + threadIdx.x;
    const bool fin = c < n && a.P[c] != TLOAM_PLAN_INF;
    const unsigned m = __ballot_sync(0xFFFFFFFFu, fin);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(&a.state->reachable, (unsigned long long)__popc(m));
  }
}

// the path rule's next cell from (i, j): the first allowed move in kPlanDi / kPlanDj order with the least k t(u) + P(u).
// For the fixed point that least value is pv = P(i, j), so P(u) <= pv - 70; false when it exceeds pv (never for the
// fixed point), which keeps every walk finite
__device__ __forceinline__ bool plan_next(const tloam_plan_path_args& a, int* i, int* j, unsigned long long pv) {
  const unsigned short* t = a.t;
  const int W = (int)a.width, H = (int)a.height;
  unsigned long long best = TLOAM_PLAN_INF;
  int bi = 0, bj = 0;
  for (int d = 0; d < 8; ++d) {
    const int ui = *i + kPlanDi[d], uj = *j + kPlanDj[d];
    if (ui < 0 || uj < 0 || ui >= W || uj >= H) continue;
    const unsigned long long u = (unsigned long long)uj * a.width + (unsigned)ui;
    const unsigned tu = t[u];
    if (!tu) continue;
    if (d >= 4 && (!t[(unsigned long long)*j * a.width + (unsigned)ui] || !t[(unsigned long long)uj * a.width + (unsigned)*i]))
      continue;
    const unsigned long long pu = a.P[u];
    if (pu == TLOAM_PLAN_INF) continue;
    const unsigned long long c = pu + (unsigned long long)(d < 4 ? TLOAM_PLAN_SIDE : TLOAM_PLAN_DIAG) * tu;
    if (c < best) { best = c; bi = ui; bj = uj; }
  }
  if (best > pv) return false;
  *i = bi; *j = bj;
  return true;
}

// one thread per start: the status, the cost and the number of cells of its path
__global__ void __launch_bounds__(kPlanT) k_plan_length(tloam_plan_path_args a) {
  const unsigned s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= a.n) return;
  int i = a.start[2 * s], j = a.start[2 * s + 1];
  int status = 1;
  unsigned long long cost = TLOAM_PLAN_INF;
  unsigned len = 0;
  if (i >= 0) {
    const unsigned long long c = (unsigned long long)j * a.width + (unsigned)i;
    if (!a.t[c]) status = 2;
    else if (a.P[c] == TLOAM_PLAN_INF) status = 3;
    else {
      status = 0;
      cost = a.P[c];
      unsigned long long pv = cost;
      len = 1;
      while (pv != 0 && plan_next(a, &i, &j, pv)) {
        pv = a.P[(unsigned long long)j * a.width + (unsigned)i];
        ++len;
      }
    }
  }
  a.status[s] = status;
  a.cost[s] = cost;
  a.length[s] = len;
}

// one thread per start: the cells of its path (status 0 only) from its offset on
__global__ void __launch_bounds__(kPlanT) k_plan_walk(tloam_plan_path_args a) {
  const unsigned s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= a.n || a.status[s] != 0) return;
  int i = a.start[2 * s], j = a.start[2 * s + 1];
  int* out = a.cells + 2 * a.offset[s];
  const unsigned len = a.length[s];
  out[0] = i; out[1] = j;
  unsigned long long pv = a.cost[s];
  for (unsigned k = 1; k < len && plan_next(a, &i, &j, pv); ++k) {
    pv = a.P[(unsigned long long)j * a.width + (unsigned)i];
    out[2 * k] = i; out[2 * k + 1] = j;
  }
}

static int plan_sms(int device) {
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0) sms = 132;
  return sms;
}

static unsigned plan_cell_grid(int device, unsigned long long cells) {
  const unsigned long long blocks = (unsigned long long)plan_sms(device) * 16u;   // grid-stride beyond this
  const unsigned long long need = (cells + kPlanT - 1) / kPlanT;
  return (unsigned)(need < blocks ? (need ? need : 1) : blocks);
}

}  // namespace tloam

using namespace tloam;

#define TLOAM_PLAN_API extern "C" __attribute__((visibility("default")))

TLOAM_PLAN_API int tloam_plan_init(const tloam_plan_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  const unsigned ntiles = ((a->width + TLOAM_PLAN_TILE - 1) / TLOAM_PLAN_TILE) * ((a->height + TLOAM_PLAN_TILE - 1) / TLOAM_PLAN_TILE);
  if ((e = cudaMemsetAsync(a->stamp, 0, (size_t)ntiles * sizeof(unsigned), a->stream)) != cudaSuccess) return (int)e;
  k_plan_init<<<plan_cell_grid(a->device, (unsigned long long)a->width * a->height), kPlanT, 0, a->stream>>>(*a);
  *launches += 1;
  return (int)cudaGetLastError();
}

TLOAM_PLAN_API int tloam_plan_rounds(const tloam_plan_args* a, unsigned first, unsigned rounds, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  int per_sm = 0;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_plan_round, kPlanT, 0)) != cudaSuccess) return (int)e;
  const unsigned grid = (unsigned)plan_sms(a->device) * (unsigned)(per_sm > 0 ? per_sm : 1);
  for (unsigned r = first; r < first + rounds; ++r) k_plan_round<<<grid, kPlanT, 0, a->stream>>>(*a, r);
  *launches += (int)rounds;
  return (int)cudaGetLastError();
}

TLOAM_PLAN_API int tloam_plan_count(const tloam_plan_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  k_plan_count<<<plan_cell_grid(a->device, (unsigned long long)a->width * a->height), kPlanT, 0, a->stream>>>(*a);
  *launches += 1;
  return (int)cudaGetLastError();
}

TLOAM_PLAN_API int tloam_plan_length(const tloam_plan_path_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  if (!a->n) return cudaSuccess;
  k_plan_length<<<(a->n + kPlanT - 1) / kPlanT, kPlanT, 0, a->stream>>>(*a);
  *launches += 1;
  return (int)cudaGetLastError();
}

TLOAM_PLAN_API int tloam_plan_walk(const tloam_plan_path_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  if (!a->n) return cudaSuccess;
  k_plan_walk<<<(a->n + kPlanT - 1) / kPlanT, kPlanT, 0, a->stream>>>(*a);
  *launches += 1;
  return (int)cudaGetLastError();
}
