// relocalize.cu -- libtloam_b200_reloc.so: relocalization in a prior map (hand-written CUDA for sm_90a).  The query's Scan
// Context descriptor (made by libtloam_b200_loop.so) is compared with every place of a saved session at every column
// shift (scan_context.cuh, the loop search's distance); the top_k places below max_distance become hypotheses, each
// started from its place's pose turned by its shift, and all of them are refined against the map in one launch sequence
// by the localization's ICP (localize_icp.cuh), so that hypothesis k is exactly one localization from its guess.  The
// full definition is in include/tloam_b200.h ("Relocalization in a prior map"); tests/relocalize_oracle.py restates it.
#include <cuda_runtime.h>
#include <math.h>

#include "localize_icp.cuh"
#include "relocalize.h"
#include "scan_context.cuh"
#include "scan_context.h"

namespace tloam {

constexpr unsigned kRlT = 256;
constexpr unsigned kRlTopT = 1024;
constexpr size_t kRlMaxSmem = 200 * 1024;
constexpr long long kRlNone = 0x7fffffffffffffffll;

// hypothesis k's run: its state, partial sums and match records
struct RlRun {
  const tloam_rl_args& a;
  unsigned k;
  __device__ __forceinline__ unsigned long long qb() const { return (a.loc.nq + kLocT - 1) / kLocT; }
  __device__ __forceinline__ unsigned long long stride() const { return (unsigned long long)(a.loc.max_iterations + 1) * a.loc.nq; }
  __device__ __forceinline__ tloam_loc_state* state() const { return a.states + k; }
  __device__ __forceinline__ double* sums() const { return a.sums + k * qb() * TLOAM_LOC_SUMS; }
  __device__ __forceinline__ int* match_index() const { return a.match_index + k * stride(); }
  __device__ __forceinline__ double* match_d2() const { return a.match_d2 + k * stride(); }
};

// Each block holds the query in shared memory and streams groups of `per_block` places through it; thread p of a group
// takes place p / S at shift s = p % S.  Then thread m keeps place m's first minimum over the shifts in ascending s: the
// minimum by (distance, shift).
__global__ void __launch_bounds__(kRlT) k_rl_search(tloam_rl_args a, int per_block) {
  extern __shared__ double sm[];
  const int R = a.n_ring, S = a.n_sector;
  const int bins = R * S, desc = bins + S;
  const unsigned long long slot = TLOAM_SC_SLOT_DOUBLES(R, S);
  double* qb = sm;
  for (int k = threadIdx.x; k < desc; k += blockDim.x) qb[k] = k < bins ? a.qdesc[k] : a.qdesc[bins + R + (k - bins)];
  double* dist = sm + (size_t)(1 + per_block) * desc;
  const unsigned long long M = a.n_places;
  for (unsigned long long g = blockIdx.x; g * per_block < M; g += gridDim.x) {
    __syncthreads();
    for (int k = threadIdx.x; k < per_block * desc; k += blockDim.x) {
      const int m = k / desc, o = k - m * desc;
      const unsigned long long j = g * per_block + m;
      if (j < M) sm[desc + k] = a.places[j * slot + (o < bins ? o : bins + R + (o - bins))];
    }
    __syncthreads();
    for (int p = threadIdx.x; p < per_block * S; p += blockDim.x) {
      const int m = p / S, s = p - m * S;
      if (g * per_block + m >= M) continue;
      const double* cb = sm + desc + (size_t)m * desc;
      dist[p] = sc_distance(qb, qb + bins, cb, cb + bins, R, S, s);
    }
    __syncthreads();
    for (int m = threadIdx.x; m < per_block; m += blockDim.x) {
      const unsigned long long j = g * per_block + m;
      if (j >= M) continue;
      double bd = dist[m * S];
      long long bs = 0;
      for (int s = 1; s < S; ++s)
        if (dist[m * S + s] < bd) { bd = dist[m * S + s]; bs = s; }
      a.place_distance[j] = bd;
      a.place_shift[j] = bs;
    }
  }
}

// one block: the first top_k places by (distance, place) with distance < max_distance, one block minimum per rank above
// the previous rank's (distance, place)
__global__ void __launch_bounds__(kRlTopT) k_rl_topk(tloam_rl_args a) {
  __shared__ double wd[kRlTopT / 32];
  __shared__ long long wj[kRlTopT / 32];
  __shared__ double last_d;
  __shared__ long long last_j;
  __shared__ int n;
  if (threadIdx.x == 0) { last_d = -INFINITY; last_j = -1; n = 0; }
  __syncthreads();
  for (int r = 0; r < a.top_k; ++r) {
    double bd = INFINITY;
    long long bj = kRlNone;
    for (unsigned long long j = threadIdx.x; j < a.n_places; j += blockDim.x) {
      const double d = a.place_distance[j];
      if (d < a.max_distance && sc_less(last_d, last_j, 0, d, (long long)j, 0) && sc_less(d, (long long)j, 0, bd, bj, 0)) {
        bd = d;
        bj = (long long)j;
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const double od = __shfl_down_sync(0xffffffffu, bd, o);
      const long long oj = __shfl_down_sync(0xffffffffu, bj, o);
      if (sc_less(od, oj, 0, bd, bj, 0)) { bd = od; bj = oj; }
    }
    if ((threadIdx.x & 31) == 0) { wd[threadIdx.x >> 5] = bd; wj[threadIdx.x >> 5] = bj; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (unsigned w = 1; w < blockDim.x / 32; ++w)
        if (sc_less(wd[w], wj[w], 0, bd, bj, 0)) { bd = wd[w]; bj = wj[w]; }
      if (bj != kRlNone) {
        a.top->place[n] = bj;
        a.top->shift[n] = a.place_shift[bj];
        a.top->distance[n] = bd;
        ++n;
        last_d = bd;
        last_j = bj;
      }
    }
    __syncthreads();
    if (n <= r) break;                                      // no place left below max_distance
  }
  if (threadIdx.x == 0) a.top->n = n;
}

// thread k: hypothesis k's guess G = P_j . Rz(yaw_s), direction m = (-s) mod n_sector ((1, 0) for m = 0, else the sector
// boundary table's), R_G(r, c) = (R_P(r, 0) Rz(0, c) + R_P(r, 1) Rz(1, c)) + R_P(r, 2) Rz(2, c), t_G = t_P; O_now; T = G.
// A slot past the hypotheses is done (EMPTY).
__global__ void k_rl_guess(tloam_rl_args a) {
  const int k = threadIdx.x;
  if (k >= a.top_k) return;
  tloam_loc_state* s = a.states + k;
  if (k >= a.top->n) { s->done = 1; s->term = kLocEmpty; return; }
  const int S = a.n_sector;
  const long long sh = a.top->shift[k];
  const int m = (int)((S - sh) % S);
  const double c = m == 0 ? 1.0 : a.dirs[2 * (m - 1)], sn = m == 0 ? 0.0 : a.dirs[2 * (m - 1) + 1];
  const double Rz[9] = {c, -sn, 0.0, sn, c, 0.0, 0.0, 0.0, 1.0};   // row-major
  const double* P = a.poses + 16 * a.top->place[k];
  double G[16];
  for (int r = 0; r < 3; ++r) {
    for (int j = 0; j < 3; ++j) G[4 * j + r] = nf_dot3(P[r], Rz[j], P[4 + r], Rz[3 + j], P[8 + r], Rz[6 + j]);
    G[12 + r] = P[12 + r];
    G[4 * r + 3] = 0.0;
  }
  G[15] = 1.0;
  for (int q = 0; q < 16; ++q) { s->guess[q] = G[q]; s->odom[q] = a.loc.odom[q]; }
  for (int r = 0; r < 3; ++r) {
    for (int j = 0; j < 3; ++j) s->R[3 * r + j] = G[4 * j + r];
    s->t[r] = G[12 + r];
  }
}

// grid (query blocks, top_k): the localization's pass for every hypothesis
__global__ void __launch_bounds__(kLocT) k_rl_match(tloam_rl_args a, int pass, int final_pass) {
  if (blockIdx.y >= (unsigned)a.top->n) return;
  loc_match_run(a.loc, RlRun{a, blockIdx.y}, pass, final_pass);
}

__global__ void __launch_bounds__(kLocT) k_rl_reduce(tloam_rl_args a, int pass, int final_pass) {
  if (blockIdx.y >= (unsigned)a.top->n) return;
  loc_reduce_run(a.loc, RlRun{a, blockIdx.y}, pass, final_pass);
}

// one warp per hypothesis (block k)
__global__ void k_rl_step(tloam_rl_args a) {
  if (blockIdx.x >= (unsigned)a.top->n) return;
  const RlRun run{a, blockIdx.x};
  tloam_loc_state* s = run.state();
  if (s->done) return;
  __shared__ double tot[TLOAM_LOC_SUMS];
  loc_total(a.loc, run.sums(), tot);
  if (threadIdx.x != 0) return;
  loc_step_solve(s, tot, a.loc.eps_translation, a.loc.eps_rotation, a.loc.corr_dist_fine, a.loc.max_iterations);
}

__global__ void k_rl_final(tloam_rl_args a) {
  if (blockIdx.x >= (unsigned)a.top->n) return;
  loc_final_run<false>(a.loc, RlRun{a, blockIdx.x});
}

// one thread: the winner (the accepted hypothesis minimal by (fitness, rank), else the minimal one), the ambiguity check
// against every other accepted hypothesis, and on acceptance the prediction's memory L = T, O = O_now
__global__ void k_rl_select(tloam_rl_args a) {
  if (threadIdx.x != 0) return;
  tloam_rl_top* top = a.top;
  const int n = top->n;
  int w = -1;
  for (int k = 0; k < n; ++k)
    if (a.states[k].accepted && (w < 0 || a.states[k].fitness < a.states[w].fitness)) w = k;
  if (w < 0)
    for (int k = 0; k < n; ++k)
      if (w < 0 || a.states[k].fitness < a.states[w].fitness) w = k;
  top->winner = w;
  top->ambiguous = 0;
  top->accepted = 0;
  if (w < 0 || !a.states[w].accepted) return;
  const tloam_loc_state* sw = a.states + w;
  const double bound = __dmul_rn(a.ambiguity_ratio, sw->fitness);
  for (int k = 0; k < n; ++k) {
    const tloam_loc_state* sk = a.states + k;
    if (k == w || !sk->accepted || !(sk->fitness <= bound)) continue;
    const double dt = __dsqrt_rn(nf_d2(sk->t[0], sk->t[1], sk->t[2], sw->t[0], sw->t[1], sw->t[2]));
    double tr = 0.0;
    for (int q = 0; q < 9; ++q) tr = __dadd_rn(tr, __dmul_rn(sw->R[q], sk->R[q]));
    const double c = fmin(fmax(__dmul_rn(__dsub_rn(tr, 1.0), 0.5), -1.0), 1.0);
    if (dt > a.distinct_translation || c < a.cos_distinct_rotation) top->ambiguous = 1;
  }
  top->accepted = top->ambiguous ? 0 : 1;
  if (!top->accepted) return;
  for (int r = 0; r < 3; ++r) {
    for (int j = 0; j < 3; ++j) a.loc.memory->L[4 * j + r] = sw->R[3 * r + j];
    a.loc.memory->L[12 + r] = sw->t[r];
    a.loc.memory->L[4 * r + 3] = 0.0;
  }
  a.loc.memory->L[15] = 1.0;
  for (int q = 0; q < 16; ++q) a.loc.memory->O[q] = sw->odom[q];
}

}  // namespace tloam

using namespace tloam;

#define TLOAM_RL_API extern "C" __attribute__((visibility("default")))

TLOAM_RL_API int tloam_rl_run(const tloam_rl_args* a, int* launches) {
  *launches = 0;
  cudaError_t e = cudaSetDevice(a->device);
  if (e != cudaSuccess) return (int)e;
  const int S = a->n_sector;
  const size_t desc = (size_t)a->n_ring * S + S;
  int per_block = S >= (int)kRlT ? 1 : (int)kRlT / S;
  while (per_block > 1 && ((1 + per_block) * desc + (size_t)per_block * S) * sizeof(double) > kRlMaxSmem) --per_block;
  const size_t smem = ((1 + per_block) * desc + (size_t)per_block * S) * sizeof(double);
  const unsigned long long groups = (a->n_places + per_block - 1) / per_block;
  const unsigned grid = (unsigned)(groups < TLOAM_SC_MAX_BLOCKS ? groups : TLOAM_SC_MAX_BLOCKS);
  if (grid) {
    if (smem > 48 * 1024 &&
        (e = cudaFuncSetAttribute(k_rl_search, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess)
      return (int)e;
    k_rl_search<<<grid, kRlT, smem, a->stream>>>(*a, per_block);
    *launches += 1;
  }
  k_rl_topk<<<1, kRlTopT, 0, a->stream>>>(*a);
  k_rl_guess<<<1, TLOAM_RL_MAX_K, 0, a->stream>>>(*a);
  *launches += 2;
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  const unsigned long long nq = a->loc.nq;
  const unsigned K = (unsigned)a->top_k;
  if (nq) {
    const dim3 qg((unsigned)((nq + kLocT - 1) / kLocT), K);
    for (int k = 0; k <= a->loc.max_iterations; ++k) {
      const int fin = k == a->loc.max_iterations;
      k_rl_match<<<qg, kLocT, 0, a->stream>>>(*a, k, fin);
      k_rl_reduce<<<qg, kLocT, 0, a->stream>>>(*a, k, fin);
      if (!fin) k_rl_step<<<K, 32, 0, a->stream>>>(*a);
      *launches += fin ? 2 : 3;
      if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    }
  }
  k_rl_final<<<K, 32, 0, a->stream>>>(*a);
  k_rl_select<<<1, 32, 0, a->stream>>>(*a);
  *launches += 2;
  return (int)cudaGetLastError();
}
