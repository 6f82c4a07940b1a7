// scan_context.cuh -- the Scan Context distance of a query descriptor and a candidate at one column shift, and the
// lexicographic order of search results, shared by the loop search (scan_context.cu) and the place search of
// relocalization (relocalize.cu), so that both run the same code and give the same bits.  Device functions only.
#pragma once
#include <cuda_runtime.h>

namespace tloam {

__device__ __forceinline__ bool sc_less(double d1, long long j1, long long s1, double d2, long long j2, long long s2) {
  return d1 < d2 || (d1 == d2 && (j1 < j2 || (j1 == j2 && s1 < s2)));
}

// query bins qb / norms qn against candidate bins cb / norms cn at shift s (R rings, S sectors): candidate column
// (c - s) mod S meets query column c; a column pair counts when both norms are non-zero, and its cosine is (sum over
// rings of a * b) / (|a| * |b|).  The distance is 1 - (sum of the cosines in ascending c) / count, or 1 when no column
// counts.
__device__ __forceinline__ double sc_distance(const double* qb, const double* qn, const double* cb, const double* cn, int R,
                                              int S, int s) {
  double sum = 0.0;
  int count = 0;
  int cc = s == 0 ? 0 : S - s;                           // (c - s) mod S at c = 0
  for (int c = 0; c < S; ++c) {
    const double na = qn[c], nb = cn[cc];
    if (na != 0.0 && nb != 0.0) {
      double dot = 0.0;
      for (int r = 0; r < R; ++r) dot = __dadd_rn(dot, __dmul_rn(qb[r * S + c], cb[r * S + cc]));
      sum = __dadd_rn(sum, __ddiv_rn(dot, __dmul_rn(na, nb)));
      ++count;
    }
    if (++cc == S) cc = 0;
  }
  return count ? __dsub_rn(1.0, __ddiv_rn(sum, (double)count)) : 1.0;
}

}  // namespace tloam
