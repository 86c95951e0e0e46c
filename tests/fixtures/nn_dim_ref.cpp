// The matcher's two exact nearest-neighbour searches (feature_matcher.cc's FLANN trees, as this project restates them) for descriptor
// rows of any length: row i of A against every row of B and the reverse, the squared L2 distance being the chain
// acc = fmaf(a_d - b_d, a_d - b_d, acc) over d = 0 .. dim - 1 in ascending order from acc = 0.  Rows are `stride` floats apart and
// their first `dim` floats are the descriptor.  Minima are packed (distance bits << 32 | index), so ties go to the lowest index; a NaN
// distance never wins, and ~0 means no candidate.  Built with -ffp-contract=off -mfma: every fmaf is one fused instruction and no
// other product is fused.
#include <stdint.h>
#include <string.h>

#include <vector>

static inline uint64_t pack(float d, int idx) {
  uint32_t u;
  memcpy(&u, &d, 4);
  return ((uint64_t)u << 32) | (uint32_t)idx;
}

extern "C" int nn_tables_dim(const float* A, int nA, const float* B, int nB, int dim, int stride, uint64_t* bestA, uint64_t* bestB) {
  if (nA < 0 || nB < 0 || dim < 1 || stride < dim) return -1;
  std::vector<float> acc(nB > 0 ? nB : 1);
  for (int j = 0; j < nB; ++j) bestB[j] = ~0ull;
  for (int i = 0; i < nA; ++i) {
    const float* a = A + (size_t)i * stride;
    for (int j = 0; j < nB; ++j) {
      const float* b = B + (size_t)j * stride;
      float s = 0.0f;
      for (int d = 0; d < dim; ++d) {
        const float diff = a[d] - b[d];
        s = __builtin_fmaf(diff, diff, s);
      }
      acc[j] = s;
    }
    uint64_t best = ~0ull;
    for (int j = 0; j < nB; ++j) {
      const float dj = acc[j];
      if (dj != dj) continue;
      const uint64_t kj = pack(dj, j), ki = pack(dj, i);
      if (kj < best) best = kj;
      if (ki < bestB[j]) bestB[j] = ki;
    }
    bestA[i] = best;
  }
  return 0;
}
