// =====================================================================================
// quatro_oracle.cpp -- TEST INFRASTRUCTURE.  Deterministic CPU restatement of the reference's
// global-registration hot path (url-kaist/Quatro).  Only tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs may load this library; the product
// (quatro_b200/) never links, imports or calls it.
//
// PARITY UNPINNED: the reference ships no tests, golden vectors or fixtures, and cannot be built
// here (PCL / FLANN / Eigen / pmc / ROS absent, no network; SURVEY.md section 8c).  The heavy
// arithmetic of the reference lives in un-vendored third-party code:
//   PCL >= 1.8 (tested 1.8.1, README.md:70-72): VoxelGrid, NormalEstimation, FPFHEstimationOMP
//   FLANN (1.9.1 on the reference's platform): exact 1-NN, radius search
//   Eigen >= 3.2 (3.3.4): JacobiSVD 2x2
//   pmc  github.com/LimHyungTae/pmc tag libpmc, sha256 64ea6e62...969d (3rdparty/pmc/pmc.cmake:28-29)
// Their published algorithms are restated below ([EXT] marks recalled-from-upstream semantics)
// and anchored on the reference's own call sites.  Pins created by this repo: the known-answer
// tests in tests/test_oracle_kat.py and the golden stage dumps under tests/golden/.
//
// Determinism fixes (each a documented deviation from the literal reference, SURVEY.md 8c):
//   D1 tuple-test RNG: Philox4x32-10(seed, trial) % ncorr replaces srand(time(NULL))/rand()
//      (src/teaser_utils/feature_matcher.cc:189,199-201)
//   D2 nearest-neighbour ties: lowest index; 33-D distance = fmaf chain over d = 0..32
//   D3 stable sorts where the reference's std::sort is unstable on tied keys
//      (include/quatro.hpp:641, pmc's sort of P, PCL VoxelGrid's (key,idx) sort)
//   D4 pmc heuristic runs its start vertices sequentially (reference: 12 racy OpenMP threads,
//      src/graph.cc:39)
//   D5 median COTE: n_card == 1 -> that value, n_card <= 0 -> x_hat (reference: UB, quatro.hpp:714-730)
//   D6 NaN Darboux features -> histogram bin 0 (reference: UB cast, lands on bin 0 on x86)
//   D7 atan2f/acosf/sinf/cosf -> fixed-order float32 kernels of oracle/qo_math.h (< 2 ulp of libm)
//   D8 neighbour accumulation order = ascending (lattice cell (k,j,i), point index); PCL's is
//      kd-tree distance order.  Dot products / norms are evaluated left to right.  The lattice cell defaults to
//      (1 + 2^-9) * fpfh_radius (params.grid_cell overrides it): the neighbour SETS never depend on the cell,
//      the accumulation order does, so the CUDA library uses the same default.
//   D9 2x2 rotation: own two-sided Jacobi SVD (Eigen::JacobiSVD unavailable); fp64 sums in index order
//   D10 VoxelGrid refuses a cloud (QB200_ERR_VOXEL_OVERFLOW, input returned unfiltered) not only on PCL's own check
//      (truncated spans dx*dy*dz > INT_MAX) but wherever PCL's int arithmetic would overflow (UB, wraps in practice): a kept
//      point's floor(p * inv) outside int32, a product of the floor-based div_b above INT_MAX, or a largest linear index above
//      INT_MAX (PCL subtracts floor(p * inv) - min_b in float, which can round ijk up to div_b, so the index can exceed the product)
//   D18 KCORE_HEU limit (int)(kcore_heuristic_threshold * n) (src/graph.cc:69-70): undefined for NaN and out-of-range products; both
//      sides compute what x86-64's cvttsd2si gives, INT_MIN, through qb_kcore_heu_limit (quatro_b200/csrc/kcore_cutoff.cuh)
//   D19 radii are float32 (qb200_params, qb200_compute_fpfh): the squared radius is float(double(r) * double(r)) of the float radius,
//      which equals float(r * r); PCL receives the reference's radii as doubles, and for 0.1 or 1/3 the float of the double square is
//      one ulp lower, so a neighbour at exactly that d2 is kept here and dropped by PCL (tests/test_fpfh_adversarial.py)
// =====================================================================================
#include <algorithm>
#include <cfloat>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <numeric>
#include <utility>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "../include/quatro_b200.h"
#include "qo_math.h"
#include "../quatro_b200/csrc/kcore_cutoff.cuh"

namespace {

struct P4 {
  float x, y, z, w;
};

inline bool finite3(const P4& p) { return std::isfinite(p.x) && std::isfinite(p.y) && std::isfinite(p.z); }

// LITERAL mode (qo_set_literal): undo the determinism fixes D3 and D8 where the literal behaviour of the reference's libraries can
// be reproduced with this toolchain -- libstdc++'s unstable std::sort on tied keys (VoxelGrid's (voxel, point) sort, pmc's sort of
// P, the COTE event sort of quatro.hpp:641) and PCL's distance-ordered neighbour accumulation (KdTreeFLANN returns sorted radius
// results).  It exists only to MEASURE how far "bit-exact with the canonical oracle" can be from the literal reference
// (tests/test_literal_mode.py); the CUDA library is compared with the canonical mode.
int g_literal = 0;

// ---------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al., SC'11), counter = (ctr_lo, ctr_hi, 0, 0), key = (seed_lo, seed_hi)
// ---------------------------------------------------------------------------------------------
inline void philox4x32_10(uint64_t seed, uint64_t ctr, uint32_t out[4]) {
  uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32), c2 = 0, c3 = 0;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0;
    const uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
    const uint32_t n1 = (uint32_t)p1;
    const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    const uint32_t n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// ---------------------------------------------------------------------------------------------
// a1. voxelize -- include/quatro.hpp:49-57 -> [EXT] pcl::VoxelGrid<PointXYZ>::applyFilter (1.8.1)
// ---------------------------------------------------------------------------------------------
int voxelize(const P4* pts, int n, float leaf, int skip_flagged, std::vector<P4>& out) {
  out.clear();
  const float inv = 1.0f / leaf;  // inverse_leaf_size_ = Array4f::Ones() / leaf_size_.array()
  // getMinMax3D over the points the filter keeps
  float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  std::vector<int> kept;
  kept.reserve(n);
  for (int i = 0; i < n; ++i) {
    const P4& p = pts[i];
    if (!finite3(p)) continue;
    if (skip_flagged && p.w < 0.0f) continue;
    kept.push_back(i);
    mn[0] = std::min(mn[0], p.x); mn[1] = std::min(mn[1], p.y); mn[2] = std::min(mn[2], p.z);
    mx[0] = std::max(mx[0], p.x); mx[1] = std::max(mx[1], p.y); mx[2] = std::max(mx[2], p.z);
  }
  if (kept.empty()) return QB200_OK;
  // overflow check: PCL warns and copies the input through.  D10: also refused wherever PCL's own int arithmetic would overflow
  // (a floor(p * inv) outside int32 -- the bbox corners decide, floor(p * inv) is monotone in p --, a product of the floor-based
  // div_b above INT_MAX, or a largest linear index above INT_MAX), and PCL's int64 span product is evaluated without overflowing.
  const int64_t lim = std::numeric_limits<int32_t>::max();
  const auto product_exceeds = [lim](int64_t a, int64_t b, int64_t c) {  // factors >= 1
    return a > lim || b > lim || c > lim || a * b > lim || a * b * c > lim;
  };
  bool refuse = false;
  int64_t span[3], min_b[3], div_b[3], top[3];
  for (int a = 0; a < 3; ++a) {
    const float lo = std::floor(mn[a] * inv), hi = std::floor(mx[a] * inv);
    const float s = (mx[a] - mn[a]) * inv;
    if (!(lo >= -2147483648.0f && hi < 2147483648.0f && s < 2147483648.0f)) { refuse = true; break; }
    span[a] = (int64_t)s + 1;
    min_b[a] = (int64_t)lo;
    div_b[a] = (int64_t)hi - min_b[a] + 1;
    top[a] = (int64_t)(hi - lo);  // the largest ijk of the axis: PCL's float subtraction rounds monotonically, the max corner decides
  }
  // top[a] <= 2^31 (fl(hi - lo) can round up to 2^31) and the div_b product is within INT_MAX: every term below is <= 2^62
  if (refuse || product_exceeds(span[0], span[1], span[2]) || product_exceeds(div_b[0], div_b[1], div_b[2]) ||
      top[0] + top[1] * div_b[0] + top[2] * div_b[0] * div_b[1] > lim) {
    for (int i : kept) out.push_back(pts[i]);
    return QB200_ERR_VOXEL_OVERFLOW;
  }
  const int64_t mul[3] = {1, div_b[0], div_b[0] * div_b[1]};
  std::vector<std::pair<int, int>> iv;  // (voxel idx, point idx)
  iv.reserve(kept.size());
  for (int i : kept) {
    const P4& p = pts[i];
    const int ijk0 = (int)(std::floor(p.x * inv) - (float)min_b[0]);
    const int ijk1 = (int)(std::floor(p.y * inv) - (float)min_b[1]);
    const int ijk2 = (int)(std::floor(p.z * inv) - (float)min_b[2]);
    iv.emplace_back((int)(ijk0 * mul[0] + ijk1 * mul[1] + ijk2 * mul[2]), i);  // <= the largest index, so it fits an int
  }
  const auto by_voxel = [](const std::pair<int, int>& a, const std::pair<int, int>& b) { return a.first < b.first; };
  if (g_literal) std::sort(iv.begin(), iv.end(), by_voxel);  // [EXT] PCL: std::sort with operator< on the voxel index only
  else std::stable_sort(iv.begin(), iv.end(), by_voxel);      // D3
  size_t first = 0;
  while (first < iv.size()) {
    size_t last = first + 1;
    while (last < iv.size() && iv[last].first == iv[first].first) ++last;
    float sx = 0.f, sy = 0.f, sz = 0.f;  // CentroidPoint<PointXYZ>: float accumulators, xyz / n
    for (size_t t = first; t < last; ++t) {
      const P4& p = pts[iv[t].second];
      sx += p.x; sy += p.y; sz += p.z;
    }
    const float cnt = (float)(last - first);
    out.push_back(P4{sx / cnt, sy / cnt, sz / cnt, 1.0f});
    first = last;
  }
  return QB200_OK;
}

// ---------------------------------------------------------------------------------------------
// Neighbour lattice (stands in for pcl::search::KdTree / FLANN radius search, fpfh.cc:58-72).
// Neighbour SET = {q : ((dx*dx + dy*dy) + dz*dz) < float(r*r)} incl. the query itself
// ([EXT] flann::L2_Simple, strict '<' in RadiusResultSet); ORDER = ascending (cell key, index)  (D8).
// ---------------------------------------------------------------------------------------------
constexpr int kOffIJ = 1 << 17, kOffK = 1 << 15;
inline bool cell_ok(int i, int j, int k) {
  // the all-ones cell value is reserved (device sort keys use it as the "dropped point" marker)
  return i >= -kOffIJ && i < kOffIJ - 1 && j >= -kOffIJ && j < kOffIJ - 1 && k >= -kOffK && k < kOffK - 1;
}
inline uint64_t cell_key(int i, int j, int k) {
  return ((uint64_t)(k + kOffK) << 36) | ((uint64_t)(j + kOffIJ) << 18) | (uint64_t)(i + kOffIJ);
}

struct Lattice {
  float inv = 1.f;
  std::vector<uint64_t> ckeys;   // unique occupied cells, ascending
  std::vector<int> cstart;       // ckeys.size()+1
  std::vector<int> order;        // point indices sorted by (cell key, index)
  std::vector<int> ci, cj, ck;   // per point cell coords (valid only if in lattice)
  std::vector<uint8_t> in;       // per point: in lattice

  void build(const P4* pts, int n, float cell) {
    inv = 1.0f / cell;
    ci.assign(n, 0); cj.assign(n, 0); ck.assign(n, 0); in.assign(n, 0);
    std::vector<std::pair<uint64_t, int>> kv;
    kv.reserve(n);
    for (int p = 0; p < n; ++p) {
      if (!finite3(pts[p])) continue;
      const int i = (int)std::floor(pts[p].x * inv), j = (int)std::floor(pts[p].y * inv),
                k = (int)std::floor(pts[p].z * inv);
      if (!cell_ok(i, j, k)) continue;
      ci[p] = i; cj[p] = j; ck[p] = k; in[p] = 1;
      kv.emplace_back(cell_key(i, j, k), p);
    }
    std::sort(kv.begin(), kv.end());  // (key, index) pairs are unique -> total order
    order.resize(kv.size());
    ckeys.clear(); cstart.clear();
    for (size_t t = 0; t < kv.size(); ++t) {
      order[t] = kv[t].second;
      if (t == 0 || kv[t].first != kv[t - 1].first) {
        ckeys.push_back(kv[t].first);
        cstart.push_back((int)t);
      }
    }
    cstart.push_back((int)kv.size());
  }

  static int reach(float radius, float inv) { return (int)std::ceil(radius * inv + 1e-3f); }

  // f(index, dist2) in canonical order ((cell, index), D8); literal mode: ascending distance like a sorted FLANN radius search
  template <class F>
  void for_each_neighbor(const P4* pts, int q, float radius, F&& f) const {
    if (!in[q]) return;
    if (g_literal) {
      std::vector<std::pair<float, int>> found;
      walk(pts, q, radius, [&](int p, float d2) { found.emplace_back(d2, p); });
      std::sort(found.begin(), found.end());
      for (const auto& e : found) f(e.second, e.first);
      return;
    }
    walk(pts, q, radius, f);
  }
  template <class F>
  void walk(const P4* pts, int q, float radius, F&& f) const {
    const int m = reach(radius, inv);
    const float r2 = (float)((double)radius * (double)radius);
    const P4& pq = pts[q];
    for (int dk = -m; dk <= m; ++dk) {
      for (int dj = -m; dj <= m; ++dj) {
        const int k = ck[q] + dk, j = cj[q] + dj;
        int ilo = ci[q] - m, ihi = ci[q] + m;
        if (k < -kOffK || k >= kOffK - 1 || j < -kOffIJ || j >= kOffIJ - 1) continue;
        ilo = std::max(ilo, -kOffIJ); ihi = std::min(ihi, kOffIJ - 2);
        const uint64_t lo = cell_key(ilo, j, k), hi = cell_key(ihi, j, k);
        size_t c = std::lower_bound(ckeys.begin(), ckeys.end(), lo) - ckeys.begin();
        for (; c < ckeys.size() && ckeys[c] <= hi; ++c) {
          for (int t = cstart[c]; t < cstart[c + 1]; ++t) {
            const int p = order[t];
            const float dx = pq.x - pts[p].x, dy = pq.y - pts[p].y, dz = pq.z - pts[p].z;
            const float d2 = (dx * dx + dy * dy) + dz * dz;
            if (d2 < r2) f(p, d2);
          }
        }
      }
    }
  }
};

// ---------------------------------------------------------------------------------------------
// a3 (normals). [EXT] pcl::NormalEstimation::computeFeature -> computePointNormal ->
// computeMeanAndCovarianceMatrix (single-pass float, PCL 1.8.1) -> solvePlaneParameters ->
// pcl::eigen33 / computeRoots; flipNormalTowardsViewpoint with vp = (0,0,0).   fpfh.cc:58-63
// ---------------------------------------------------------------------------------------------
inline void compute_roots2(float b, float c, float roots[3]) {
  roots[0] = 0.0f;
  float d = (float)((double)(b * b) - 4.0 * (double)c);
  if (d < 0.0f) d = 0.0f;
  const float sd = sqrtf(d);
  roots[2] = 0.5f * (b + sd);
  roots[1] = 0.5f * (b - sd);
}

inline void compute_roots(const float m[9], float roots[3]) {
  const float m00 = m[0], m01 = m[1], m02 = m[2], m11 = m[4], m12 = m[5], m22 = m[8];
  const float c0 = m00 * m11 * m22 + 2.0f * m01 * m02 * m12 - m00 * m12 * m12 - m11 * m02 * m02 - m22 * m01 * m01;
  const float c1 = m00 * m11 - m01 * m01 + m00 * m22 - m02 * m02 + m11 * m22 - m12 * m12;
  const float c2 = m00 + m11 + m22;
  if (fabsf(c0) < FLT_EPSILON) {
    compute_roots2(c2, c1, roots);
    return;
  }
  const float s_inv3 = (float)(1.0 / 3.0);
  const float s_sqrt3 = sqrtf(3.0f);
  const float c2_over_3 = c2 * s_inv3;
  float a_over_3 = (c1 - c2 * c2_over_3) * s_inv3;
  if (a_over_3 > 0.0f) a_over_3 = 0.0f;
  const float half_b = 0.5f * (c0 + c2_over_3 * (2.0f * c2_over_3 * c2_over_3 - c1));
  float q = half_b * half_b + a_over_3 * a_over_3 * a_over_3;
  if (q > 0.0f) q = 0.0f;
  const float rho = sqrtf(-a_over_3);
  const float theta = qo_atan2f(sqrtf(-q), half_b) * s_inv3;  // D7
  float sin_theta, cos_theta;
  qo_sincosf(theta, &sin_theta, &cos_theta);                  // D7
  roots[0] = c2_over_3 + 2.0f * rho * cos_theta;
  roots[1] = c2_over_3 - rho * (cos_theta + s_sqrt3 * sin_theta);
  roots[2] = c2_over_3 - rho * (cos_theta - s_sqrt3 * sin_theta);
  if (roots[0] >= roots[1]) std::swap(roots[0], roots[1]);
  if (roots[1] >= roots[2]) {
    std::swap(roots[1], roots[2]);
    if (roots[0] >= roots[1]) std::swap(roots[0], roots[1]);
  }
  if (roots[0] <= 0.0f) compute_roots2(c2, c1, roots);
}

inline void cross3(const float a[3], const float b[3], float o[3]) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}
inline float dot3(const float a[3], const float b[3]) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

// smallest eigenvalue / eigenvector of a symmetric 3x3 (row-major m[9])
inline void eigen33_smallest(const float cov[9], float* eigenvalue, float evec[3]) {
  float scale = 0.0f;
  for (int i = 0; i < 9; ++i) scale = std::max(scale, fabsf(cov[i]));
  if (!(scale > FLT_MIN)) scale = 1.0f;  // also catches NaN like cwiseAbs().maxCoeff() <= min
  float s[9];
  for (int i = 0; i < 9; ++i) s[i] = cov[i] / scale;
  float roots[3];
  compute_roots(s, roots);
  *eigenvalue = roots[0] * scale;
  s[0] -= roots[0]; s[4] -= roots[0]; s[8] -= roots[0];
  float v1[3], v2[3], v3[3];
  cross3(&s[0], &s[3], v1);
  cross3(&s[0], &s[6], v2);
  cross3(&s[3], &s[6], v3);
  const float l1 = dot3(v1, v1), l2 = dot3(v2, v2), l3 = dot3(v3, v3);
  const float* v; float l;
  if (l1 >= l2 && l1 >= l3) { v = v1; l = l1; }
  else if (l2 >= l1 && l2 >= l3) { v = v2; l = l2; }
  else { v = v3; l = l3; }
  const float sl = sqrtf(l);
  evec[0] = v[0] / sl; evec[1] = v[1] / sl; evec[2] = v[2] / sl;
}

// covariance sums -> normal + curvature (computeMeanAndCovarianceMatrix tail, solvePlaneParameters, flip)
inline P4 normal_from_accu(float accu[9], int cnt, const P4& pq) {
  P4 nn{NAN, NAN, NAN, NAN};
  if (cnt >= 3) {
    const float fc = (float)cnt;
    for (int i = 0; i < 9; ++i) accu[i] /= fc;
    float cov[9];
    cov[0] = accu[0] - accu[6] * accu[6];
    cov[1] = accu[1] - accu[6] * accu[7];
    cov[2] = accu[2] - accu[6] * accu[8];
    cov[4] = accu[3] - accu[7] * accu[7];
    cov[5] = accu[4] - accu[7] * accu[8];
    cov[8] = accu[5] - accu[8] * accu[8];
    cov[3] = cov[1]; cov[6] = cov[2]; cov[7] = cov[5];
    float ev, e[3];
    eigen33_smallest(cov, &ev, e);
    const float eig_sum = cov[0] + cov[4] + cov[8];
    const float curv = (eig_sum != 0.0f) ? fabsf(ev / eig_sum) : 0.0f;
    // flipNormalTowardsViewpoint, vp = 0
    const float vx = 0.0f - pq.x, vy = 0.0f - pq.y, vz = 0.0f - pq.z;
    const float cos_theta = (vx * e[0] + vy * e[1]) + vz * e[2];
    if (cos_theta < 0.0f) { e[0] *= -1.0f; e[1] *= -1.0f; e[2] *= -1.0f; }
    nn = P4{e[0], e[1], e[2], curv};
  }
  return nn;
}

void compute_normals(const P4* pts, int n, const Lattice& lat, float radius, P4* normals) {
#pragma omp parallel for schedule(dynamic, 64)
  for (int q = 0; q < n; ++q) {
    float accu[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    int cnt = 0;
    lat.for_each_neighbor(pts, q, radius, [&](int p, float) {
      const float x = pts[p].x, y = pts[p].y, z = pts[p].z;
      accu[0] += x * x; accu[1] += x * y; accu[2] += x * z;
      accu[3] += y * y; accu[4] += y * z; accu[5] += z * z;
      accu[6] += x; accu[7] += y; accu[8] += z;
      ++cnt;
    });
    normals[q] = normal_from_accu(accu, cnt, pts[q]);
  }
}

// ---------------------------------------------------------------------------------------------
// a3 (FPFH). [EXT] pcl::computePairFeatures, FPFHEstimation::computePointSPFHSignature,
// weightPointSPFHSignature (PCL 1.8.1), driven by fpfh.cc:68-72.
// ---------------------------------------------------------------------------------------------
inline bool pair_features(const P4& p1, const P4& n1, const P4& p2, const P4& n2, float& f1, float& f2, float& f3) {
  float dp[3] = {p2.x - p1.x, p2.y - p1.y, p2.z - p1.z};
  const float f4 = sqrtf(dot3(dp, dp));
  if (f4 == 0.0f) return false;
  float n1c[3] = {n1.x, n1.y, n1.z}, n2c[3] = {n2.x, n2.y, n2.z};
  const float angle1 = dot3(n1c, dp) / f4;
  const float angle2 = dot3(n2c, dp) / f4;
  if (qo_acosf(fabsf(angle1)) > qo_acosf(fabsf(angle2))) {  // D7
    std::swap(n1c[0], n2c[0]); std::swap(n1c[1], n2c[1]); std::swap(n1c[2], n2c[2]);
    dp[0] *= -1.0f; dp[1] *= -1.0f; dp[2] *= -1.0f;
    f3 = -angle2;
  } else {
    f3 = angle1;
  }
  float v[3];
  cross3(dp, n1c, v);
  const float v_norm = sqrtf(dot3(v, v));
  if (v_norm == 0.0f) return false;
  v[0] /= v_norm; v[1] /= v_norm; v[2] /= v_norm;
  float w[3];
  cross3(n1c, v, w);
  f2 = dot3(v, n2c);
  f1 = qo_atan2f(dot3(w, n2c), dot3(n1c, n2c));  // D7
  return true;
}

inline int bin_of(double scaled) {  // scaled = nr_bins * normalised feature
  if (scaled != scaled) return 0;   // D6
  int h = (int)std::floor(scaled);
  if (h < 0) h = 0;
  if (h >= 11) h = 10;
  return h;
}

void compute_spfh(const P4* pts, const P4* normals, int n, const Lattice& lat, float radius, float* spfh /* n x 33 */) {
  const float d_pi = 1.0f / (2.0f * (float)M_PI);
#pragma omp parallel for schedule(dynamic, 64)
  for (int q = 0; q < n; ++q) {
    float* h = spfh + (size_t)q * 33;
    for (int b = 0; b < 33; ++b) h[b] = 0.0f;
    int k = 0;
    lat.for_each_neighbor(pts, q, radius, [&](int, float) { ++k; });
    if (k < 2) continue;
    const float incr = 100.0f / (float)(k - 1);
    lat.for_each_neighbor(pts, q, radius, [&](int p, float) {
      if (p == q) return;
      float f1, f2, f3;
      if (!pair_features(pts[q], normals[q], pts[p], normals[p], f1, f2, f3)) return;
      h[bin_of(11 * (((double)f1 + M_PI) * (double)d_pi))] += incr;
      h[11 + bin_of(11 * (((double)f2 + 1.0) * 0.5))] += incr;
      h[22 + bin_of(11 * (((double)f3 + 1.0) * 0.5))] += incr;
    });
  }
}

void compute_fpfh(const P4* pts, int n, const Lattice& lat, float radius, const float* spfh, float* fpfh /* n x 33 */) {
#pragma omp parallel for schedule(dynamic, 64)
  for (int q = 0; q < n; ++q) {
    float* o = fpfh + (size_t)q * 33;
    for (int b = 0; b < 33; ++b) o[b] = 0.0f;
    double sum[3] = {0.0, 0.0, 0.0};
    lat.for_each_neighbor(pts, q, radius, [&](int p, float d2) {
      if (d2 == 0.0f) return;  // "minus the query point itself"
      const float weight = 1.0f / d2;
      const float* s = spfh + (size_t)p * 33;
      for (int t = 0; t < 3; ++t)
        for (int b = 0; b < 11; ++b) {
          const float val = s[t * 11 + b] * weight;
          sum[t] += val;
          o[t * 11 + b] += val;
        }
    });
    for (int t = 0; t < 3; ++t) {
      if (sum[t] != 0.0) sum[t] = 100.0 / sum[t];
      const float f = (float)sum[t];
      for (int b = 0; b < 11; ++b) o[t * 11 + b] *= f;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// a4-a7. Matcher::calculateCorrespondences / normalizePoints / advancedMatching
// include/teaser_utils/feature_matcher.h:42-74, src/teaser_utils/feature_matcher.cc:18-265
// ---------------------------------------------------------------------------------------------
struct MatchOut {
  std::vector<std::pair<int, int>> mutual;  // (i in larger cloud fi, j in smaller fj), ascending i
  std::vector<std::pair<int, int>> corr;    // (src, tgt) sorted unique
  bool swapped = false;
};

// D2: squared L2 as a fused-multiply-add chain over d = 0..32
inline uint64_t pack_dist(float d, int idx) {
  uint32_t u;
  memcpy(&u, &d, 4);
  return ((uint64_t)u << 32) | (uint32_t)idx;
}

// packA / packB (optional): the packed (distance bits << 32 | index) minima themselves, ~0 = no candidate
void nn_both_ways(const float* A, int nA, const float* B, int nB, std::vector<int>& nnA /* per A row: argmin B */,
                  std::vector<int>& nnB /* per B row: argmin A */, uint64_t* packA = nullptr, uint64_t* packB = nullptr) {
  // B transposed so the inner loop runs over candidates
  std::vector<float> Bt((size_t)33 * nB);
  for (int j = 0; j < nB; ++j)
    for (int d = 0; d < 33; ++d) Bt[(size_t)d * nB + j] = B[(size_t)j * 33 + d];
  nnA.assign(nA, -1);
  std::vector<uint64_t> bestB(nB, ~0ull);
#pragma omp parallel
  {
    std::vector<float> acc(nB);
    std::vector<uint64_t> myB(nB, ~0ull);
#pragma omp for schedule(static)
    for (int i = 0; i < nA; ++i) {
      std::fill(acc.begin(), acc.end(), 0.0f);
      const float* a = A + (size_t)i * 33;
      for (int d = 0; d < 33; ++d) {
        const float ad = a[d];
        const float* bt = &Bt[(size_t)d * nB];
        for (int j = 0; j < nB; ++j) {
          const float diff = ad - bt[j];
          acc[j] = __builtin_fmaf(diff, diff, acc[j]);
        }
      }
      uint64_t best = ~0ull;
      for (int j = 0; j < nB; ++j) {
        const float dj = acc[j];
        if (dj != dj) continue;  // NaN never wins
        const uint64_t kj = pack_dist(dj, j);
        if (kj < best) best = kj;
        const uint64_t ki = pack_dist(dj, i);
        if (ki < myB[j]) myB[j] = ki;
      }
      nnA[i] = best == ~0ull ? -1 : (int)(uint32_t)best;
      if (packA) packA[i] = best;
    }
#pragma omp critical
    for (int j = 0; j < nB; ++j)
      if (myB[j] < bestB[j]) bestB[j] = myB[j];
  }
  nnB.assign(nB, -1);
  for (int j = 0; j < nB; ++j) nnB[j] = bestB[j] == ~0ull ? -1 : (int)(uint32_t)bestB[j];
  if (packB) std::copy(bestB.begin(), bestB.end(), packB);
}

void center_points(const P4* pts, int n, std::vector<float>& out /* n x 3 */) {
  // normalizePoints(use_absolute_scale = true): subtract the float mean, scale stays 1
  float mx = 0.f, my = 0.f, mz = 0.f;
  for (int i = 0; i < n; ++i) { mx = mx + pts[i].x; my = my + pts[i].y; mz = mz + pts[i].z; }
  const float fn = (float)n;
  mx = mx / fn; my = my / fn; mz = mz / fn;
  out.resize((size_t)n * 3);
  for (int i = 0; i < n; ++i) {
    out[3 * i + 0] = pts[i].x - mx; out[3 * i + 1] = pts[i].y - my; out[3 * i + 2] = pts[i].z - mz;
  }
}

inline float side(const float* c, int a, int b) {
  const float dx = c[3 * a] - c[3 * b], dy = c[3 * a + 1] - c[3 * b + 1], dz = c[3 * a + 2] - c[3 * b + 2];
  return sqrtf((dx * dx + dy * dy) + dz * dz);
}

int match(const P4* src, int n_src, const float* sdesc, const P4* tgt, int n_tgt, const float* tdesc,
          const qb200_params& prm, MatchOut& mo) {
  mo = MatchOut();
  if (!prm.use_crosscheck) return QB200_ERR_UNSUPPORTED;
  if (n_src <= 0 || n_tgt <= 0) return QB200_OK;
  // fi = larger cloud (source on ties), fj = smaller: feature_matcher.cc:79-92
  mo.swapped = n_tgt > n_src;
  const P4* pi = mo.swapped ? tgt : src; const P4* pj = mo.swapped ? src : tgt;
  const float* fi = mo.swapped ? tdesc : sdesc; const float* fj = mo.swapped ? sdesc : tdesc;
  const int nPti = mo.swapped ? n_tgt : n_src, nPtj = mo.swapped ? n_src : n_tgt;
  std::vector<int> nn_i, nn_j;  // nn_i[i] = NN in fj of feature i;  nn_j[j] = NN in fi of feature j
  nn_both_ways(fi, nPti, fj, nPtj, nn_i, nn_j);
  // initial matching + cross check (:115-177) == mutual nearest neighbours, ascending i
  for (int i = 0; i < nPti; ++i) {
    const int j = nn_i[i];
    if (j >= 0 && nn_j[j] == i) mo.mutual.emplace_back(i, j);
  }
  std::vector<std::pair<int, int>> corres = mo.mutual;
  // tuple constraint (:187-247)
  if (prm.use_tuple_test && prm.tuple_scale != 0.0f && !corres.empty()) {
    std::vector<float> ci, cj;
    center_points(pi, nPti, ci);
    center_points(pj, nPtj, cj);
    const float scale = prm.tuple_scale;
    const int ncorr = (int)corres.size();
    const int64_t trials = (int64_t)ncorr * prm.tuple_trials_per_corr;
    std::vector<uint8_t> mark(ncorr, 0);
#pragma omp parallel for schedule(static)
    for (int64_t t = 0; t < trials; ++t) {
      uint32_t r[4];
      philox4x32_10(prm.seed, (uint64_t)t, r);  // D1
      const int r0 = (int)(r[0] % (uint32_t)ncorr), r1 = (int)(r[1] % (uint32_t)ncorr), r2 = (int)(r[2] % (uint32_t)ncorr);
      const int idi0 = corres[r0].first, idj0 = corres[r0].second;
      const int idi1 = corres[r1].first, idj1 = corres[r1].second;
      const int idi2 = corres[r2].first, idj2 = corres[r2].second;
      const float li0 = side(ci.data(), idi0, idi1), li1 = side(ci.data(), idi1, idi2), li2 = side(ci.data(), idi2, idi0);
      const float lj0 = side(cj.data(), idj0, idj1), lj1 = side(cj.data(), idj1, idj2), lj2 = side(cj.data(), idj2, idj0);
      if ((li0 * scale < lj0) && (lj0 < li0 / scale) && (li1 * scale < lj1) && (lj1 < li1 / scale) &&
          (li2 * scale < lj2) && (lj2 < li2 / scale)) {
        mark[r0] = 1; mark[r1] = 1; mark[r2] = 1;  // benign race: all writers store 1
      }
    }
    std::vector<std::pair<int, int>> kept;
    for (int c = 0; c < ncorr; ++c)
      if (mark[c]) kept.push_back(corres[c]);
    corres.swap(kept);
  }
  // swap back, sort, unique (:249-264)
  if (mo.swapped)
    for (auto& c : corres) std::swap(c.first, c.second);
  std::sort(corres.begin(), corres.end());
  corres.erase(std::unique(corres.begin(), corres.end()), corres.end());
  mo.corr.swap(corres);
  return QB200_OK;
}

// ---------------------------------------------------------------------------------------------
// a9-a11. computeTIMs + solveForScale + inlier graph   include/quatro.hpp:307-386, 784-789
// The TIMs are never materialised: edge(i,j), i<j, is the literal fp64 mask expression.
// ---------------------------------------------------------------------------------------------
inline bool tim_consistent(const P4& ai, const P4& aj, const P4& bi, const P4& bj, double beta) {
  const double ax = (double)aj.x - (double)ai.x, ay = (double)aj.y - (double)ai.y, az = (double)aj.z - (double)ai.z;
  const double bx = (double)bj.x - (double)bi.x, by = (double)bj.y - (double)bi.y, bz = (double)bj.z - (double)bi.z;
  const double v1 = std::sqrt(ax * ax + ay * ay + az * az);  // src TIM norm
  const double v2 = std::sqrt(bx * bx + by * by + bz * bz);  // dst TIM norm
  const double alpha_f = beta * (1.0 / v1);
  const double raw_f = v2 / v1;
  const bool in_f = std::fabs(raw_f - 1.0) <= alpha_f;
  const double alpha_r = beta * (1.0 / v2);
  const double raw_r = v1 / v2;
  const bool in_r = std::fabs(raw_r - 1.0) <= alpha_r;
  return in_f && in_r;
}

void build_graph(const P4* a, const P4* b, int L, double noise_bound, double cbar2, uint32_t* adj, int wpr,
                 int* degree, int64_t* n_edges) {
  const double beta = 2 * noise_bound * std::sqrt(cbar2);
  std::memset(adj, 0, (size_t)L * wpr * sizeof(uint32_t));
  // upper triangle in parallel (row i only writes bits j>i of row i), mirror afterwards
#pragma omp parallel for schedule(dynamic, 16)
  for (int i = 0; i < L; ++i)
    for (int j = i + 1; j < L; ++j)
      if (tim_consistent(a[i], a[j], b[i], b[j], beta)) adj[(size_t)i * wpr + (j >> 5)] |= 1u << (j & 31);
  int64_t e = 0;
  for (int i = 0; i < L; ++i)
    for (int j = i + 1; j < L; ++j)
      if (adj[(size_t)i * wpr + (j >> 5)] >> (j & 31) & 1u) {
        adj[(size_t)j * wpr + (i >> 5)] |= 1u << (i & 31);
        ++e;
      }
  if (degree)
    for (int i = 0; i < L; ++i) {
      int d = 0;
      for (int w = 0; w < wpr; ++w) d += __builtin_popcount(adj[(size_t)i * wpr + w]);
      degree[i] = d;
    }
  if (n_edges) *n_edges = e;
}

// ---------------------------------------------------------------------------------------------
// a12. MaxCliqueSolver::findMaxClique   src/graph.cc:12-130  -> [EXT] pmc
// ---------------------------------------------------------------------------------------------
struct Csr {
  std::vector<int64_t> vertices;  // L+1
  std::vector<int> edges;         // ascending per row (graph.h:96-104 insertion order)
};

Csr to_csr(const uint32_t* adj, int L, int wpr) {
  Csr g;
  g.vertices.push_back(0);
  for (int i = 0; i < L; ++i) {
    for (int w = 0; w < wpr; ++w) {
      uint32_t x = adj[(size_t)i * wpr + w];
      while (x) {
        const int b = __builtin_ctz(x);
        x &= x - 1;
        const int j = w * 32 + b;
        if (j < L) g.edges.push_back(j);
      }
    }
    g.vertices.push_back((int64_t)g.edges.size());
  }
  return g;
}

// [EXT] pmc_graph::compute_cores -- Batagelj-Zaversnik, restated 0-based.
// Returns kcore[v] = core(v) + 1 (pmc's "K+1"), kcore_order = peel order, max_core = max core number.
void compute_cores(const Csr& g, std::vector<int>& kcore, std::vector<int>& order, int& max_core) {
  const int n = (int)g.vertices.size() - 1;
  kcore.assign(n, 0); order.assign(n, 0);
  max_core = 0;
  if (n == 0) return;
  std::vector<int> pos(n), deg(n);
  int md = 0;
  for (int v = 0; v < n; ++v) {
    deg[v] = (int)(g.vertices[v + 1] - g.vertices[v]);
    md = std::max(md, deg[v]);
  }
  std::vector<int> bin(md + 2, 0);
  for (int v = 0; v < n; ++v) bin[deg[v]]++;
  int start = 0;
  for (int d = 0; d <= md; ++d) { const int num = bin[d]; bin[d] = start; start += num; }
  for (int v = 0; v < n; ++v) { pos[v] = bin[deg[v]]; order[pos[v]] = v; bin[deg[v]]++; }
  for (int d = md; d >= 1; --d) bin[d] = bin[d - 1];
  bin[0] = 0;
  for (int i = 0; i < n; ++i) {
    const int v = order[i];
    for (int64_t e = g.vertices[v]; e < g.vertices[v + 1]; ++e) {
      const int u = g.edges[e];
      if (deg[u] > deg[v]) {
        const int du = deg[u], pu = pos[u], pw = bin[du], w = order[pw];
        if (u != w) { pos[u] = pw; order[pu] = w; pos[w] = pu; order[pw] = u; }
        bin[du]++; deg[u]--;
      }
    }
  }
  for (int v = 0; v < n; ++v) kcore[v] = deg[v] + 1;
  max_core = deg[order[n - 1]];
}

// [EXT] pmc_heu::search_bounds / branch with heu_strat = "kcore", sequential start order (D4),
// stable sort of P (D3).  Returns mc; C_max in pmc's push order.
int pmc_heuristic(const Csr& g, const std::vector<int>& K, const std::vector<int>& order, int ub, std::vector<int>& C_max) {
  const int n = (int)order.size();
  int mc = 0;
  C_max.clear();
  std::vector<uint8_t> ind(n, 0);
  std::vector<std::pair<int, int>> P, R;  // (id, bound)
  for (int i = n - 1; i >= 0; --i) {
    if (mc >= ub) break;  // found_ub
    const int v = order[i];
    if (K[v] <= mc) continue;
    P.clear();
    for (int64_t e = g.vertices[v]; e < g.vertices[v + 1]; ++e) {
      const int u = g.edges[e];
      if (K[u] > mc) P.emplace_back(u, K[u]);
    }
    if ((int)P.size() <= mc) continue;
    const auto by_bound = [](const std::pair<int, int>& a, const std::pair<int, int>& b) { return a.second < b.second; };
    if (g_literal) std::sort(P.begin(), P.end(), by_bound);
    else std::stable_sort(P.begin(), P.end(), by_bound);
    // branch(): a single greedy descent, no backtracking
    std::vector<int> popped;
    int sz = 1;
    while (!P.empty()) {
      const int u = P.back().first;
      P.pop_back();
      popped.push_back(u);
      for (int64_t e = g.vertices[u]; e < g.vertices[u + 1]; ++e) ind[g.edges[e]] = 1;
      R.clear();
      for (const auto& p : P)
        if (ind[p.first] && K[p.first] > mc) R.push_back(p);
      for (int64_t e = g.vertices[u]; e < g.vertices[u + 1]; ++e) ind[g.edges[e]] = 0;
      P.swap(R);
      ++sz;
    }
    if (sz > mc) {
      mc = sz;
      C_max.assign(popped.rbegin(), popped.rend());
      C_max.push_back(v);
    }
  }
  return mc;
}

// [EXT] pmc::pmcx_maxclique::search_dense (src/graph.cc:106-127, PMC_EXACT), restated as its RESULT CONTRACT.  pmc's exact
// finder is a branch and bound over k-core-pruned, greedily coloured candidate sets run by 12 OpenMP threads (graph.cc:40); which
// of several maximum cliques it returns depends on thread timing, so the reference itself is only deterministic in the clique
// SIZE (and in returning the heuristic clique unchanged when that one already reaches the bound).  The canonical form here is one
// sequential bit-parallel branch and bound (greedy sequential colouring bound, Tomita & Seki / San Segundo) in RANK space:
// vertices renumbered by (core number, id) ascending -- the order the device path keeps its adjacency in.  Rules that make the
// returned clique unique:
//   * the incumbent is the heuristic clique; only a STRICTLY larger clique replaces it (pmc: `if (C.size() > mc)`);
//   * root candidates: every vertex with core number >= |incumbent| (pmc's k-core pruning, K[v] > mc);
//   * colouring: colour classes are built one after the other, each takes the lowest-ranked uncoloured candidate that has no
//     neighbour in the class; only entries whose colour can still beat the incumbent are listed;
//   * branching: from the END of the (colour, rank)-ascending list; a level is abandoned when |C| + colour <= |incumbent|;
//   * the search stops after `node_limit` expanded nodes (the deterministic stand-in for pmc's wall-clock time_limit,
//     graph.cc:44) and then returns the best clique found so far with QB200_FLAG_CLIQUE_TRUNCATED.
// Returns the new clique size; `clique` (ids, any order) is replaced only when a larger clique was found.
int pmc_exact(const uint32_t* adj, int L, int wpr, const std::vector<int>& K, int max_core, long long node_limit,
              std::vector<int>& clique, int& flags) {
  int best = (int)clique.size();
  const int ub = max_core + 1;
  if (L <= 0 || best >= ub) return best;
  // ranks: stable bucket sort by core number (K = core + 1)
  std::vector<int> rank_of(L), by_rank(L), kb(max_core + 3, 0);
  for (int v = 0; v < L; ++v) kb[K[v] - 1 + 1]++;
  for (int d = 1; d <= max_core + 2; ++d) kb[d] += kb[d - 1];   // kb[d] = first rank with core d
  {
    std::vector<int> cur(kb.begin(), kb.end());
    for (int v = 0; v < L; ++v) { rank_of[v] = cur[K[v] - 1]++; by_rank[rank_of[v]] = v; }
  }
  const int nbw = (L + 31) / 32;
  std::vector<uint32_t> rows((size_t)L * nbw, 0u);
  for (int v = 0; v < L; ++v)
    for (int w = 0; w < wpr; ++w) {
      uint32_t x = adj[(size_t)v * wpr + w];
      while (x) {
        const int b = __builtin_ctz(x);
        x &= x - 1;
        const int u = w * 32 + b;
        if (u < L) rows[(size_t)rank_of[v] * nbw + (rank_of[u] >> 5)] |= 1u << (rank_of[u] & 31);
      }
    }
  struct Level { std::vector<uint32_t> P; std::vector<uint32_t> list; };  // list entry: rank | colour << 16
  std::vector<Level> st(1);
  std::vector<int> C, bestC;
  // greedy sequential colouring of P; entries with colour > kmin only
  auto colour_sort = [&](const std::vector<uint32_t>& P, int kmin, std::vector<uint32_t>& list) {
    list.clear();
    std::vector<uint32_t> Q(P), Qk(nbw);
    int col = 0;
    for (;;) {
      bool any = false;
      for (int w = 0; w < nbw; ++w) any |= Q[w] != 0;
      if (!any) break;
      ++col;
      Qk = Q;
      for (;;) {
        int v = -1;
        for (int w = 0; w < nbw; ++w)
          if (Qk[w]) { v = w * 32 + __builtin_ctz(Qk[w]); break; }
        if (v < 0) break;
        const uint32_t* N = &rows[(size_t)v * nbw];
        for (int w = 0; w < nbw; ++w) Qk[w] &= ~N[w];
        Qk[v >> 5] &= ~(1u << (v & 31));
        Q[v >> 5] &= ~(1u << (v & 31));
        if (col > kmin) list.push_back((uint32_t)v | ((uint32_t)col << 16));
      }
    }
  };
  const int thr = kb[std::min(best, max_core + 1)];
  st[0].P.assign(nbw, 0u);
  for (int r = thr; r < L; ++r) st[0].P[r >> 5] |= 1u << (r & 31);
  colour_sort(st[0].P, best, st[0].list);
  long long nodes = 0;
  int depth = 0;
  C.assign(1, 0);
  bool done = false;
  while (depth >= 0 && !done) {
    Level& lv = st[depth];
    if (lv.list.empty()) { --depth; continue; }
    const uint32_t e = lv.list.back();
    lv.list.pop_back();
    const int v = (int)(e & 0xFFFFu), col = (int)(e >> 16);
    if (depth + col <= best) { lv.list.clear(); continue; }
    if ((int)C.size() <= depth) C.resize(depth + 1);
    C[depth] = v;
    std::vector<uint32_t> NP(nbw);
    int cnt = 0;
    const uint32_t* N = &rows[(size_t)v * nbw];
    for (int w = 0; w < nbw; ++w) { NP[w] = lv.P[w] & N[w]; cnt += __builtin_popcount(NP[w]); }
    lv.P[v >> 5] &= ~(1u << (v & 31));
    if (cnt == 0) {
      if (depth + 1 > best) {
        best = depth + 1;
        bestC.assign(C.begin(), C.begin() + depth + 1);
        if (best >= ub) done = true;
      }
      continue;
    }
    if (depth + 1 + cnt <= best) continue;
    if (++nodes > node_limit) { flags |= QB200_FLAG_CLIQUE_TRUNCATED; break; }
    if ((int)st.size() <= depth + 1) st.resize(depth + 2);
    st[depth + 1].P.swap(NP);
    colour_sort(st[depth + 1].P, best - (depth + 1), st[depth + 1].list);
    ++depth;
  }
  if (!bestC.empty()) {
    clique.clear();
    for (int r : bestC) clique.push_back(by_rank[r]);
  }
  return best;
}

int max_clique(const uint32_t* adj, int L, int wpr, int mode, double kcore_thr, std::vector<int>& clique,
               std::vector<int>& kcore, std::vector<int>& order, int& max_core, long long node_limit = 0, int* flags_out = nullptr) {
  clique.clear();
  if (flags_out) *flags_out = 0;
  const Csr g = to_csr(adj, L, wpr);
  compute_cores(g, kcore, order, max_core);
  if (mode == QB200_KCORE_HEU && qb_kcore_heu_shortcut(kcore_thr, L, max_core)) {  // graph.cc:67-82 (D18: the int cast as x86-64)
    for (int v = 0; v < L; ++v)
      if (kcore[v] >= max_core) clique.push_back(v);   // literal: k_cores[i] (= core+1) >= max_core
    return QB200_OK;
  }
  const int ub = max_core + 1;  // graph.cc:84-86
  pmc_heuristic(g, kcore, order, ub, clique);
  if (mode == QB200_PMC_EXACT && (int)clique.size() != ub && !clique.empty()) {  // graph.cc:96-127 (lb == ub returns the heuristic clique)
    int flags = 0;
    pmc_exact(adj, L, wpr, kcore, max_core, node_limit > 0 ? node_limit : QB200_DEFAULT_CLIQUE_NODE_LIMIT, clique, flags);
    if (flags_out) *flags_out = flags;
  }
  std::sort(clique.begin(), clique.end());  // quatro.hpp:806
  return QB200_OK;
}

// ---------------------------------------------------------------------------------------------
// a16. svdRot2d -- include/teaser/utils.h:151-166 (Eigen::JacobiSVD<Matrix2d> restated, D9)
// Matrices are row-major 2x2: {m00, m01, m10, m11}.
// ---------------------------------------------------------------------------------------------
void svd2x2(const double H[4], double U[4], double S[2], double V[4]) {
  // 1) rotation making H symmetric: G = rot1^T-style left rotation
  const double a = H[0], b = H[1], c = H[2], d = H[3];
  const double t = a + d, dd = c - b;
  double c1, s1;
  if (std::fabs(dd) < std::numeric_limits<double>::min()) { c1 = 1.0; s1 = 0.0; }
  else { const double u = t / dd; const double tmp = std::sqrt(1.0 + u * u); s1 = 1.0 / tmp; c1 = u / tmp; }
  // M = Rl * H with Rl = [[c1, s1], [-s1, c1]]  (symmetric result)
  const double m00 = c1 * a + s1 * c, m01 = c1 * b + s1 * d, m10 = -s1 * a + c1 * c, m11 = -s1 * b + c1 * d;
  (void)m10;
  // 2) Jacobi rotation diagonalising the symmetric M: J^T M J = diag
  double cj, sj;
  const double y = m01, deno = 2.0 * std::fabs(y);
  if (deno < std::numeric_limits<double>::min()) { cj = 1.0; sj = 0.0; }
  else {
    const double tau = (m00 - m11) / deno;
    const double w = std::sqrt(tau * tau + 1.0);
    const double tt = tau > 0 ? 1.0 / (tau + w) : 1.0 / (tau - w);
    const double sign_t = tt > 0 ? 1.0 : -1.0;
    const double nn = 1.0 / std::sqrt(tt * tt + 1.0);
    sj = -sign_t * (y / std::fabs(y)) * std::fabs(tt) * nn;
    cj = nn;
  }
  // J = [[cj, sj], [-sj, cj]];  diag = J^T M J;  H = Rl^T M = Rl^T J diag J^T  => U = Rl^T J, V = J
  const double J[4] = {cj, sj, -sj, cj};
  const double RlT[4] = {c1, -s1, s1, c1};
  double Uu[4] = {RlT[0] * J[0] + RlT[1] * J[2], RlT[0] * J[1] + RlT[1] * J[3],
                  RlT[2] * J[0] + RlT[3] * J[2], RlT[2] * J[1] + RlT[3] * J[3]};
  double Vv[4] = {J[0], J[1], J[2], J[3]};
  // singular values = diag(U^T H V); fix signs, sort descending
  double s[2];
  for (int k = 0; k < 2; ++k) {
    const double hv0 = H[0] * Vv[k] + H[1] * Vv[2 + k], hv1 = H[2] * Vv[k] + H[3] * Vv[2 + k];
    s[k] = Uu[k] * hv0 + Uu[2 + k] * hv1;
    if (s[k] < 0) { s[k] = -s[k]; Uu[k] = -Uu[k]; Uu[2 + k] = -Uu[2 + k]; }
  }
  if (s[0] < s[1]) {
    std::swap(s[0], s[1]);
    std::swap(Uu[0], Uu[1]); std::swap(Uu[2], Uu[3]);
    std::swap(Vv[0], Vv[1]); std::swap(Vv[2], Vv[3]);
  }
  for (int k = 0; k < 4; ++k) { U[k] = Uu[k]; V[k] = Vv[k]; }
  S[0] = s[0]; S[1] = s[1];
}

// R = V * U^T with the determinant fix on V.col(1)
void svd_rot2d(const double* X /*2 x c, xs then ys*/, const double* Y, const double* W, int c, double R[4]) {
  double H[4] = {0, 0, 0, 0};  // H = X * diag(W) * Y^T
  const double *x0 = X, *x1 = X + c, *y0 = Y, *y1 = Y + c;
  for (int j = 0; j < c; ++j) {
    H[0] += x0[j] * W[j] * y0[j]; H[1] += x0[j] * W[j] * y1[j];
    H[2] += x1[j] * W[j] * y0[j]; H[3] += x1[j] * W[j] * y1[j];
  }
  double U[4], S[2], V[4];
  svd2x2(H, U, S, V);
  const double detU = U[0] * U[3] - U[1] * U[2], detV = V[0] * V[3] - V[1] * V[2];
  if (detU * detV < 0) { V[1] *= -1; V[3] *= -1; }
  R[0] = V[0] * U[0] + V[1] * U[1]; R[1] = V[0] * U[2] + V[1] * U[3];
  R[2] = V[2] * U[0] + V[3] * U[1]; R[3] = V[2] * U[2] + V[3] * U[3];
}

// a16. solveForRotation2D  include/quatro.hpp:430-572
int gnc_tls_2d(const double* src2 /*2 x c*/, const double* dst2, int c, const qb200_params& prm, double rot_noise_bound,
               double R[4], std::vector<uint8_t>& inliers, double& cost_out) {
  double mu = 1;
  double prev_cost = std::numeric_limits<double>::infinity();
  double cost = std::numeric_limits<double>::infinity();
  double noise_bound_sq = rot_noise_bound * rot_noise_bound;  // std::pow(x, 2)
  if (noise_bound_sq < 1e-16) noise_bound_sq = 1e-2;
  std::vector<double> weights(c, 1.0), residuals_sq(c);
  R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 1;
  int iters = 0;
  for (int i = 0; i < prm.rotation_max_iterations; ++i) {
    iters = i + 1;
    svd_rot2d(src2, dst2, weights.data(), c, R);
    double max_residual = -std::numeric_limits<double>::infinity();
    for (int j = 0; j < c; ++j) {
      const double dx = dst2[j] - (R[0] * src2[j] + R[1] * src2[c + j]);
      const double dy = dst2[c + j] - (R[2] * src2[j] + R[3] * src2[c + j]);
      residuals_sq[j] = dx * dx + dy * dy;
      max_residual = std::max(max_residual, residuals_sq[j]);
    }
    if (i == 0) {
      mu = 1 / (2 * max_residual / noise_bound_sq - 1);
      if (mu <= 0) break;
    }
    const double th1 = (mu + 1) / mu * noise_bound_sq;
    const double th2 = mu / (mu + 1) * noise_bound_sq;
    cost = 0;
    for (int j = 0; j < c; ++j) {
      cost += weights[j] * residuals_sq[j];
      if (residuals_sq[j] >= th1) weights[j] = 0;
      else if (residuals_sq[j] <= th2) weights[j] = 1;
      else weights[j] = std::sqrt(noise_bound_sq * mu * (mu + 1) / residuals_sq[j]) - mu;
    }
    const double cost_diff = std::fabs(cost - prev_cost);
    mu = mu * prm.rotation_gnc_factor;
    prev_cost = cost;
    if (cost_diff < prm.rotation_cost_threshold) break;
  }
  inliers.assign(c, 0);
  for (int j = 0; j < c; ++j) inliers[j] = weights[j] >= 0.4;
  cost_out = cost;
  return iters;
}

// a18. Quatro::estimate  include/quatro.hpp:618-747
double cote_estimate(const double* X, int N, double range, bool median_mode, std::vector<uint8_t>& inliers) {
  std::vector<std::pair<double, int>> h;
  h.reserve(2 * N);
  for (int i = 0; i < N; ++i) {
    h.emplace_back(X[i] - range, i + 1);
    h.emplace_back(X[i] + range, -i - 1);
  }
  const auto by_value = [](const std::pair<double, int>& a, const std::pair<double, int>& b) { return a.first < b.first; };
  if (g_literal) std::sort(h.begin(), h.end(), by_value);  // quatro.hpp:641
  else std::stable_sort(h.begin(), h.end(), by_value);      // D3
  const double weight = 1.0 / (range * range);  // ranges.square().inverse()
  const int nr_centers = 2 * N;
  std::vector<double> x_hat(nr_centers, 0.0), x_cost(nr_centers, 0.0);
  std::vector<int> set_card(nr_centers, 0);
  double ranges_inverse_sum = 0.0;
  for (int i = 0; i < N; ++i) ranges_inverse_sum += range;  // ranges.sum()
  double dot_X_weights = 0, dot_weights_consensus = 0, sum_xi = 0, sum_xi_square = 0;
  int consensus_set_cardinal = 0;
  for (int i = 0; i < nr_centers; ++i) {
    const int idx = std::abs(h[i].second) - 1;
    const int epsilon = (h[i].second > 0) ? 1 : -1;
    consensus_set_cardinal += epsilon;
    dot_weights_consensus += epsilon * weight;
    dot_X_weights += epsilon * weight * X[idx];
    ranges_inverse_sum -= epsilon * range;
    sum_xi += epsilon * X[idx];
    sum_xi_square += epsilon * X[idx] * X[idx];
    set_card[i] = consensus_set_cardinal;
    x_hat[i] = dot_X_weights / dot_weights_consensus;
    const double residual = consensus_set_cardinal * x_hat[i] * x_hat[i] + sum_xi_square - 2 * sum_xi * x_hat[i];
    x_cost[i] = residual + ranges_inverse_sum;
  }
  int min_idx = 0;  // Eigen minCoeff visitor: first minimum, NaN never replaces
  for (int i = 1; i < nr_centers; ++i)
    if (x_cost[i] < x_cost[min_idx]) min_idx = i;
  double est = x_hat[min_idx];
  if (median_mode) {
    const int n_card = set_card[min_idx];
    if (n_card > 0) {
      std::vector<double> cand;
      cand.reserve(n_card);
      for (int j = 0; j < n_card; ++j) cand.push_back(X[std::abs(h[min_idx - j].second) - 1]);
      std::sort(cand.begin(), cand.end());
      if (cand.size() == 1) est = cand[0];  // D5
      else est = (cand[cand.size() / 2 - 1] + cand[cand.size() / 2]) / 2.0;
    }  // else D5: keep x_hat
  }
  inliers.assign(N, 0);
  for (int i = 0; i < N; ++i) inliers[i] = std::fabs(X[i] - est) <= range;
  return est;
}

inline void set_identity(double T[16]) {
  for (int i = 0; i < 16; ++i) T[i] = 0.0;
  T[0] = T[5] = T[10] = T[15] = 1.0;
}

// a13-a19. include/quatro.hpp:806-936 given the sorted clique
int solve_pose(const P4* a, const P4* b, int L, const int* clique, int nc, const qb200_params& prm, qb200_result& res,
               std::vector<uint8_t>& rot_mask, std::vector<uint8_t>& trans_mask, std::vector<int>& final_inliers) {
  set_identity(res.T);
  res.valid = 0; res.clique_size = nc; res.gnc_iters = 0; res.n_rot_inliers = 0; res.n_final_inliers = 0; res.cost = 0;
  rot_mask.clear(); trans_mask.clear(); final_inliers.clear();
  if (nc <= 1) {  // fewer than 2 correspondences is a degenerate input, as in solve_correspondences and the device
    res.status = L < 2 ? QB200_DEGENERATE_INPUT : QB200_DEGENERATE_CLIQUE;
    return res.status;
  }
  // chain TIMs (:817-844), XY rows only feed the rotation (:396-402)
  std::vector<double> s2(2 * (size_t)nc), d2(2 * (size_t)nc);
  for (int i = 0; i < nc; ++i) {
    const int root = clique[i], leaf = (i != nc - 1) ? clique[i + 1] : clique[0];
    s2[i] = (double)a[leaf].x - (double)a[root].x; s2[nc + i] = (double)a[leaf].y - (double)a[root].y;
    d2[i] = ((double)b[leaf].x - (double)b[root].x) * (1 / 1.0); d2[nc + i] = ((double)b[leaf].y - (double)b[root].y) * (1 / 1.0);
  }
  // noise bound handed to the rotation solver: static latched after params_.noise_bound *= 2 (:851, :469)
  const double rot_nb = prm.rot_noise_bound > 0 ? prm.rot_noise_bound : 2.0 * prm.noise_bound;
  double R2[4];
  res.gnc_iters = gnc_tls_2d(s2.data(), d2.data(), nc, prm, rot_nb, R2, rot_mask, res.cost);
  double R[9] = {R2[0], R2[1], 0, R2[2], R2[3], 0, 0, 0, 1};  // rot_yaw (:404-408)
  double RyRx[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (prm.use_pre_estimated_RyRx) {  // :419-426
    for (int i = 0; i < 9; ++i) RyRx[i] = prm.RyRx[i];
    double Rn[9];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) Rn[3 * r + c] = R[3 * r] * RyRx[c] + R[3 * r + 1] * RyRx[3 + c] + R[3 * r + 2] * RyRx[6 + c];
    for (int i = 0; i < 9; ++i) R[i] = Rn[i];
  }
  // rotation inliers (:857-874)
  std::vector<int> rot_inl;
  for (int i = 0; i < nc; ++i) {
    const int prev = (i == 0) ? nc - 1 : i - 1;
    if (rot_mask[prev] && rot_mask[i]) rot_inl.push_back(i);
  }
  res.n_rot_inliers = (int)rot_inl.size();
  const int N_R = (int)rot_inl.size();
  const bool use_rot = prm.using_rot_inliers_when_estimating_cote && N_R > 0;
  const int N = use_rot ? N_R : nc;
  // translation inputs (:879-907): dst - R * (RyRx * src)   [the RyRx product only in the default branch]
  std::vector<double> X(3 * (size_t)N);
  for (int i = 0; i < N; ++i) {
    const int v = use_rot ? clique[rot_inl[i]] : clique[i];
    double sx = (double)a[v].x, sy = (double)a[v].y, sz = (double)a[v].z;
    if (!use_rot) {
      const double tx = RyRx[0] * sx + RyRx[1] * sy + RyRx[2] * sz;
      const double ty = RyRx[3] * sx + RyRx[4] * sy + RyRx[5] * sz;
      const double tz = RyRx[6] * sx + RyRx[7] * sy + RyRx[8] * sz;
      sx = tx; sy = ty; sz = tz;
    }
    const double rx = 1.0 * R[0] * sx + 1.0 * R[1] * sy + 1.0 * R[2] * sz;
    const double ry = 1.0 * R[3] * sx + 1.0 * R[4] * sy + 1.0 * R[5] * sz;
    const double rz = 1.0 * R[6] * sx + 1.0 * R[7] * sy + 1.0 * R[8] * sz;
    X[i] = (double)b[v].x - rx; X[N + i] = (double)b[v].y - ry; X[2 * (size_t)N + i] = (double)b[v].z - rz;
  }
  const double range = prm.cote_noise_bound * std::sqrt(prm.cbar2);  // :600-601
  double t[3];
  trans_mask.assign(N, 1);
  std::vector<uint8_t> tmp;
  for (int ax = 0; ax < 3; ++ax) {
    t[ax] = cote_estimate(&X[(size_t)ax * N], N, range, prm.cote_mode == QB200_COTE_MEDIAN, tmp);
    for (int i = 0; i < N; ++i) trans_mask[i] = trans_mask[i] && tmp[i];
  }
  for (int i = 0; i < N; ++i)
    if (trans_mask[i]) final_inliers.push_back(use_rot ? clique[rot_inl[i]] : clique[i]);
  res.n_final_inliers = (int)final_inliers.size();
  res.valid = 1; res.status = QB200_OK;
  // column-major 4x4
  res.T[0] = R[0]; res.T[1] = R[3]; res.T[2] = R[6]; res.T[3] = 0;
  res.T[4] = R[1]; res.T[5] = R[4]; res.T[6] = R[7]; res.T[7] = 0;
  res.T[8] = R[2]; res.T[9] = R[5]; res.T[10] = R[8]; res.T[11] = 0;
  res.T[12] = t[0]; res.T[13] = t[1]; res.T[14] = t[2]; res.T[15] = 1;
  return QB200_OK;
}

struct SolveOut {
  std::vector<int> clique, final_inliers, kcore, order;
  std::vector<uint8_t> rot_mask, trans_mask;
};

int solve_correspondences(const P4* a, const P4* b, int L, const qb200_params& prm, qb200_result& res, SolveOut& so) {
  set_identity(res.T);
  res.valid = 0; res.n_corr = L; res.n_edges = 0; res.max_core = 0; res.clique_size = 0; res.flags = 0;
  res.gnc_iters = 0; res.n_rot_inliers = 0; res.n_final_inliers = 0; res.cost = 0;
  if (L < 2) { res.status = QB200_DEGENERATE_INPUT; return QB200_DEGENERATE_INPUT; }
  if (prm.inlier_selection_mode == QB200_INLIER_NONE) {
    // reference leaves max_clique_ empty here (quatro.hpp:782); TEASER++'s semantics: every measurement
    so.clique.resize(L);
    std::iota(so.clique.begin(), so.clique.end(), 0);
  } else {
    const int wpr = (L + 31) / 32;
    std::vector<uint32_t> adj((size_t)L * wpr);
    build_graph(a, b, L, prm.noise_bound, prm.cbar2, adj.data(), wpr, nullptr, &res.n_edges);
    int fl = 0;
    const int st = max_clique(adj.data(), L, wpr, prm.inlier_selection_mode, prm.kcore_heuristic_threshold, so.clique,
                              so.kcore, so.order, res.max_core, prm.max_clique_node_limit, &fl);
    res.flags = fl;
    if (st < 0) { res.status = st; return st; }
  }
  return solve_pose(a, b, L, so.clique.data(), (int)so.clique.size(), prm, res, so.rot_mask, so.trans_mask, so.final_inliers);
}

#include "preprocess_oracle.inc"

double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

}  // namespace

// =====================================================================================
// C interface (loaded by tests/ and bench.py via ctypes)
// =====================================================================================
extern "C" {

// 1 = literal mode (see g_literal), 0 = canonical (default).  Returns the previous value.
int qo_set_literal(int on) {
  const int prev = g_literal;
  g_literal = on ? 1 : 0;
  return prev;
}

int qo_set_num_threads(int n) {
#ifdef _OPENMP
  if (n > 0) omp_set_num_threads(n);
  return omp_get_max_threads();
#else
  (void)n;
  return 1;
#endif
}

int qo_voxelize(const float* pts4, int n, float leaf, int skip_flagged, float* out4, int cap, int* n_out) {
  std::vector<P4> out;
  const int st = voxelize(reinterpret_cast<const P4*>(pts4), n, leaf, skip_flagged, out);
  *n_out = (int)out.size();
  const int m = std::min((int)out.size(), cap);
  std::memcpy(out4, out.data(), (size_t)m * sizeof(P4));
  if ((int)out.size() > cap) return QB200_CAPACITY_EXCEEDED;
  return st;
}

int qo_compute_fpfh(const float* pts4, int n, float normal_radius, float fpfh_radius, float grid_cell, float* normals4,
                    float* desc33, float* spfh33) {
  if (normal_radius > fpfh_radius) return QB200_ERR_BAD_ARG;  // fpfh_manager.hpp:99-102
  const P4* pts = reinterpret_cast<const P4*>(pts4);
  Lattice lat;
  lat.build(pts, n, grid_cell);
  std::vector<P4> nrm(n);
  compute_normals(pts, n, lat, normal_radius, nrm.data());
  std::vector<float> spfh((size_t)n * 33), fpfh((size_t)n * 33);
  compute_spfh(pts, nrm.data(), n, lat, fpfh_radius, spfh.data());
  compute_fpfh(pts, n, lat, fpfh_radius, spfh.data(), fpfh.data());
  if (normals4) std::memcpy(normals4, nrm.data(), (size_t)n * sizeof(P4));
  if (desc33) std::memcpy(desc33, fpfh.data(), fpfh.size() * sizeof(float));
  if (spfh33) std::memcpy(spfh33, spfh.data(), spfh.size() * sizeof(float));
  return QB200_OK;
}

// radius-search neighbour list of one query (brute-force cross-check target for tests)
int qo_neighbors(const float* pts4, int n, float grid_cell, int q, float radius, int* idx, float* d2, int cap) {
  const P4* pts = reinterpret_cast<const P4*>(pts4);
  Lattice lat;
  lat.build(pts, n, grid_cell);
  int k = 0;
  lat.for_each_neighbor(pts, q, radius, [&](int p, float dd) {
    if (k < cap) { idx[k] = p; d2[k] = dd; }
    ++k;
  });
  return k;
}

int qo_match(const float* src4, int n_src, const float* sdesc, const float* tgt4, int n_tgt, const float* tdesc,
             const qb200_params* prm, int* corr, int cap, int* n_corr, int* n_mutual, int* mutual /*2*min(n) or NULL*/) {
  MatchOut mo;
  const int st = match(reinterpret_cast<const P4*>(src4), n_src, sdesc, reinterpret_cast<const P4*>(tgt4), n_tgt, tdesc, *prm, mo);
  if (st < 0) return st;
  *n_corr = (int)mo.corr.size();
  if (n_mutual) *n_mutual = (int)mo.mutual.size();
  if (mutual)
    for (size_t i = 0; i < mo.mutual.size(); ++i) { mutual[2 * i] = mo.mutual[i].first; mutual[2 * i + 1] = mo.mutual[i].second; }
  const int m = std::min((int)mo.corr.size(), cap);
  for (int i = 0; i < m; ++i) { corr[2 * i] = mo.corr[i].first; corr[2 * i + 1] = mo.corr[i].second; }
  return (int)mo.corr.size() > cap ? QB200_CAPACITY_EXCEEDED : QB200_OK;
}

// both nearest-neighbour tables of match() for A (nA x 33) against B (nB x 33), in the given order (no larger-cloud swap):
// bestA[i] = packed (distance bits << 32 | j) of row i's nearest B, bestB[j] = the same for column j's nearest A, ~0 = none
int qo_nn_tables(const float* A, int nA, const float* B, int nB, uint64_t* bestA, uint64_t* bestB) {
  if (nA < 0 || nB < 0) return QB200_ERR_BAD_ARG;
  std::vector<int> nnA, nnB;
  nn_both_ways(A, nA, B, nB, nnA, nnB, bestA, bestB);
  return QB200_OK;
}

int qo_build_graph(const float* a4, const float* b4, int L, double noise_bound, double cbar2, uint32_t* adj, int wpr,
                   int* degree, int64_t* n_edges) {
  if (wpr < (L + 31) / 32) return QB200_ERR_BAD_ARG;
  build_graph(reinterpret_cast<const P4*>(a4), reinterpret_cast<const P4*>(b4), L, noise_bound, cbar2, adj, wpr, degree, n_edges);
  return QB200_OK;
}

int qo_patchwork(const float* pts4, int n, const qb200_patchwork_params* pp, float* ground4, int* n_ground, float* nonground4,
                 int* n_nonground) {
  std::vector<P4> g, ng;
  const int st = patchwork(reinterpret_cast<const P4*>(pts4), n, *pp, g, ng);
  if (st < 0) return st;
  *n_ground = (int)g.size();
  *n_nonground = (int)ng.size();
  if (ground4 && !g.empty()) memcpy(ground4, g.data(), g.size() * sizeof(P4));
  if (nonground4 && !ng.empty()) memcpy(nonground4, ng.data(), ng.size() * sizeof(P4));
  return st;
}

int qo_segment_cloud(const float* pts4, int n, const qb200_segment_params* sp, float* valid4, int* n_valid, float* outlier4, int* n_outlier) {
  std::vector<P4> v, o;
  const int st = segment_cloud(reinterpret_cast<const P4*>(pts4), n, *sp, v, o);
  if (st < 0) return st;
  *n_valid = (int)v.size();
  *n_outlier = (int)o.size();
  if (valid4 && !v.empty()) memcpy(valid4, v.data(), v.size() * sizeof(P4));
  if (outlier4 && !o.empty()) memcpy(outlier4, o.data(), o.size() * sizeof(P4));
  return st;
}

int qo_max_clique_ex(const uint32_t* adj, int L, int wpr, int mode, double kcore_thr, int64_t node_limit, int* clique, int* n_clique,
                     int* kcore, int* kcore_order, int* max_core, int* flags) {
  std::vector<int> c, k, o;
  int mcore = 0, fl = 0;
  const int st = max_clique(adj, L, wpr, mode, kcore_thr, c, k, o, mcore, node_limit, &fl);
  if (st < 0) return st;
  if (flags) *flags = fl;
  *n_clique = (int)c.size();
  std::copy(c.begin(), c.end(), clique);
  if (kcore) std::copy(k.begin(), k.end(), kcore);
  if (kcore_order) std::copy(o.begin(), o.end(), kcore_order);
  if (max_core) *max_core = mcore;
  return QB200_OK;
}

int qo_max_clique(const uint32_t* adj, int L, int wpr, int mode, double kcore_thr, int* clique, int* n_clique, int* kcore,
                  int* kcore_order, int* max_core) {
  return qo_max_clique_ex(adj, L, wpr, mode, kcore_thr, 0, clique, n_clique, kcore, kcore_order, max_core, nullptr);
}

int qo_solve_pose(const float* a4, const float* b4, int L, const int* clique, int n_clique, const qb200_params* prm,
                  qb200_result* res, uint8_t* rot_mask, uint8_t* trans_mask, int* final_inliers) {
  std::vector<uint8_t> rm, tm;
  std::vector<int> fi;
  qb200_result r;
  std::memset(&r, 0, sizeof(r));
  const int st = solve_pose(reinterpret_cast<const P4*>(a4), reinterpret_cast<const P4*>(b4), L, clique, n_clique, *prm, r, rm, tm, fi);
  r.n_corr = L;
  *res = r;
  if (rot_mask) std::copy(rm.begin(), rm.end(), rot_mask);
  if (trans_mask) std::copy(tm.begin(), tm.end(), trans_mask);
  if (final_inliers) std::copy(fi.begin(), fi.end(), final_inliers);
  return st;
}

int qo_solve_correspondences(const float* a4, const float* b4, int L, const qb200_params* prm, qb200_result* res,
                             int* clique, int* n_clique, int* final_inliers, int* n_final) {
  SolveOut so;
  qb200_result r;
  std::memset(&r, 0, sizeof(r));
  const int st = solve_correspondences(reinterpret_cast<const P4*>(a4), reinterpret_cast<const P4*>(b4), L, *prm, r, so);
  *res = r;
  if (n_clique) *n_clique = (int)so.clique.size();
  if (clique) std::copy(so.clique.begin(), so.clique.end(), clique);
  if (n_final) *n_final = (int)so.final_inliers.size();
  if (final_inliers) std::copy(so.final_inliers.begin(), so.final_inliers.end(), final_inliers);
  return st;
}

// FPFHManager::setFeaturePair, include/fpfh_manager.hpp:98-153 (voxelized clouds in)
int qo_match_and_pack(const float* src4, int n_src, const float* tgt4, int n_tgt, const qb200_params* prm, int* corr,
                      float* src_matched4, float* tgt_matched4, int cap, int* n_corr, int* n_mutual) {
  if (prm->normal_radius > prm->fpfh_radius) return QB200_ERR_BAD_ARG;
  const float cell = prm->grid_cell > 0 ? prm->grid_cell : prm->fpfh_radius * 1.001953125f;  // (1 + 2^-9) r: a 3 x 3 x 3 cell walk is then provably enough
  std::vector<float> sd((size_t)n_src * 33), td((size_t)n_tgt * 33);
  qo_compute_fpfh(src4, n_src, prm->normal_radius, prm->fpfh_radius, cell, nullptr, sd.data(), nullptr);
  qo_compute_fpfh(tgt4, n_tgt, prm->normal_radius, prm->fpfh_radius, cell, nullptr, td.data(), nullptr);
  MatchOut mo;
  const int st = match(reinterpret_cast<const P4*>(src4), n_src, sd.data(), reinterpret_cast<const P4*>(tgt4), n_tgt, td.data(), *prm, mo);
  if (st < 0) return st;
  *n_corr = (int)mo.corr.size();
  if (n_mutual) *n_mutual = (int)mo.mutual.size();
  const int m = std::min((int)mo.corr.size(), cap);
  const P4* s = reinterpret_cast<const P4*>(src4); const P4* t = reinterpret_cast<const P4*>(tgt4);
  for (int i = 0; i < m; ++i) {
    corr[2 * i] = mo.corr[i].first; corr[2 * i + 1] = mo.corr[i].second;
    const P4 ps = s[mo.corr[i].first], pt = t[mo.corr[i].second];
    // 3xL double -> eigen2pcl float (exact round trip), pad w = 1
    src_matched4[4 * i] = ps.x; src_matched4[4 * i + 1] = ps.y; src_matched4[4 * i + 2] = ps.z; src_matched4[4 * i + 3] = 1.0f;
    tgt_matched4[4 * i] = pt.x; tgt_matched4[4 * i + 1] = pt.y; tgt_matched4[4 * i + 2] = pt.z; tgt_matched4[4 * i + 3] = 1.0f;
  }
  return (int)mo.corr.size() > cap ? QB200_CAPACITY_EXCEEDED : QB200_OK;
}

// examples/run_global_registration.cpp:206-246: voxelize x2 -> setFeaturePair -> computeTransformation.
// stage_s (8 doubles, may be NULL): [1]=voxel [2]=fpfh [3]=match [4]=graph [5]=clique [6]=pose
int qo_register_pair(const float* src4, int n_src, const float* tgt4, int n_tgt, const qb200_params* prm, qb200_result* res,
                     double* stage_s) {
  qb200_result r;
  std::memset(&r, 0, sizeof(r));
  set_identity(r.T);
  double ts[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  double t0 = now_s();
  std::vector<P4> sv, tv;
  int st = voxelize(reinterpret_cast<const P4*>(src4), n_src, prm->voxel_size, prm->skip_flagged, sv);
  if (st < 0) { r.status = st; *res = r; return st; }
  st = voxelize(reinterpret_cast<const P4*>(tgt4), n_tgt, prm->voxel_size, prm->skip_flagged, tv);
  if (st < 0) { r.status = st; *res = r; return st; }
  ts[1] = now_s() - t0; t0 = now_s();
  r.n_src_vox = (int)sv.size(); r.n_tgt_vox = (int)tv.size();
  if (sv.empty() || tv.empty()) { r.status = QB200_DEGENERATE_INPUT; *res = r; return r.status; }
  const float cell = prm->grid_cell > 0 ? prm->grid_cell : prm->fpfh_radius * 1.001953125f;  // (1 + 2^-9) r: a 3 x 3 x 3 cell walk is then provably enough
  std::vector<float> sd((size_t)sv.size() * 33), td((size_t)tv.size() * 33);
  qo_compute_fpfh(&sv[0].x, (int)sv.size(), prm->normal_radius, prm->fpfh_radius, cell, nullptr, sd.data(), nullptr);
  qo_compute_fpfh(&tv[0].x, (int)tv.size(), prm->normal_radius, prm->fpfh_radius, cell, nullptr, td.data(), nullptr);
  ts[2] = now_s() - t0; t0 = now_s();
  MatchOut mo;
  st = match(sv.data(), (int)sv.size(), sd.data(), tv.data(), (int)tv.size(), td.data(), *prm, mo);
  if (st < 0) { r.status = st; *res = r; return st; }
  ts[3] = now_s() - t0; t0 = now_s();
  r.n_mutual = (int)mo.mutual.size();
  const int L = (int)mo.corr.size();
  std::vector<P4> a(L), b(L);
  for (int i = 0; i < L; ++i) { a[i] = sv[mo.corr[i].first]; b[i] = tv[mo.corr[i].second]; }
  // solve (graph / clique / pose timed separately)
  qb200_result rs;
  std::memset(&rs, 0, sizeof(rs));
  SolveOut so;
  if (L >= 2 && prm->inlier_selection_mode != QB200_INLIER_NONE) {
    const int wpr = (L + 31) / 32;
    std::vector<uint32_t> adj((size_t)L * wpr);
    set_identity(rs.T);
    build_graph(a.data(), b.data(), L, prm->noise_bound, prm->cbar2, adj.data(), wpr, nullptr, &rs.n_edges);
    ts[4] = now_s() - t0; t0 = now_s();
    st = max_clique(adj.data(), L, wpr, prm->inlier_selection_mode, prm->kcore_heuristic_threshold, so.clique, so.kcore, so.order, rs.max_core);
    ts[5] = now_s() - t0; t0 = now_s();
    if (st >= 0) st = solve_pose(a.data(), b.data(), L, so.clique.data(), (int)so.clique.size(), *prm, rs, so.rot_mask, so.trans_mask, so.final_inliers);
    else rs.status = st;
    ts[6] = now_s() - t0;
  } else {
    st = solve_correspondences(a.data(), b.data(), L, *prm, rs, so);
    ts[6] = now_s() - t0;
  }
  rs.n_src_vox = r.n_src_vox; rs.n_tgt_vox = r.n_tgt_vox; rs.n_mutual = r.n_mutual; rs.n_corr = L;
  *res = rs;
  if (stage_s) std::memcpy(stage_s, ts, sizeof(ts));
  return st;
}

// ---- small exports used by the known-answer tests ------------------------------------------
float qo_test_atan2f(float y, float x) { return qo_atan2f(y, x); }
float qo_test_acosf(float x) { return qo_acosf(x); }
void qo_test_sincosf(float x, float* s, float* c) { qo_sincosf(x, s, c); }
void qo_test_philox(uint64_t seed, uint64_t ctr, uint32_t* out4) { philox4x32_10(seed, ctr, out4); }
void qo_test_svd2x2(const double* H, double* U, double* S, double* V) { svd2x2(H, U, S, V); }
void qo_test_svd_rot2d(const double* X, const double* Y, const double* W, int c, double* R) { svd_rot2d(X, Y, W, c, R); }
void qo_test_normal_from_accu(const float* accu9, int cnt, const float* p3, float* out4) {
  float a[9];
  for (int i = 0; i < 9; ++i) a[i] = accu9[i];
  const P4 n = normal_from_accu(a, cnt, P4{p3[0], p3[1], p3[2], 1.0f});
  out4[0] = n.x; out4[1] = n.y; out4[2] = n.z; out4[3] = n.w;
}
void qo_test_feature_bins(float f1, float f2, float f3, int* b) {
  const float d_pi = 1.0f / (2.0f * (float)M_PI);
  b[0] = bin_of(11 * (((double)f1 + M_PI) * (double)d_pi));
  b[1] = bin_of(11 * (((double)f2 + 1.0) * 0.5));
  b[2] = bin_of(11 * (((double)f3 + 1.0) * 0.5));
}
int qo_test_pair_features(const float* p1, const float* n1, const float* p2, const float* n2, float* f) {
  return pair_features(*reinterpret_cast<const P4*>(p1), *reinterpret_cast<const P4*>(n1), *reinterpret_cast<const P4*>(p2),
                       *reinterpret_cast<const P4*>(n2), f[0], f[1], f[2]) ? 1 : 0;
}
double qo_test_cote(const double* X, int N, double range, int median_mode, uint8_t* inliers) {
  std::vector<uint8_t> in;
  const double e = cote_estimate(X, N, range, median_mode != 0, in);
  std::copy(in.begin(), in.end(), inliers);
  return e;
}
int qo_test_gnc(const double* src2, const double* dst2, int c, const qb200_params* prm, double rot_nb, double* R, uint8_t* inl, double* cost) {
  std::vector<uint8_t> in;
  const int it = gnc_tls_2d(src2, dst2, c, *prm, rot_nb, R, in, *cost);
  std::copy(in.begin(), in.end(), inl);
  return it;
}
int qo_test_kcore(const uint32_t* adj, int L, int wpr, int* kcore, int* order) {
  const Csr g = to_csr(adj, L, wpr);
  std::vector<int> k, o;
  int mc = 0;
  compute_cores(g, k, o, mc);
  std::copy(k.begin(), k.end(), kcore);
  std::copy(o.begin(), o.end(), order);
  return mc;
}

}  // extern "C"
