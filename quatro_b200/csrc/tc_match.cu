// tc_match.cu -- K6 on the Hopper tensor cores (wgmma, TF32), sm_90a.   (QB200_MATCH_EXACT=1 bypasses it.)
//
// The N_src x N_tgt x 33 descriptor-distance matrix is the one genuinely dense contraction of the path
// (north_star): d(i,j) = |a_i|^2 + |b_j|^2 - 2 a_i.b_j.  The reference does two exact 1-NN searches (FLANN kd-trees,
// src/teaser_utils/feature_matcher.cc:97-125); the exact answer here is DEFINED by the fp32 fma chain of match.cu
// (lowest-index ties).  Tensor cores cannot reproduce that rounding, so they act as a conservative FILTER and the
// survivors are evaluated exactly inside the same kernel -- results are bit-identical to the exact kernel.
//
//   norm_key_kernel   : |x - mu|^2 by the fp32 chain (mu = FPFH signature of a plane: 100 in bins 5, 16, 27 -- street scenes
//                       are dominated by planar points, centring makes THEIR dot products tiny and therefore the filter's
//                       absolute error tiny exactly where near-ties are dense) -> one radix sort orders every cloud by norm
//   dedup_kernel      : runs of bit-identical descriptors (adjacent after the sort) collapse to their first rank = lowest index
//   split_desc_kernel : hi = TF32(x'), lo = TF32(x' - hi), exact x, per block of 64 unique descriptors as ready-made
//                       shared-memory operand images (hi | lo | exact), so an image is ONE cp.async.bulk
//   tc_seed_kernel    : every unique row and column starts with the exact distance to its nearest-norm candidates of the
//                       other cloud, so the filter and the tile skip have finite thresholds from the first tile on
//   tc_nn_kernel      : per 128-row stripe, 64-column tiles in nearest-norm-first order; a tile whose lower bound
//                       (gap of the norm ranges)^2 exceeds every current best of the stripe's rows and of its columns is
//                       skipped unloaded; otherwise
//                         d~ = |a'|^2 + |b'|^2 - 2 (hi.hi + hi.lo + lo.hi)      3 x 5 wgmma m64n64k8 TF32 per warpgroup, fp32 in registers
//                         |d~ - d| <= e_ij = c/2 (|a'_i|^2 + |b'_j|^2),  c = 6e-5   (split + accumulation + chain rounding)
//                         (i,j) is evaluated EXACTLY (fp32 chain from the exact images) iff its lower bound d~ - e_ij
//                         does not exceed the best exact distance known so far for row i or for column j;
//                         row bests live in shared memory, column bests in global memory (atomicMin on packed
//                         distance|index words).
//                       A stripe that evaluates too many entries (massive near-ties) flags its pair, which is redone by the
//                       exact CUDA-core kernel, so results never depend on the filter.
//   broadcast_best_kernel : class results -> every member, in point order for the mutual-NN stage
//
// tc_nn_kernel, two CTAs per SM (320 threads, <= 96 registers, 100 KB dynamic shared memory each), mbarrier hand-offs only:
// warp 9 chooses tiles and issues the exact-image copies (2 stages), warp 8 the operand copies (1 stage); warps 0..7 are
// 2 warpgroups, each issues the 15 wgmma of its 64 rows x the tile's 64 columns and runs the filter / exact evaluation on the
// accumulator fragment it holds.  One CTA's wgmma runs while the other CTA of the SM filters and evaluates (DESIGN.md 5.1).
#include "handle.cuh"
#include <cstdlib>

namespace qb {

constexpr int kTcM = 128, kTcN = 64;              // stripe rows x column-tile width
constexpr int kTcBlk = 64;                        // points per operand-image block: a stripe is 2 blocks, a column tile 1
constexpr int kTcKB = kDescK / 8;                 // K blocks of 8 (TF32 MMA K)
constexpr int kTcTileBytes = kDescK * kTcBlk * 4; // one operand image (64 points x 40 dims) = 10240 B
constexpr int kTileFloats = kDescK * kTcBlk;      // 2560
constexpr int kTcImages = 3;                      // hi | lo | exact
constexpr int kTcEpiWarps = 8;                    // MMA + filter / evaluation warps: warpgroup g = rows 64 g .. 64 g + 63
constexpr int kTcThreads = (kTcEpiWarps + 2) * 32;  // + operand-copy warp + scheduler warp
constexpr int kTcDone = 4;                         // ring of "MMAs of position k done by every warp" barriers
constexpr int kTcStages = 2;                      // ring of exact B images (prefetch distance 1); operand images: 1 stage
constexpr int kTcSmemTiles = 256;                 // column tiles whose lower bounds live in shared memory (V <= 16384)
constexpr float kTcC = 1.2e-4f;                   // |d~ - d| <= kTcC/2 * (|a'|^2 + |b'|^2): 3x the worst error measured (test_tc_filter_error_bound)
// Largest centred squared norm the tensor-core path takes: below it every term of kLow (|a'|^2 + |b'|^2) - 2 a'.b' and every exact
// distance stays below 2^127 < FLT_MAX.  A pair with a larger, infinite or NaN norm goes to the exact kernel (split_desc_kernel).
constexpr float kTcNormMax = 0x1p124f;
// Relative part of the tile-skip slack, per unit of square-rooted norm (tile_lb in tc_nn_kernel).  The norm chain rounds
// x' = x - mu (1 ulp), 33 fma (33 ulp of |x'|^2) and the square root (1 ulp): |x'| computed = |x'| (1 + e), |e| <= 18.5 * 2^-24
// = 1.1e-6, so the gap of two norm ranges is off by at most 1.1e-6 (amax + bmax).  4e-6 leaves a factor of 3.6 for the float
// arithmetic of the bound itself.  The 0.9999 factor covers the exact chain's own rounding (d computed >= d (1 - 36 * 2^-24)).
constexpr float kTcNormRel = 4.0e-6f;
constexpr int kSpinLimit = 400000;
constexpr int kSeedW = 16;                        // seed candidates on either side of a descriptor's norm (tools/tc_seed_study.py)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Operand images use the canonical K-major / no-swizzle (interleave) wgmma layout: core matrix = 8 points x 16 B
// (4 consecutive K values), byte offset kc*1024 + p*16 for K chunk kc (4 dims) and point p of the 64-point block.
__device__ __forceinline__ uint64_t tc_smem_desc(uint32_t addr) {
  // start address >> 4 | LBO = 1024 B (next 4-wide K chunk) | SBO = 128 B (next 8-point group) | no swizzle (bits 62-63 = 0)
  return (uint64_t)((addr & 0x3FFFF) >> 4) | ((uint64_t)((kTcBlk * 16) >> 4) << 16) | ((uint64_t)(128 >> 4) << 32);
}

// D (64 x 64, fp32, registers of the warpgroup) (+)= A (64 x 8) * B (64 x 8)^T, both TF32 and K-major in shared memory.
// Fragment: thread (warp w of the warpgroup, lane l) holds d[i] = D[16 w + l / 4 + 8 ((i >> 1) & 1)][8 (i >> 2) + 2 (l & 3) + (i & 1)].
__device__ __forceinline__ void wgmma_tf32_64x64x8(float (&d)[32], uint64_t adesc, uint64_t bdesc, int accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}

// AND of v over the 128 threads of warpgroup g (named barrier 1 + g): every exit from the tile loop is decided by this vote,
// so no warp of a warpgroup can leave while the others enter a wgmma
__device__ __forceinline__ bool wg_all(bool v, int g) {
  uint32_t r;
  asm volatile(
      "{\n\t.reg .pred p, q;\n\t"
      "setp.ne.u32 p, %1, 0;\n\t"
      "bar.red.and.pred q, %2, 128, p;\n\t"
      "selp.u32 %0, 1, 0, q;\n\t}\n"
      : "=r"(r)
      : "r"((uint32_t)v), "r"(1 + g)
      : "memory");
  return r != 0;
}

__device__ __forceinline__ float tc_mu(int d) { return (d == 5 || d == 16 || d == 27) ? 100.0f : 0.0f; }

// centred squared norm of every descriptor (the fp32 chain split_desc_kernel repeats) as the sort key cloud | norm bits:
// K6 processes the points of a cloud in ascending-norm order, which turns the reverse triangle inequality
// d(a,b) >= (|a'| - |b'|)^2 into a tile-level lower bound (whole 128 x 64 blocks are skipped without being loaded).
__global__ void __launch_bounds__(256) norm_key_kernel(const float* __restrict__ desc_t, const int* __restrict__ n_vox, int V,
                                                       uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const int cloud = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= V) return;
  uint32_t bits = 0xFFFFFFFFu;  // padding sorts last
  if (q < n_vox[cloud]) {
    const size_t base = (size_t)cloud * kDescK * V + q;
    float acc = 0.0f;
#pragma unroll
    for (int d = 0; d < kDescDim; ++d) {
      const float xc = desc_t[base + (size_t)d * V] - tc_mu(d);
      acc = __fmaf_rn(xc, xc, acc);
    }
    bits = acc == acc ? __float_as_uint(acc) : 0xFFFFFFFEu;  // squared norms are >= 0: the bit pattern orders them
  }
  keys[(size_t)cloud * V + q] = ((uint64_t)cloud << 32) | bits;
  vals[(size_t)cloud * V + q] = (uint32_t)q;
}

// centred TF32 split + exact image + centred squared norm, written block-wise in the shared-memory operand layout;
// rank r of the cloud (ascending norm, ties by index) is point perm[r].  A norm above kTcNormMax, +inf or NaN (a non-finite bin,
// or finite values whose squares overflow) would turn the filter's lower bounds into NaN or inf, which no threshold passes:
// such a pair is flagged for the exact kernel, whose NaN / inf handling is the oracle's.
__global__ void __launch_bounds__(256) split_desc_kernel(const float* __restrict__ desc_t, const int* __restrict__ n_vox, int V,
                                                         const uint32_t* __restrict__ perm, float* __restrict__ tiles,
                                                         float* __restrict__ norm, int* __restrict__ fallback) {
  const int cloud = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = n_vox[cloud];
  const int NB = V / kTcBlk;
  // the last stripe (both of its blocks) is padded with zeros so stale data never reaches the tensor core
  if (q >= ((n + kTcM - 1) & ~(kTcM - 1))) return;
  const size_t base = (size_t)cloud * kDescK * V + (q < n ? perm[(size_t)cloud * V + q] : 0u);
  const int blk = q / kTcBlk, p = q % kTcBlk;
  float4* __restrict__ img = reinterpret_cast<float4*>(tiles + (size_t)(cloud * NB + blk) * kTcImages * kTileFloats) + p;
  // The tensor core delivers the filter's LOWER BOUND itself: rows (source clouds, even) carry x' in dims 0..32, kLow |x'|^2 in
  // dim 33 and 1 in dim 34; columns (target clouds, odd) carry -2 x', 1 and kLow |x'|^2 -- the contraction over the 35 dims is
  // kLow (|a'|^2 + |b'|^2) - 2 a'.b'.  (Scaling by -2 is exact; the norm term is split hi | lo like every other value.)
  const bool is_col = (cloud & 1) != 0;
  const float kLow = 1.0f - 0.5f * kTcC;
  float acc = 0.0f;
#pragma unroll
  for (int kc = 0; kc < kDescK / 4; ++kc) {
    float xv[4], hv[4], lv[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int d = 4 * kc + e;
      const bool live = d < kDescDim && q < n;
      const float x = live ? desc_t[base + (size_t)d * V] : 0.0f;
      const float xc = live ? x - tc_mu(d) : 0.0f;
      xv[e] = x;
      acc = __fmaf_rn(xc, xc, acc);
      float xs = is_col ? -2.0f * xc : xc;
      if (q < n && d == kDescDim) xs = is_col ? 1.0f : kLow * acc;       // acc is complete here: d runs upwards
      if (q < n && d == kDescDim + 1) xs = is_col ? kLow * acc : 1.0f;
      hv[e] = __uint_as_float(__float_as_uint(xs) & 0xFFFFE000u);
      lv[e] = __uint_as_float(__float_as_uint(xs - hv[e]) & 0xFFFFE000u);
    }
    img[0 * (kTileFloats / 4) + kc * kTcBlk] = make_float4(hv[0], hv[1], hv[2], hv[3]);
    img[1 * (kTileFloats / 4) + kc * kTcBlk] = make_float4(lv[0], lv[1], lv[2], lv[3]);
    if (kc < kDescK / 4 - 1) img[2 * (kTileFloats / 4) + kc * kTcBlk] = make_float4(xv[0], xv[1], xv[2], xv[3]);
  }
  // the exact image has no data in dims 36..39: slot 36 carries the column's filter term kLow |x'|^2 (+inf = padding)
  img[2 * (kTileFloats / 4) + (kDescK / 4 - 1) * kTcBlk] = make_float4(q < n ? kLow * acc : INFINITY, 0.0f, 0.0f, 0.0f);
  if (q < n) norm[(size_t)cloud * V + q] = acc;  // rank order
  if (q < n && !(acc <= kTcNormMax)) fallback[cloud >> 1] = 1;
}

// Exact duplicates.  Street scenes contain hundreds of points with bit-identical descriptors (the histogram of a perfect
// plane, ...): every pair of them ties at distance 0 and would have to go through the exact chain.  Identical descriptors
// have identical norms, so after the norm sort they are neighbours: each run is collapsed to its first rank (the stable
// sort makes that the LOWEST point index, exactly the tie-break of the reference search), K6 runs on the unique
// descriptors only and broadcast_best_kernel hands the class result to every member.  One CTA per cloud.
__global__ void __launch_bounds__(1024) dedup_kernel(const float* __restrict__ desc_t, const int* __restrict__ n_vox, int V,
                                                     const uint64_t* __restrict__ sorted_keys, const uint32_t* __restrict__ perm, int enable,
                                                     uint32_t* __restrict__ uperm, uint32_t* __restrict__ class_of, int* __restrict__ n_unique) {
  __shared__ int scan_smem[33];
  const int cloud = blockIdx.x;
  const int n = n_vox[cloud];
  const float* __restrict__ D = desc_t + (size_t)cloud * kDescK * V;
  const uint32_t* __restrict__ pm = perm + (size_t)cloud * V;
  const uint64_t* __restrict__ sk = sorted_keys + (size_t)cloud * V;
  int base = 0;
  for (int start = 0; start < n; start += blockDim.x) {
    const int r = start + threadIdx.x;
    int flag = 0;
    if (r < n) {
      flag = 1;
      if (enable && r > 0 && sk[r] == sk[r - 1]) {  // same norm bits: compare the descriptors bit by bit
        const uint32_t a = pm[r], b = pm[r - 1];
        bool same = true;  // 11 dimensions per round trip (true duplicates need all 33: one dependent load pair each was 33 L2 latencies)
#pragma unroll
        for (int g = 0; g < 3; ++g) {
          if (!same) break;
          unsigned diff = 0;
#pragma unroll
          for (int j = 0; j < 11; ++j) {
            const int d = 11 * g + j;
            diff |= __float_as_uint(D[(size_t)d * V + a]) ^ __float_as_uint(D[(size_t)d * V + b]);
          }
          same = diff == 0;
        }
        flag = same ? 0 : 1;
      }
    }
    int total;
    const int ex = block_excl_scan(flag, scan_smem, &total);
    if (r < n) {
      const int u = base + ex + flag - 1;  // a duplicate belongs to the class opened by the closest earlier rank
      class_of[(size_t)cloud * V + r] = (uint32_t)u;
      if (flag) uperm[(size_t)cloud * V + u] = pm[r];
    }
    base += total;
  }
  if (threadIdx.x == 0) n_unique[cloud] = base;
}

// class results (unique-rank order) -> every point of the class, in point order for the mutual-NN stage
__global__ void __launch_bounds__(256) broadcast_best_kernel(const unsigned long long* __restrict__ rowbest_u,
                                                             const unsigned long long* __restrict__ colbest_u, const int* __restrict__ n_vox,
                                                             int V, const uint32_t* __restrict__ perm, const uint32_t* __restrict__ class_of,
                                                             unsigned long long* __restrict__ rowbest, unsigned long long* __restrict__ colbest) {
  const int cloud = blockIdx.y, pair = cloud >> 1;
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_vox[cloud]) return;
  const uint32_t u = class_of[(size_t)cloud * V + r], q = perm[(size_t)cloud * V + r];
  if (cloud & 1) colbest[(size_t)pair * V + q] = colbest_u[(size_t)pair * V + u];
  else rowbest[(size_t)pair * V + q] = rowbest_u[(size_t)pair * V + u];
}

// ---- mbarrier / bulk-copy helpers ---------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(dst), "l"(src), "r"(bytes),
               "r"(bar)
               : "memory");
}
// bounded wait: returns false if the barrier never completed (a descriptor bug must not hang the box)
__device__ __forceinline__ bool mbar_wait(uint32_t bar, uint32_t parity) {
  for (int spin = 0; spin < kSpinLimit; ++spin) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    if (ok) return true;
  }
  return false;
}

__device__ __forceinline__ unsigned long long tc_pack(float d, int idx) {
  return ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)idx;
}

// exact distance of two descriptors given as their 9 float4 chunks of the exact image (a(kc), b(kc) = bins 4 kc .. 4 kc + 3)
template <class FA, class FB>
__device__ __forceinline__ float tc_exact_dist(FA a, FB b) {
  float acc = 0.0f;
#pragma unroll
  for (int kc = 0; kc < (kDescDim + 3) / 4; ++kc) {
    const float4 x = a(kc), y = b(kc);
    acc = desc_dist_step(acc, x.x, y.x);
    if (4 * kc + 1 < kDescDim) acc = desc_dist_step(acc, x.y, y.y);
    if (4 * kc + 2 < kDescDim) acc = desc_dist_step(acc, x.z, y.z);
    if (4 * kc + 3 < kDescDim) acc = desc_dist_step(acc, x.w, y.w);
  }
  return acc;
}

// Seeds.  Every unique rank of both clouds of a pair gets the exact distance to the 2 kSeedW unique descriptors of the other
// cloud nearest to it in norm (kSeedW on either side), as a packed (distance | point index) word: rows into rowbest, columns
// into colbest, and the max of each 32-column group's seeds into tile_cmax.  Seeds are exact distances to real points, so they
// are upper bounds of the exact minima: tc_nn_kernel's filter (<=), its tile skip (strict >) and the atomicMin on packed words
// (lowest index at equal distance) leave its results unchanged, and every row and column has a finite threshold before its
// first tile.  Pairs flagged for the exact kernel are left alone.  One thread per rank; a warp is one 32-column group.
__global__ void __launch_bounds__(256) tc_seed_kernel(const float* __restrict__ tiles, const float* __restrict__ norm,
                                                      const int* __restrict__ n_vox, int V, const uint32_t* __restrict__ perm,
                                                      const int* __restrict__ fallback, unsigned long long* __restrict__ rowbest,
                                                      unsigned long long* __restrict__ colbest, unsigned* __restrict__ tile_cmax) {
  const int cloud = blockIdx.y, pair = cloud >> 1, other = cloud ^ 1;
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = n_vox[cloud], no = n_vox[other];
  // warp-uniform: every warp of a 64-column tile with a valid column writes its group's maximum, a group of padding included
  if (fallback[pair] || (r & ~(kTcN - 1)) >= n) return;
  const int NB = V / kTcBlk;
  auto image = [&](int c, int q) {  // exact image of rank q of cloud c, chunk kc at [kc * kTcBlk]
    return reinterpret_cast<const float4*>(tiles + ((size_t)(c * NB + q / kTcBlk) * kTcImages + 2) * kTileFloats) + q % kTcBlk;
  };
  unsigned long long best = ~0ull;
  if (r < n && no > 0) {
    const float4* __restrict__ ia = image(cloud, r);
    float4 own[(kDescDim + 3) / 4];
#pragma unroll
    for (int kc = 0; kc < (kDescDim + 3) / 4; ++kc) own[kc] = ia[kc * kTcBlk];
    // first rank of the other cloud whose norm is not below this one's (norms ascend with the rank)
    const float* __restrict__ nrm = norm + (size_t)other * V;
    const float key = norm[(size_t)cloud * V + r];
    int lo = 0, hi = no;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (nrm[mid] < key) lo = mid + 1; else hi = mid;
    }
    const int j1 = min(no, lo + kSeedW);
    for (int j = max(0, lo - kSeedW); j < j1; ++j) {
      const float4* __restrict__ ib = image(other, j);
      const float d = tc_exact_dist([&](int kc) { return own[kc]; }, [&](int kc) { return ib[kc * kTcBlk]; });
      if (d == d) best = min(best, tc_pack(d, (int)perm[(size_t)other * V + j]));  // NaN never wins
    }
  }
  if (cloud & 1) {
    if (r < n) colbest[(size_t)pair * V + r] = best;
    // padding columns do not count (as in tc_nn_kernel's refresh); a column without a seed keeps its group above +inf
    const unsigned m = __reduce_max_sync(0xffffffffu, r < n ? (unsigned)(best >> 32) : 0u);
    if ((threadIdx.x & 31) == 0) tile_cmax[((size_t)pair * (V / kTcN) + r / kTcN) * 2 + ((r / 32) & 1)] = m;
  } else if (r < n) {
    rowbest[(size_t)pair * V + r] = best;
  }
}

__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar) : "memory");
}
__device__ __forceinline__ unsigned tc_fkey(float f) {  // order-preserving float -> uint, NaN last
  unsigned key = __float_as_uint(f);
  key = (key & 0x80000000u) ? ~key : (key | 0x80000000u);
  return f == f ? key : 0xFFFFFFFFu;
}
__device__ __forceinline__ float tc_fkey_inv(unsigned key) { return __uint_as_float((key & 0x80000000u) ? (key & 0x7FFFFFFFu) : ~key); }

// rows = source cloud (2*pair), columns = target cloud (2*pair+1): their UNIQUE descriptors in ascending-norm (rank) order;
// n_vox / perm are the per-cloud unique counts and the point index of every unique rank.  rowbest / colbest_r are indexed by
// unique rank (broadcast_best_kernel maps them back) and hold tc_seed_kernel's seeds on entry, tile_cmax their column maxima.
// kDbg: additionally
// dump d~ of every tile of stripe 0 (validation hook, at most 128 x 128 descriptors).
//
// Warp roles (no CTA-wide barrier inside the tile loop, everything is handed over through mbarriers):
//   warp 9       : schedule warp.  Picks the stripe's next column tile, nearest norm range first, and SKIPS a tile when
//                  its lower bound (gap between the norm ranges)^2 exceeds every current best of the stripe's rows and of
//                  the tile's columns; issues the exact-image copies (2 stages)
//   warp 8       : operand-copy warp (A images once, hi | lo images of every decided tile, 1 stage)
//   warps 0..7   : warpgroup g = warps 4g .. 4g+3 owns rows 64 g .. +63 and the 64 columns of every tile; warp w of it
//                  holds the accumulators of 16 of those rows (wgmma fragment).  15 wgmma -> release the operand stage ->
//                  branch-free filter -> the warp's survivors are compacted into batches of 32 and evaluated exactly,
//                  ONE CANDIDATE PER LANE -> release the exact-image stage.
// Two CTAs share an SM: the tensor core works for one while the other filters and evaluates, so one operand stage is enough
// (the next tile's operands load during this tile's filter and evaluation).
// kProf: clock64 accounting of every role's waits into stats[8..31] (tools/tc_profile.py; QB200_TC_PROF=1)
template <bool kDbg, bool kProf = false>
__global__ void __launch_bounds__(kTcThreads, 2)
tc_nn_kernel(const float* __restrict__ tiles, const float* __restrict__ norm, const int* __restrict__ n_vox, int V,
             const uint32_t* __restrict__ perm, unsigned long long* __restrict__ rowbest, unsigned long long* __restrict__ colbest_r,
             unsigned* __restrict__ tile_cmax, int* __restrict__ fallback, unsigned long long* __restrict__ stats,
             float* __restrict__ dbg_tile) {
  extern __shared__ __align__(128) unsigned char smem[];  // 100 KB of operand images; two CTAs (static + dynamic + 1 KB each) fit in 228 KB
  __shared__ uint64_t s_fullx[kTcStages], s_sfree[kTcStages], s_fullhl, s_mma[kTcDone], s_afull;
  __shared__ unsigned long long s_rbest[kTcM];                 // best exact (distance | target index) per row of the stripe
  __shared__ __align__(16) float s_wcj[kTcEpiWarps][kTcN];     // per warp: threshold of each of the tile's 64 columns (best exact distance)
  __shared__ unsigned short s_queue[kTcEpiWarps][32];          //           one batch of candidates (lane << 5 | fragment index)
  __shared__ int s_seq[8];                                     // column tile of sequence position n (ring), -1 = end of the stripe
  __shared__ float s_tlb[kTcSmemTiles];                        // lower bound of every distance between the stripe and column tile t
  __shared__ int s_dead, s_abort, s_evals, s_npos;
  __shared__ int s_ndec;                                       // sequence positions 0 .. s_ndec-1 have been decided (s_seq ring)

  const int pair = blockIdx.y, stripe = blockIdx.x;
  const int cloudA = 2 * pair, cloudB = 2 * pair + 1;
  const int nA = n_vox[cloudA], nB = n_vox[cloudB];
  const int r0 = stripe * kTcM;
  if (r0 >= nA || nB <= 0) return;  // uniform for the CTA, before any barrier / allocation

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int NB = V / kTcBlk;
  auto tick = [&]() -> long long { return kProf ? clock64() : 0ll; };
  auto prof = [&](int slot, long long cyc) { if (kProf && lane == 0) atomicAdd(stats + slot, (unsigned long long)cyc); };
  const long long t_begin = tick();
  // shared-memory map: A (2 blocks of hi | lo | exact, 60 KB) | 1 stage of B (hi | lo, 20 KB) | 2 stages of B exact images
  // (10 KB each).  The operand images are dead as soon as the MMAs of their tile completed, the exact image only when every
  // warp evaluated the tile.
  constexpr uint32_t kABytes = (kTcM / kTcBlk) * kTcImages * kTcTileBytes;
  constexpr uint32_t kHLBytes = 2 * kTcTileBytes;
  constexpr uint32_t kXBytes = kTcTileBytes;
  const uint32_t sA = smem_u32(smem), sHL = sA + kABytes, sX0 = sHL + kHLBytes;
  const float* __restrict__ tA = tiles + (size_t)cloudA * NB * kTcImages * kTileFloats;
  const float* __restrict__ tB = tiles + (size_t)cloudB * NB * kTcImages * kTileFloats;
  const float* __restrict__ nrmA = norm + (size_t)cloudA * V;   // rank order, ascending
  const float* __restrict__ nrmB = norm + (size_t)cloudB * V;
  const uint32_t* __restrict__ permA = perm + (size_t)cloudA * V;
  const uint32_t* __restrict__ permB = perm + (size_t)cloudB * V;
  unsigned long long* __restrict__ cbg = colbest_r + (size_t)pair * V;
  const uint32_t bar_fullx0 = smem_u32(&s_fullx[0]), bar_sfree0 = smem_u32(&s_sfree[0]), bar_fullhl = smem_u32(&s_fullhl),
                 bar_mma0 = smem_u32(&s_mma[0]), bar_a = smem_u32(&s_afull);
  const int n_tiles = (nB + kTcN - 1) / kTcN;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kTcStages; ++i) { mbar_init(bar_fullx0 + 8 * i, 1); mbar_init(bar_sfree0 + 8 * i, kTcEpiWarps); }
    mbar_init(bar_fullhl, 1);
    for (int i = 0; i < kTcDone; ++i) mbar_init(bar_mma0 + 8 * i, kTcEpiWarps);
    mbar_init(bar_a, 1);
    s_dead = 0; s_abort = 0; s_evals = 0; s_npos = 0; s_ndec = 0;
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  if (threadIdx.x < kTcM) s_rbest[threadIdx.x] = r0 + (int)threadIdx.x < nA ? rowbest[(size_t)pair * V + r0 + threadIdx.x] : ~0ull;  // seeds
  __syncthreads();
  const long long t_setup = tick();
  if (kProf && threadIdx.x == 0) { atomicAdd(stats + 8, 1ull); atomicAdd(stats + 10, (unsigned long long)(t_setup - t_begin)); }
  volatile int* v_dead = &s_dead;
  volatile int* v_abort = &s_abort;
  volatile int* v_seq = s_seq;
  volatile int* v_ndec = &s_ndec;
  // bounded wait until sequence position n has been decided by the scheduler warp
  auto wait_decided = [&](int n) -> bool {
    for (int spin = 0; spin < kSpinLimit; ++spin) {
      if (*v_ndec > n) { __threadfence_block(); return true; }
      __nanosleep(32);
    }
    return false;
  };
  volatile unsigned long long* v_rbest = s_rbest;

  if (warp == kTcEpiWarps) {
    // ================= operand-copy warp: A images once, then the hi | lo images of every decided position =================
    auto issue_hl = [&](int n) {  // operand images (hi | lo, 20 KB) of position n -> the operand stage; end marker: plain arrive
      const int t = v_seq[n & 7];
      if (lane != 0) return;
      if (t < 0) { mbar_arrive(bar_fullhl); return; }
      mbar_expect_tx(bar_fullhl, kHLBytes);
      bulk_g2s(sHL, tB + (size_t)t * kTcImages * kTileFloats, kHLBytes, bar_fullhl);
    };
    if (lane == 0) {
      mbar_expect_tx(bar_a, kABytes);
      bulk_g2s(sA, tA + (size_t)stripe * (kTcM / kTcBlk) * kTcImages * kTileFloats, kABytes, bar_a);
    }
    bool ok = wait_decided(0);
    if (ok) issue_hl(0);
    long long p_wm = 0, p_wd = 0;
    bool ended = !ok || v_seq[0] < 0;  // (an end marker has gone out already)
    for (int k = 0; ok && !ended; ++k) {
      // the operand stage is free once every warp completed its MMAs of position k
      const long long t0 = tick();
      ok = mbar_wait(bar_mma0 + 8 * (k & (kTcDone - 1)), (uint32_t)((k >> 2) & 1));
      const long long t1 = tick();
      p_wm += t1 - t0;
      if (ok) ok = wait_decided(k + 1);
      p_wd += tick() - t1;
      if (!ok) break;
      issue_hl(k + 1);
      ended = v_seq[(k + 1) & 7] < 0;  // that was the end marker
    }
    prof(12, p_wm); prof(28, p_wd);
    if (!ok) *v_dead = 1;
  } else if (warp == kTcEpiWarps + 1) {
    // ================= scheduler warp: chooses the tiles and issues the exact-image copies =================
    // norm range of the stripe's rows and of a column tile (ranks are sorted by norm: first / last valid entry)
    const float amin = sqrtf(nrmA[r0]), amax = sqrtf(nrmA[(r0 + kTcM < nA ? r0 + kTcM : nA) - 1]);
    auto tile_lb = [&](int t) -> float {  // lower bound of every exact distance between the stripe and column tile t
      const float bmin = sqrtf(nrmB[t * kTcN]), bmax = sqrtf(nrmB[(t * kTcN + kTcN < nB ? t * kTcN + kTcN : nB) - 1]);
      // slack: rounding of the norm chains and square roots (kTcNormRel), absolute 2e-3 for norms near 0
      const float gap = fmaxf(amin - bmax, bmin - amax) - (2.0e-3f + kTcNormRel * (amax + bmax));
      if (!(amin <= amax && bmin <= bmax)) return 0.0f;               // NaN norms: never skip
      return gap > 0.0f ? gap * gap * 0.9999f : 0.0f;
    };
    // Shared per-tile column maxima: tcm2[t][g] = an upper bound of the best exact distances of columns 32 g .. 32 g + 31 of tile t
    // (float bits; every filter warp refreshes both groups after evaluating the tile, bests only shrink).  The values of the first
    // 256 tiles (8 tiles per lane: tile 32 i + lane in pq[i]) are fetched at the END of a choice for the NEXT one, so no choice
    // waits for L2.
    constexpr int kPq = kTcSmemTiles / 32;
    const uint2* __restrict__ tcm2 = reinterpret_cast<const uint2*>(tile_cmax) + (size_t)pair * (V / kTcN);
    uint2 pq[kPq];
    auto fetch_tcm = [&]() {
#pragma unroll
      for (int i = 0; i < kPq; ++i) pq[i] = lane + 32 * i < n_tiles ? __ldcg(tcm2 + lane + 32 * i) : make_uint2(0xFFFFFFFFu, 0xFFFFFFFFu);
    };
    fetch_tcm();
    // lower bounds of all column tiles: tiles 0..255 (V <= 16384) are kept in shared memory, later ones (up to 4096 at
    // max_voxel_points = 262144) are recomputed from the norms by tlb() and their column maxima read from tcm2 in global memory;
    // the loop stride covers any count.  Start at the tile whose norm range is closest to the stripe's, then walk outwards.
    int t0 = 0;
    {
      float best = INFINITY;
      for (int t = lane; t < n_tiles; t += 32) {
        const float g = tile_lb(t);
        if (t < kTcSmemTiles) s_tlb[t] = g;
        if (g < best) { best = g; t0 = t; }
      }
      const unsigned key = __reduce_min_sync(0xffffffffu, tc_fkey(best));
      const unsigned who = __ballot_sync(0xffffffffu, tc_fkey(best) == key);
      t0 = __shfl_sync(0xffffffffu, t0, __ffs(who) - 1);
      __syncwarp();
    }
    auto tlb = [&](int t) -> float { return t < kTcSmemTiles ? s_tlb[t] : tile_lb(t); };
    int lo = t0, hi = t0 + 1;
    bool done = false;
    auto next_tile = [&]() -> int {  // warp-uniform
      // Inputs of a choice: the current worst row best of the stripe and the prefetched per-tile column maxima, seeded before
      // the first choice (+inf only in a pair flagged for the exact kernel).  A tile whose lower bound exceeds both is skipped
      // for good (bests only shrink).
      unsigned rmax = 0;
#pragma unroll
      for (int i = 0; i < kTcM / 32; ++i) {
        const int row = lane + 32 * i;
        if (r0 + row < nA) {
          const unsigned long long rb = v_rbest[row];
          rmax = max(rmax, rb == ~0ull ? 0x7F800000u : (unsigned)(rb >> 32));
        }
      }
      const float rmaxf = __uint_as_float(__reduce_max_sync(0xffffffffu, rmax));  // distances are >= 0: the bit patterns order them
      unsigned tcm[kPq];
#pragma unroll
      for (int i = 0; i < kPq; ++i) tcm[i] = max(pq[i].x, pq[i].y);
      if (*v_abort || *v_dead) return -1;
      // The walk, 32 candidates per round: lanes 0..15 look at the next 16 tiles on the left (lo, lo-1, ...), lanes 16..31 at the
      // next 16 on the right.  Lower bounds grow outwards on either side, so the next tile in nearest-first order is the first
      // one that cannot be skipped on the left or on the right, whichever has the smaller bound (left on ties); the tiles in
      // front of them are skipped for good.
      const bool is_left = lane < 16;
      while (true) {
        if (lo < 0 && hi >= n_tiles) return -1;
        const int t = is_left ? lo - lane : hi + (lane - 16);
        const bool valid = is_left ? t >= 0 : t < n_tiles;
        const float lb = valid ? tlb(t) : INFINITY;
        unsigned cm = 0xFFFFFFFFu;
        {
          const int src = t & 31, sl = (t >> 5) & (kPq - 1);
#pragma unroll
          for (int i = 0; i < kPq; ++i) {
            const unsigned a = __shfl_sync(0xffffffffu, tcm[i], src);
            if (sl == i) cm = a;
          }
          if (!valid) cm = 0xFFFFFFFFu;
          else if (t >= kTcSmemTiles) { const uint2 q = __ldcg(tcm2 + t); cm = max(q.x, q.y); }
        }
        const bool visit = valid && (lb <= 0.0f || !(lb > rmaxf) || !(lb > __uint_as_float(cm)));
        const unsigned vb = __ballot_sync(0xffffffffu, visit);
        const int fl = (vb & 0xFFFFu) ? __ffs(vb & 0xFFFFu) - 1 : 16;   // first tile to visit on either side (16 = none in this window)
        const int fr = (vb >> 16) ? __ffs(vb >> 16) - 1 : 16;
        if (fl == 16 && fr == 16) { lo -= 16; hi += 16; continue; }
        const float gl = __shfl_sync(0xffffffffu, lb, fl & 15), gh = __shfl_sync(0xffffffffu, lb, 16 + (fr & 15));
        const bool left = fr == 16 || (fl < 16 && gl <= gh);
        const int tv = left ? lo - fl : hi + fr;
        lo -= left ? fl + 1 : fl;
        hi += left ? fr : fr + 1;
        return tv;
      }
    };
    int n_issued = 0;
    auto decide = [&](int n) {  // fix the tile of sequence position n
      int t = -1;
      if (!done) {
        t = next_tile();
        if (t < 0) done = true; else ++n_issued;
      }
      if (lane == 0) {  // (no loads are in flight here: the fence is cheap)
        v_seq[n & 7] = t;
        __threadfence_block();
        *v_ndec = n + 1;
      }
      __syncwarp();
      if (!done) fetch_tcm();  // for the next choice: lands while this warp waits for the MMAs / the free exact-image stage
      return t;
    };
    auto issue_x = [&](int n) {  // exact image (10 KB) of position n -> stage n % kTcStages
      const int t = v_seq[n & 7];
      if (lane != 0) return;
      const uint32_t bar = bar_fullx0 + 8 * (n % kTcStages);
      if (t < 0) { mbar_arrive(bar); return; }
      mbar_expect_tx(bar, kXBytes);
      bulk_g2s(sX0 + (n % kTcStages) * kXBytes, tB + ((size_t)t * kTcImages + 2) * kTileFloats, kXBytes, bar);
    };
    // positions 0 .. 2 up to the end marker (the first choice is a skip test like every other one), then their exact images
    int nd = 0;
    bool end_decided = false;
    while (nd < 3 && !end_decided) end_decided = decide(nd++) < 0;
    int nx = 0;
    while (nx < kTcStages && nx < nd) issue_x(nx++);
    prof(11, tick() - t_setup);
    long long p_wm = 0, p_dec = 0, p_sf = 0;
    auto mbar_test = [&](uint32_t bar, uint32_t parity) -> bool {
      uint32_t ready;
      asm volatile(
          "{\n\t.reg .pred p;\n\t"
          "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
          "selp.u32 %0, 1, 0, p;\n\t}\n"
          : "=r"(ready)
          : "r"(bar), "r"(parity)
          : "memory");
      return __all_sync(0xffffffffu, ready != 0);
    };
    // Two duties, neither blocks the other: the exact image of position nx goes out as soon as every warp evaluated position
    // nx - kTcStages (its stage), and positions are chosen ahead (at most 3 beyond nx: the s_seq ring, and not before the MMAs of
    // position nd-3 completed, so that a choice sees the bests of the tiles before it) while that stage is still busy.
    bool ok = true;
    int idle = 0;
    long long t_idle = 0;
    while (ok && !(end_decided && nx == nd)) {
      const uint32_t bar_s = bar_sfree0 + 8 * (nx % kTcStages), par_s = (uint32_t)((nx / kTcStages - 1) & 1);
      const uint32_t bar_m = bar_mma0 + 8 * ((nd - 3) & (kTcDone - 1)), par_m = (uint32_t)(((nd - 3) >> 2) & 1);
      const bool can_x = nx < nd, can_d = !end_decided && nd < nx + 4;
      if (can_x && mbar_test(bar_s, par_s)) {
        if (kProf && idle) { (can_d ? p_wm : p_sf) += tick() - t_idle; }
        idle = 0;
        issue_x(nx);
        ++nx;
        continue;
      }
      if (can_d && mbar_test(bar_m, par_m)) {
        const long long t1 = tick();
        if (kProf && idle) { (can_x ? p_wm : p_sf) += t1 - t_idle; }
        idle = 0;
        if (decide(nd) < 0) end_decided = true;
        ++nd;
        p_dec += tick() - t1;
        continue;
      }
      // nothing is ready: poll both events (bounded)
      if (idle == 0) t_idle = tick();
      if (++idle > kSpinLimit) { ok = false; break; }
      __nanosleep(32);
    }
    prof(29, p_wm); prof(13, p_dec); prof(14, p_sf);
    if (!ok) *v_dead = 1;
    if (lane == 0) s_npos = n_issued;
  } else {
    // ================= MMA + filter / evaluation warps =================
    const int wg = warp >> 2;                                // warpgroup = 64-row block of the stripe
    const int rbase = wg * 64 + 16 * (warp & 3);            // this warp's 16 rows of the stripe
    const int cl = 2 * (lane & 3);                           // fragment d[i]: row rbase + lane / 4 + 8 ((i >> 1) & 1),
                                                             //                column 8 (i >> 2) + cl + (i & 1) of the tile
    // the accumulators hold LB_ij = d~_ij - e_ij = kLow (na' + nb') - 2 dot (split_desc_kernel); an entry is a candidate iff
    // LB_ij <= the best exact distance known for row i or for column j
    const float kLow = 1.0f - 0.5f * kTcC;
    const float kW = kTcC / kLow;                            // d~ + e = LB + kW (kLow na' + kLow nb') (kDbg dump)
    bool row_ok[2];
    float nam[2];
    unsigned oa[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int gi = r0 + rbase + (lane >> 2) + 8 * h;
      row_ok[h] = gi < nA;
      nam[h] = row_ok[h] ? kLow * nrmA[gi] : INFINITY;
      oa[h] = row_ok[h] ? permA[gi] : 0u;                    // point index of the row
    }
    const uint32_t row_bits = (row_ok[0] ? 0x33333333u : 0u) | (row_ok[1] ? 0xCCCCCCCCu : 0u);  // fragment entries of valid rows
    // the warpgroup's A block (hi | lo | exact): operand rows of the MMAs, exact image of rows 64 wg + p (index p)
    const float4* __restrict__ aex = reinterpret_cast<const float4*>(smem + (wg * kTcImages + 2) * kTcTileBytes);
    const uint32_t aH = sA + (uint32_t)(wg * kTcImages * kTcTileBytes), aL = aH + kTcTileBytes;
    float* wcj = s_wcj[warp];
    unsigned short* wq = s_queue[warp];
    int evals_w = 0;
    bool alive = mbar_wait(bar_a, 0);
    const long long t_loop = tick();
    prof(19, t_loop - t_setup);
    long long p_wx = 0, p_wmm = 0, p_ld = 0, p_prep = 0, p_fil = 0, p_ev = 0;
    int p_tiles = 0;
    // column snapshot (best | point index) of the NEXT tile, fetched while the current one is processed when the scheduler
    // has already published it (pf_tile = tile the prefetch belongs to, -1 = none).  Lane l snapshots columns l, 32 + l.
    int pf_tile = -1;
    unsigned long long pf_cb[2] = {~0ull, ~0ull};
    unsigned pf_ob[2] = {0u, 0u};
    // shared per-tile column maxima (scheduler warp): after a tile is evaluated its 64 column bests are read again, and one tile
    // later (the load has landed) their max refreshes tcm2[tile][g] of both 32-column groups g
    unsigned* __restrict__ tcmw = tile_cmax + ((size_t)pair * (V / kTcN)) * 2;
    int rr_tile = -1;
    unsigned rr_val[2] = {0u, 0u};
    auto rr_flush = [&]() {
      if (rr_tile < 0) return;
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const unsigned m = __reduce_max_sync(0xffffffffu, rr_val[s]);
        if (lane == 0) atomicMin(tcmw + (size_t)rr_tile * 2 + s, m);
      }
      rr_tile = -1;
    };
    for (int k = 0;; ++k) {
      const int ts = k & (kTcDone - 1), st = k % kTcStages;
      const long long q0 = tick();
      if (alive) alive = mbar_wait(bar_fullx0 + 8 * st, (uint32_t)((k / kTcStages) & 1));  // the exact image is read below
      const long long q1 = tick();
      p_wx += q1 - q0;
      alive = __all_sync(0xffffffffu, alive);
      const int jt = alive ? v_seq[k & 7] : -1;
      const int c0 = jt * kTcN;
      // snapshot of the columns' bests and their point indices; the loads overlap the wait for the operands and the MMAs
      unsigned long long cb_cur[2] = {~0ull, ~0ull};
      unsigned ob[2] = {0u, 0u};
      if (jt >= 0) {
        if (pf_tile == jt) {
#pragma unroll
          for (int s = 0; s < 2; ++s) { cb_cur[s] = pf_cb[s]; ob[s] = pf_ob[s]; }
        } else {
#pragma unroll
          for (int s = 0; s < 2; ++s)
            if (c0 + 32 * s + lane < nB) {
              cb_cur[s] = __ldcg(cbg + c0 + 32 * s + lane);
              ob[s] = permB[c0 + 32 * s + lane];
            }
        }
        pf_tile = -1;
        // the next position is normally decided already (the scheduler runs 3 ahead): start its snapshot loads now
        if (__all_sync(0xffffffffu, *v_ndec > k + 1)) {  // (volatile shared loads of one warp are performed in order: no fence,
          const int jn = v_seq[(k + 1) & 7];               //  which would wait for this warp's global loads in flight)
          if (jn >= 0) {
            pf_tile = jn;
#pragma unroll
            for (int s = 0; s < 2; ++s) {
              pf_cb[s] = ~0ull; pf_ob[s] = 0u;
              if (jn * kTcN + 32 * s + lane < nB) {
                pf_cb[s] = __ldcg(cbg + jn * kTcN + 32 * s + lane);
                pf_ob[s] = permB[jn * kTcN + 32 * s + lane];
              }
            }
          }
        }
      }
      const long long q2 = tick();
      if (alive && jt >= 0) alive = mbar_wait(bar_fullhl, (uint32_t)(k & 1));  // operand images of the tile
      alive = __all_sync(0xffffffffu, alive);
      if (!wg_all(alive && jt >= 0, wg)) {  // end of the stripe, or a barrier that never completed: the warpgroup leaves together
        if (!alive) *v_dead = 1;
        break;
      }
      // ---- 15 wgmma: small cross terms first, then hi.hi
      float d[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) d[i] = 0.0f;
      {
        constexpr uint32_t kKB = 2 * kTcBlk * 16;  // bytes per K block of 8 (two 4-wide K chunks)
        const uint32_t bH = sHL, bL = bH + kTcTileBytes;
        asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory");
#pragma unroll
        for (int kb = 0; kb < kTcKB; ++kb) {
          wgmma_tf32_64x64x8(d, tc_smem_desc(aH + kb * kKB), tc_smem_desc(bL + kb * kKB), kb > 0);
          wgmma_tf32_64x64x8(d, tc_smem_desc(aL + kb * kKB), tc_smem_desc(bH + kb * kKB), 1);
        }
#pragma unroll
        for (int kb = 0; kb < kTcKB; ++kb) wgmma_tf32_64x64x8(d, tc_smem_desc(aH + kb * kKB), tc_smem_desc(bH + kb * kKB), 1);
        asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory");
        asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory");
#pragma unroll
        for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[i])::"memory");
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_mma0 + 8 * ts);  // this warp no longer reads the operand stage
      const long long q3 = tick();
      p_wmm += q3 - q2;
      p_prep += q2 - q1;
      ++p_tiles;
      const bool skip = __any_sync(0xffffffffu, (*v_abort | *v_dead) != 0);
      const long long q4 = tick();
      p_ld += q4 - q3;
      if (!skip) {
        const float4* __restrict__ bex = reinterpret_cast<const float4*>(smem + kABytes + kHLBytes + st * kXBytes);  // exact image
        // ---- per-column filter data of the lane's two snapshot columns
        float dbest[2];
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          const float nbm = bex[9 * kTcBlk + 32 * s + lane].x;  // kLow |b'_j|^2, +inf for padded columns (split_desc_kernel)
          dbest[s] = cb_cur[s] == ~0ull ? INFINITY : __uint_as_float((unsigned)(cb_cur[s] >> 32));
          wcj[32 * s + lane] = nbm == INFINITY ? -INFINITY : dbest[s];  // column threshold: the seed or a better exact distance
        }
        float Ri[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const unsigned long long rb = v_rbest[rbase + (lane >> 2) + 8 * h];
          Ri[h] = rb == ~0ull ? INFINITY : __uint_as_float((unsigned)(rb >> 32));  // +inf: no seed (a pair flagged for the exact kernel)
        }
        __syncwarp();
        const long long q5 = tick();
        p_prep += q5 - q4;
        // ---- branch-free filter of the lane's 32 entries: two compares and a predicated OR per entry
        const int ncol = nB - c0;  // valid columns of the tile (padding never competes, see below)
        uint32_t mask = 0, col_bits = 0;
#pragma unroll
        for (int i = 0; i < 32; i += 4) {
          const float2 x = *reinterpret_cast<const float2*>(wcj + 2 * i + cl);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float lbv = d[i + e];
            const float xc = (e & 1) ? x.y : x.x;
            asm("{\n\t.reg .pred p, q;\n\t"
                "setp.le.f32 p, %1, %2;\n\t"
                "setp.le.or.f32 q, %1, %3, p;\n\t"
                "@q or.b32 %0, %0, %4;\n\t}\n"
                : "+r"(mask)
                : "f"(lbv), "f"(xc), "f"(Ri[e >> 1]), "r"(1u << (i + e)));
            if (2 * i + cl + (e & 1) < ncol) col_bits |= 1u << (i + e);
            if (kDbg) {
              const int h = e >> 1, c = 2 * i + cl + (e & 1);
              if (stripe == 0 && row_ok[h] && c < ncol)  // 128 x 128 dump, row = source point
                dbg_tile[(size_t)oa[h] * 128 + permB[c0 + c]] = fmaf(0.5f * kW, nam[h] + bex[9 * kTcBlk + c].x, lbv);
            }
          }
        }
        // padding never competes: a padded row (-inf thresholds) would pass the column test of a column without a best
        // (-inf <= -inf), a padded column (+inf terms) the row test of a row without one -- and their zero images look
        // like the all-zero descriptor of an isolated point
        mask &= col_bits & row_bits;
        // ---- exact evaluation, one candidate per lane, 32 per round
        int remaining = __reduce_add_sync(0xffffffffu, __popc(mask));
        const long long q6 = tick();
        p_fil += q6 - q5;
        evals_w += remaining;
        while (remaining > 0) {  // warp-uniform
          int tot;
          int p = warp_excl_scan(__popc(mask), &tot);
          while (mask && p < 32) {
            const int i = __ffs(mask) - 1;
            mask &= mask - 1;
            wq[p++] = (unsigned short)((lane << 5) | i);
          }
          __syncwarp();
          const int nb = tot < 32 ? tot : 32;
          const int q = lane < nb ? wq[lane] : 0;
          const int sl = q >> 5, i = q & 31, h = (i >> 1) & 1;
          const int rr = rbase + (sl >> 2) + 8 * h;            // row of the stripe
          const int c = 8 * (i >> 2) + 2 * (sl & 3) + (i & 1);  // column of the tile
          const float acc = tc_exact_dist([&](int kc) { return aex[kc * kTcBlk + (rr & (kTcBlk - 1))]; },
                                          [&](int kc) { return bex[kc * kTcBlk + c]; });
          // column data live in lane c & 31 (snapshot s = c >> 5), row point indices in lane sl & ~3 (h)
          const float db0 = __shfl_sync(0xffffffffu, dbest[0], c & 31), db1 = __shfl_sync(0xffffffffu, dbest[1], c & 31);
          const unsigned ob0 = __shfl_sync(0xffffffffu, ob[0], c & 31), ob1 = __shfl_sync(0xffffffffu, ob[1], c & 31);
          const unsigned oa0 = __shfl_sync(0xffffffffu, oa[0], sl & ~3), oa1 = __shfl_sync(0xffffffffu, oa[1], sl & ~3);
          const float dbc = c < 32 ? db0 : db1;
          const unsigned oc = c < 32 ? ob0 : ob1;  // point index of the candidate's column
          const unsigned orow = h ? oa1 : oa0;      // ... and of its row
          if (lane < nb && acc == acc) {  // NaN never wins
            const unsigned long long pr = tc_pack(acc, (int)oc);
            if (pr < v_rbest[rr]) atomicMin(&s_rbest[rr], pr);
            if (acc <= dbc) atomicMin(cbg + c0 + c, tc_pack(acc, (int)orow));
          }
          __syncwarp();
          remaining = tot - nb;
        }
        // massive ties: once more than half of the entries seen needed the exact chain (after at least 8 x 128 x 128 entries),
        // hand the pair to the exact kernel
        if (lane == 0 && evals_w) {
          const int seen = atomicAdd(&s_evals, evals_w) + evals_w;
          if ((k + 1) * (kTcM * kTcN) >= 8 * 128 * 128 && seen > (k + 1) * (kTcM * kTcN / 2)) *v_abort = 1;
        }
        evals_w = 0;
        p_ev += tick() - q6;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_sfree0 + 8 * st);  // the exact-image stage may be refilled
      rr_flush();
      if (!skip) {
        rr_tile = jt;
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          rr_val[s] = 0;  // padding columns do not count
          if (c0 + 32 * s + lane < nB) {
            const unsigned long long cbn = __ldcg(cbg + c0 + 32 * s + lane);
            rr_val[s] = cbn == ~0ull ? 0x7F800000u : (unsigned)(cbn >> 32);
          }
        }
      }
    }
    rr_flush();
    prof(20, p_wx); prof(21, p_wmm); prof(22, p_ld); prof(23, p_prep); prof(24, p_fil); prof(25, p_ev);
    prof(26, tick() - t_loop); prof(27, p_tiles);
  }
  __syncthreads();
  const bool aborted = (s_abort | s_dead) != 0;
  if (kProf && threadIdx.x == 0) atomicAdd(stats + 9, (unsigned long long)(tick() - t_begin));
  if (threadIdx.x == 0) {
    atomicAdd(stats + 0, (unsigned long long)s_evals);
    atomicAdd(stats + 1, (unsigned long long)s_npos);
    if (aborted) {
      atomicAdd(stats + 3, 1ull);
      fallback[pair] = 1;
    }
  }
  if (!aborted && threadIdx.x < kTcM && r0 + (int)threadIdx.x < nA) rowbest[(size_t)pair * V + r0 + threadIdx.x] = s_rbest[threadIdx.x];
}

// A (2 blocks x 3 images) + operand stage (hi | lo) + exact-image stages = 100 KB
static size_t tc_smem_bytes() {
  return ((size_t)(kTcM / kTcBlk) * kTcImages + 2 + kTcStages) * kTcTileBytes;
}

// dynamic shared memory of tc_nn_kernel and a shared-memory-first carveout, so that two CTAs fit on every SM
static int tc_prepare(Lane* h, const void* kernel) {
  QB_CUDA_TRY(h, ensure_dyn_smem(h->device, kernel, tc_smem_bytes()));
  QB_CUDA_TRY(h, cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  return QB200_OK;
}

// threads, dynamic and static shared bytes, registers per thread and resident CTAs per SM of tc_nn_kernel as launched
int tc_footprint(Lane* h, int* out5) {
  const void* kernel = (const void*)tc_nn_kernel<false>;
  if (int rc = tc_prepare(h, kernel)) return rc;
  cudaFuncAttributes fa;
  QB_CUDA_TRY(h, cudaFuncGetAttributes(&fa, kernel));
  int ctas = 0;
  QB_CUDA_TRY(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, kernel, kTcThreads, tc_smem_bytes()));
  out5[0] = kTcThreads;
  out5[1] = (int)tc_smem_bytes();
  out5[2] = (int)fa.sharedSizeBytes;
  out5[3] = fa.numRegs;
  out5[4] = ctas;
  return QB200_OK;
}

// norm keys -> one radix sort for all clouds (h->val_b = rank -> point) -> duplicate classes.
// Scratch (free once the sort consumed its inputs): val_a = unique rank -> point, key_a = [class of rank | unique counts].
static int sort_and_dedup(Lane* h, int n_clouds, int dedup, const int* n_pts) {
  const int V = h->V;
  const dim3 g((V + 255) / 256, n_clouds);
  norm_key_kernel<<<g, 256, 0, h->stream>>>(h->desc_t, n_pts, V, h->key_a, h->val_a);
  h->launches += 1;
  int bits = 0;
  while ((1 << bits) < n_clouds) ++bits;
  int rc = launch_cloud_sort(h, n_clouds, n_pts, 32, 32);  // per-cloud shared-memory sort; device-wide radix sort for very large clouds
  if (rc == QB200_ERR_UNSUPPORTED) rc = sort_pairs(h, n_clouds * V, 32 + bits);
  if (rc) return rc;
  dedup_kernel<<<n_clouds, 1024, 0, h->stream>>>(h->desc_t, n_pts, V, h->key_b, h->val_b, dedup, h->val_a, h->class_of(), h->n_unique());
  h->launches += 1;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

int launch_match_nn(Lane* h, int n_pairs, const int* n_pts) {
  const int V = h->V;
  const size_t smem = tc_smem_bytes();
  if (int rc = tc_prepare(h, (const void*)tc_nn_kernel<false>)) return rc;
  int rc = sort_and_dedup(h, 2 * n_pairs, 1, n_pts);
  if (rc) return rc;
  const uint32_t* uperm = h->val_a;
  const uint32_t* class_of = h->class_of();
  const int* n_unique = h->n_unique();
  // class results, indexed by unique rank (colpart is this kernel's scratch; the exact fallback works in rowbest / colbest)
  unsigned long long* colbest_u = h->colpart_col();
  unsigned long long* rowbest_u = h->colpart_row();
  unsigned* tile_cmax = h->colpart_tile_cmax();  // [S][V/64][2] float bits: the seeds' column maxima
  QB_CUDA_TRY(h, cudaMemsetAsync(h->rowbest, 0xFF, (size_t)n_pairs * V * 8, h->stream));
  QB_CUDA_TRY(h, cudaMemsetAsync(h->colbest, 0xFF, (size_t)n_pairs * V * 8, h->stream));
  QB_CUDA_TRY(h, cudaMemsetAsync(h->colpart, 0xFF, h->colpart_count() * 8, h->stream));  // 0xFFFFFFFF > +inf bits
  QB_CUDA_TRY(h, cudaMemsetAsync(h->tc_fallback, 0, (size_t)n_pairs * sizeof(int), h->stream));
  const dim3 gsplit((V + 255) / 256, 2 * n_pairs);
  split_desc_kernel<<<gsplit, 256, 0, h->stream>>>(h->desc_t, n_unique, V, uperm, h->desc_tiles, h->desc_norm, h->tc_fallback);
  tc_seed_kernel<<<gsplit, 256, 0, h->stream>>>(h->desc_tiles, h->desc_norm, n_unique, V, uperm, h->tc_fallback, rowbest_u, colbest_u, tile_cmax);
  const dim3 g(h->NS, n_pairs);
  cudaEventRecord(h->kev[0], h->stream);
  if (h->tc_prof) {
    if (int rc2 = tc_prepare(h, (const void*)tc_nn_kernel<false, true>)) return rc2;
    tc_nn_kernel<false, true><<<g, kTcThreads, smem, h->stream>>>(h->desc_tiles, h->desc_norm, n_unique, V, uperm, rowbest_u, colbest_u,
                                                                  tile_cmax, h->tc_fallback, h->tc_stats, nullptr);
  } else {
    tc_nn_kernel<false><<<g, kTcThreads, smem, h->stream>>>(h->desc_tiles, h->desc_norm, n_unique, V, uperm, rowbest_u, colbest_u,
                                                            tile_cmax, h->tc_fallback, h->tc_stats, nullptr);
  }
  cudaEventRecord(h->kev[1], h->stream);
  h->kev_armed[0] = 1;
  broadcast_best_kernel<<<gsplit, 256, 0, h->stream>>>(rowbest_u, colbest_u, n_pts, V, h->val_b, class_of, h->rowbest, h->colbest);
  h->launches += 4;
  QB_CUDA_TRY(h, cudaGetLastError());
  return launch_match_exact(h, n_pairs, h->tc_fallback, n_pts);
}

// debug/validation hook: approximate distances d~ of stripe 0 of pair 0, both 64-column tiles of up to 128 x 128 descriptors
// (descriptors already in desc_t; duplicates are kept so that every (row, column) of the dump is filled)
int launch_tc_debug_tile(Lane* h, float* d_out) {
  const size_t smem = tc_smem_bytes();
  if (int rc0 = tc_prepare(h, (const void*)tc_nn_kernel<true>)) return rc0;
  int rc = sort_and_dedup(h, 2, 0, h->ctr.n_vox);
  if (rc) return rc;
  const uint32_t* uperm = h->val_a;
  const int* n_unique = h->n_unique();
  QB_CUDA_TRY(h, cudaMemsetAsync(h->colpart, 0xFF, h->colpart_count() * 8, h->stream));
  QB_CUDA_TRY(h, cudaMemsetAsync(h->tc_fallback, 0, sizeof(int), h->stream));
  const dim3 gsplit((h->V + 255) / 256, 2);
  split_desc_kernel<<<gsplit, 256, 0, h->stream>>>(h->desc_t, n_unique, h->V, uperm, h->desc_tiles, h->desc_norm, h->tc_fallback);
  tc_seed_kernel<<<gsplit, 256, 0, h->stream>>>(h->desc_tiles, h->desc_norm, n_unique, h->V, uperm, h->tc_fallback, h->colpart_row(),
                                                h->colpart_col(), h->colpart_tile_cmax());
  const dim3 g(1, 1);
  tc_nn_kernel<true><<<g, kTcThreads, smem, h->stream>>>(h->desc_tiles, h->desc_norm, n_unique, h->V, uperm, h->colpart_row(), h->colpart_col(),
                                                         h->colpart_tile_cmax(), h->tc_fallback, h->tc_stats, d_out);
  h->launches += 3;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

}  // namespace qb
