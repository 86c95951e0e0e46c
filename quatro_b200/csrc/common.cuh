// common.cuh -- shared device/host declarations of libquatro_b200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "quatro_b200.h"

namespace qb {

// ------------------------------------------------------------------------------------------------
// Lattice / voxel sort keys.  A cell (i,j,k) = floorf(p * inv_cell) is packed so that unsigned
// comparison orders cells by (k, j, i) -- the order of PCL's linear voxel index
// i + j*dx + k*dx*dy ([EXT] pcl::VoxelGrid, called from include/quatro.hpp:49-57) -- and the cloud
// id sits above it so that ONE radix sort orders every cloud of a batch wave at once.
//   [63:52] cloud   [51:36] k + 2^15   [35:18] j + 2^17   [17:0] i + 2^17
// The all-ones cell value marks a dropped point (non-finite, flagged, outside the lattice).
// ------------------------------------------------------------------------------------------------
constexpr int kOffIJ = 1 << 17;
constexpr int kOffK = 1 << 15;
constexpr uint64_t kCellMask = (1ull << 52) - 1;
constexpr uint64_t kCellInvalid = kCellMask;
constexpr int kCloudShift = 52;

__host__ __device__ __forceinline__ bool cell_ok(int i, int j, int k) {
  return i >= -kOffIJ && i < kOffIJ - 1 && j >= -kOffIJ && j < kOffIJ - 1 && k >= -kOffK && k < kOffK - 1;
}
__host__ __device__ __forceinline__ uint64_t cell_key(int i, int j, int k) {
  return ((uint64_t)(k + kOffK) << 36) | ((uint64_t)(j + kOffIJ) << 18) | (uint64_t)(i + kOffIJ);
}

// ---- voxel keys (frontend.cu, voxsort.cu) ----
constexpr int kVoxShift = 32;
constexpr uint64_t kVoxMask = (1ull << kVoxShift) - 1;
constexpr uint64_t kVoxInvalid = kVoxMask;  // a valid index is at most INT_MAX (vox_grid())
constexpr int kVsChunks = 64;               // contiguous chunks of a raw scan whose kept points the bbox pass counts
constexpr int kVsTile = 2048;               // items per tile of the voxel sort (voxsort.cu): 8 warps x 8 rounds x 32 lanes

__device__ __forceinline__ bool raw_point_kept(const float4 p, int skip_flagged) {
  return isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && !(skip_flagged && p.w < 0.0f);
}
__host__ __device__ __forceinline__ int vox_chunk_size(int n) { return n > 0 ? (n + kVsChunks - 1) / kVsChunks : 1; }

constexpr int kDescDim = 33;   // pcl::FPFHSignature33
constexpr int kDescPad = 36;   // floats per SPFH row (16-byte multiple: float4 gathers)
constexpr int kDescK = 40;     // rows (K extent) of the dimension-major FPFH matrices: 33 bins + zero padding to a multiple of
                               // the TF32 tensor-core K step (8)
// One step of the matcher's exact descriptor distance: acc + (a - b)^2, the product-sum rounded once.  Every exact distance
// of the matcher (match_stripe_kernel, tc_nn_kernel's evaluation and its seeds) is the chain of these steps over bins
// 0 .. 32 in ascending order, so all of them produce the same bits.
__device__ __forceinline__ float desc_dist_step(float acc, float a, float b) {
  const float diff = a - b;
  return __fmaf_rn(diff, diff, acc);
}
constexpr int kMatchTile = 128;
constexpr int kNbrGlobalCap = 80;  // neighbour indices per point handed from K4 (SPFH) to K5 (FPFH)

// Per-cloud / per-pair counters that live on the device for a whole wave (no host round trips
// between stages).  Arrays are indexed by cloud (2 per pair: 2*s = source, 2*s+1 = target) or slot.
struct WaveCounters {
  int* n_valid;      // [clouds] points kept by the voxel key pass
  int* n_vox;        // [clouds]
  int* n_lat;        // [clouds] points inside the neighbour lattice
  int* n_cells;      // [clouds]
  int* cloud_status; // [clouds] qb200_status (0 ok)
  int* bbox;         // [clouds*6] ordered-int encoded min xyz / max xyz of kept raw points
  int* vox_digits;   // [clouds] 8-bit digits of the cloud's voxel keys (run_heads_kernel; -1: refused), read by voxel_centroid_kernel
  int* n_mutual;     // [slots]
  int* n_corr;       // [slots]
  int* swapped;      // [slots]  target cloud larger than source (feature_matcher.cc:84-89)
  int* n_clique;     // [slots]
  int* max_core;     // [slots]
  int* n_final;      // [slots]
  int* flags;        // [slots] QB200_FLAG_* bits of the pair
  long long* n_edges;// [slots]
};

#define QB_CUDA_TRY(h, expr)                                                                    \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess) {                                                                    \
      (h)->fail(__FILE__, __LINE__, cudaGetErrorString(_e));                                    \
      return QB200_ERR_CUDA;                                                                    \
    }                                                                                           \
  } while (0)

__device__ __forceinline__ int float_ordered(float f) {
  const int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7FFFFFFF;
}
__host__ __device__ __forceinline__ float ordered_float(int i) {
  const int j = i >= 0 ? i : i ^ 0x7FFFFFFF;
#ifdef __CUDA_ARCH__
  return __int_as_float(j);
#else
  float f;
  memcpy(&f, &j, 4);
  return f;
#endif
}

// a * b * c > INT_MAX for factors >= 1, without overflowing 64 bits
__host__ __device__ __forceinline__ bool vox_product_exceeds(long long a, long long b, long long c) {
  const long long lim = 2147483647LL;
  if (a > lim || b > lim || c > lim) return true;
  const long long ab = a * b;  // < 2^62
  return ab > lim || ab * c > lim;
}
// pcl::VoxelGrid's grid of a cloud from the ordered-int bbox of its kept points: min_b and div_b.  False when the cloud is refused
// with QB200_ERR_VOXEL_OVERFLOW, i.e. wherever PCL's own int arithmetic would overflow:
//   - PCL's check: the truncated spans (int64)((max - min) * inv) + 1 multiply to more than INT_MAX;
//   - a kept point's floor(p * inv) lies outside int32 (floor(p * inv) is monotone in p: the bbox corners decide);
//   - the floor-based div_b = max_b - min_b + 1, which can be one larger per axis than the truncated span, multiply to more than
//     INT_MAX (divb_mul would not fit an int);
//   - the largest linear index PCL computes exceeds INT_MAX.  PCL subtracts ijk = floor(p * inv) - (float)min_b in float, which
//     rounds once the difference passes 2^24 and can round up to div_b, so that index can exceed div_b0 div_b1 div_b2 - 1.  The
//     rounding is monotone, so the max corner gives each axis's largest ijk.
// The index is relative to min_b, so a cloud far from the origin is voxelised like the same cloud moved to the origin.
__device__ __forceinline__ bool vox_axis(int omin, int omax, float inv_leaf, long long* span, long long* min_b, long long* div_b,
                                         long long* top) {
  const float mn = ordered_float(omin), mx = ordered_float(omax);
  const float lo = floorf(mn * inv_leaf), hi = floorf(mx * inv_leaf);
  if (!(lo >= -2147483648.0f && hi < 2147483648.0f)) return false;
  const float s = (mx - mn) * inv_leaf;
  if (!(s < 2147483648.0f)) return false;  // a truncated span above INT_MAX (or +inf) fails PCL's check on its own
  *span = (long long)s + 1;
  *min_b = (long long)lo;
  *div_b = (long long)hi - *min_b + 1;
  *top = (long long)__fsub_rn(hi, lo);     // the largest ijk of the axis
  return true;
}
// *max_idx: the largest linear index of the cloud (valid when true is returned)
__device__ __forceinline__ bool vox_grid(const int* __restrict__ bbox, float inv_leaf, long long* min_b, long long* div_b,
                                         long long* max_idx) {
  long long t[3], a[3];
  for (int k = 0; k < 3; ++k)
    if (!vox_axis(bbox[k], bbox[k + 3], inv_leaf, &t[k], &min_b[k], &div_b[k], &a[k])) return false;
  if (vox_product_exceeds(t[0], t[1], t[2]) || vox_product_exceeds(div_b[0], div_b[1], div_b[2])) return false;
  *max_idx = a[0] + a[1] * div_b[0] + a[2] * div_b[0] * div_b[1];  // a[k] <= 2^31 and div_b0 div_b1 <= INT_MAX: no overflow
  return *max_idx <= 2147483647LL;
}

// number of 8-bit digits the voxel keys of a cloud occupy: the keys are at most the largest linear index of pcl::VoxelGrid
// (vox_grid(); voxel_pack uses the same min_b / div_b).  -1: the cloud is refused, nothing is sorted and run_heads drops it.
__device__ __forceinline__ int vox_digits(const int* __restrict__ bbox, int n_valid, float inv_leaf) {
  if (n_valid <= 0) return 0;
  long long m[3], d[3], top;
  if (!vox_grid(bbox, inv_leaf, m, d, &top)) return -1;
  int bits = 0;  // keys lie in [0, top], top <= INT_MAX
  while (bits < 31 && (1ll << bits) <= top) ++bits;
  return (bits + 7) >> 3;
}


__device__ __forceinline__ unsigned lane_id() { return threadIdx.x & 31; }

// exclusive prefix sum of one int per lane (32-wide), returns the exclusive value; total via *total
__device__ __forceinline__ int warp_excl_scan(int v, int* total) {
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int n = __shfl_up_sync(0xffffffffu, inc, o);
    if ((int)lane_id() >= o) inc += n;
  }
  *total = __shfl_sync(0xffffffffu, inc, 31);
  return inc - v;
}

// block-wide exclusive scan (blockDim.x multiple of 32, <= 1024). smem: 33 ints. All threads call.
__device__ __forceinline__ int block_excl_scan(int v, int* smem, int* block_total) {
  const int lane = lane_id(), warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int wt;
  const int ex = warp_excl_scan(v, &wt);
  __syncthreads();  // protect smem reuse across calls
  if (lane == 31) smem[warp] = wt;
  __syncthreads();
  if (warp == 0) {
    int t = lane < nw ? smem[lane] : 0, tot;
    const int e = warp_excl_scan(t, &tot);
    smem[lane] = e;
    if (lane == 0) smem[32] = tot;
  }
  __syncthreads();
  *block_total = smem[32];
  return ex + smem[warp];
}

}  // namespace qb
