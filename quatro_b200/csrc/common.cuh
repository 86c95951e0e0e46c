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
constexpr int kVoxShift = 31;
constexpr uint64_t kVoxMask = (1ull << kVoxShift) - 1;
constexpr uint64_t kVoxInvalid = kVoxMask;  // dx dy dz <= INT_MAX: a valid index is at most 2^31 - 2
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

// number of 8-bit digits the voxel keys of a cloud occupy: the keys are below dx dy dz of pcl::VoxelGrid's own linear index
// (voxel_pack uses the same min_b / div_b expressions)
__device__ __forceinline__ int vox_digits(const int* __restrict__ bbox, int n_valid, float inv_leaf) {
  if (n_valid <= 0) return 0;
  const long long m0 = (long long)floorf(ordered_float(bbox[0]) * inv_leaf), m1 = (long long)floorf(ordered_float(bbox[1]) * inv_leaf),
                  m2 = (long long)floorf(ordered_float(bbox[2]) * inv_leaf);
  const long long d0 = (long long)floorf(ordered_float(bbox[3]) * inv_leaf) - m0 + 1, d1 = (long long)floorf(ordered_float(bbox[4]) * inv_leaf) - m1 + 1,
                  d2 = (long long)floorf(ordered_float(bbox[5]) * inv_leaf) - m2 + 1;
  unsigned long long span = (unsigned long long)d0 * (unsigned long long)d1;   // each factor < 2^18 (cell_ok)
  if (span > (1ull << 31) || span * (unsigned long long)d2 > (1ull << 31)) return 4;  // refused by run_heads (overflow); any order will do
  span *= (unsigned long long)d2;
  int bits = 0;
  while (bits < 31 && (1ull << bits) < span) ++bits;
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
