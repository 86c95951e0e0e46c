// voxsort.cu -- K1: the voxel sort of a wave as a per-cloud, multi-CTA radix sort over the KEPT points only (sm_90a).
//
// Round 1 sorted (cloud | voxel | index) keys of EVERY raw point of the wave with cub::DeviceRadixSort (onesweep: 5 passes over
// 38 key bits, 13 % of a street wave) although (a) the points the voxel filter drops (non-finite, flagged ground: 3 of 4
// returns of a street scan) never need sorting, (b) a cloud's keys only span the bits of ITS lattice, dx dy dz (24 bits for a
// 160 x 160 x 10 m scan at a 0.3 m leaf), and (c) clouds never mix, so the cloud id needs no key bits.  Sizes are device-side
// (no host round trip), so this cannot be expressed as one library call.  Here:
//
//   voxel_bbox_kernel (frontend.cu)  also counts the kept points of each of the 64 contiguous chunks of a scan
//   voxel_pack_kernel                (voxel | index) items of the kept points, written COMPACTED in scan order (chunk base =
//                                    sum of the preceding chunk counts, block scans inside the chunk)
//   per 8-bit digit of the cloud's lattice bits (<= 4, the grid is launched for 4 and clouds that need fewer leave early):
//     vsort_hist_kernel     digit histogram of every 2048-item tile
//     vsort_scan_kernel     exclusive scan in (digit, tile) order: one CTA per cloud
//     vsort_scatter_kernel  stable scatter: per-warp digit histograms (match.any), warp bases by digit, second walk
//   The result of a cloud with an odd number of digits lies in the B array, otherwise in A (vox_sorted()).
//
// HBM traffic per kept point: 8 B written by the pack pass, 24 B per digit (histogram read, scatter read + write) -- for a street
// wave (27 % kept, 3 digits) 21 B per RAW point instead of 8 + 5 x 16 = 88 B.  Stable: equal voxels keep ascending point index,
// which is what makes the in-order centroid sum of voxel_centroid_kernel bit-identical to the sequential CPU sum.
#include "handle.cuh"

namespace qb {

constexpr int kVsThreads = 256;

// (voxel << idx_bits | index) of the kept points of one chunk, compacted in scan order.  grid = (kVsChunks, clouds).
__global__ void __launch_bounds__(kVsThreads) voxel_pack_kernel(const float4* const* __restrict__ cloud_ptr, const int* __restrict__ cloud_n,
                                                                const int* __restrict__ raw_off, const CloudFront* __restrict__ front,
                                                                const int* __restrict__ bbox, const int* __restrict__ n_valid,
                                                                const int* __restrict__ chunk_cnt, int idx_bits, uint64_t* __restrict__ items) {
  __shared__ int sm[33];
  const int cloud = blockIdx.y, chunk = blockIdx.x, tid = threadIdx.x;
  const int n = cloud_n[cloud], off = raw_off[cloud];
  const int cs = vox_chunk_size(n);
  const int c0 = chunk * cs, c1 = min(n, c0 + cs);
  if (c0 >= n) return;
  const float4* __restrict__ pts = cloud_ptr[cloud];
  const float inv_leaf = front[cloud].inv_leaf;
  const int skip_flagged = front[cloud].skip_flagged;
  long long m[3] = {0, 0, 0}, d[3] = {1, 1, 1}, top;  // min_b / div_b of pcl::VoxelGrid::applyFilter
  const bool grid_ok = n_valid[cloud] > 0 && vox_grid(bbox + cloud * 6, inv_leaf, m, d, &top);
  const float lo[3] = {(float)m[0], (float)m[1], (float)m[2]};  // exact: min_b is the float floor of the bbox corner
  int base = 0;  // kept points of the preceding chunks
  {
    int v = 0;
    for (int k = tid; k < chunk; k += kVsThreads) v += chunk_cnt[cloud * kVsChunks + k];
    int tot;
    block_excl_scan(v, sm, &tot);
    base = tot;
  }
  constexpr int kPer = 4;
  for (int r0 = c0; r0 < c1; r0 += kPer * kVsThreads) {
    const int i0 = r0 + kPer * tid;
    uint64_t it[kPer];
    int keep[kPer], nk = 0;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int i = i0 + j;
      keep[j] = 0; it[j] = 0;
      if (i < c1) {
        const float4 p = __ldg(pts + i);
        if (raw_point_kept(p, skip_flagged)) {  // exactly the points the bbox pass counted
          uint64_t cell = kVoxInvalid;         // refused cloud: run_heads drops it, any key will do
          if (grid_ok) {                       // every ijk fits an int and the index is at most INT_MAX
            // PCL: ijk = static_cast<int>(floor(p * inv) - static_cast<float>(min_b)), the subtraction in float
            const long long ci = (int)__fsub_rn(floorf(p.x * inv_leaf), lo[0]), cj = (int)__fsub_rn(floorf(p.y * inv_leaf), lo[1]),
                            ck = (int)__fsub_rn(floorf(p.z * inv_leaf), lo[2]);
            cell = (uint64_t)(ci + cj * d[0] + ck * d[0] * d[1]);
          }
          it[j] = (cell << idx_bits) | (uint64_t)i;
          keep[j] = 1;
        }
      }
      nk += keep[j];
    }
    int tot;
    int pos = base + block_excl_scan(nk, sm, &tot);
#pragma unroll
    for (int j = 0; j < kPer; ++j)
      if (keep[j]) items[off + pos++] = it[j];
    base += tot;
  }
}

// tile histograms of digit `pass`.  hist[cloud][digit][tile], tiles_cap tiles per cloud.  grid = (tiles_cap, clouds).
__global__ void __launch_bounds__(kVsThreads) vsort_hist_kernel(int pass, const uint64_t* __restrict__ a, const uint64_t* __restrict__ b,
                                                                const int* __restrict__ raw_off, const int* __restrict__ bbox,
                                                                const int* __restrict__ n_valid, const CloudFront* __restrict__ front, int idx_bits,
                                                                int tiles_cap, unsigned* __restrict__ hist) {
  __shared__ unsigned s_h[256];
  const int cloud = blockIdx.y, tile = blockIdx.x, tid = threadIdx.x;
  const int m = n_valid[cloud];
  if (tile * kVsTile >= m || pass >= vox_digits(bbox + cloud * 6, m, front[cloud].inv_leaf)) return;
  const uint64_t* __restrict__ src = ((pass & 1) ? b : a) + raw_off[cloud];
  s_h[tid] = 0u;
  __syncthreads();
  const int shift = idx_bits + 8 * pass;
  const int t0 = tile * kVsTile, t1 = min(m, t0 + kVsTile);
  for (int i = t0 + tid; i < t1; i += kVsThreads) atomicAdd(&s_h[(unsigned)(src[i] >> shift) & 255u], 1u);
  __syncthreads();
  hist[((size_t)cloud * 256 + tid) * tiles_cap + tile] = s_h[tid];
}

// exclusive scan of hist[cloud] in (digit, tile) order, in place.  One CTA per cloud.
__global__ void __launch_bounds__(1024) vsort_scan_kernel(int pass, const int* __restrict__ bbox, const int* __restrict__ n_valid,
                                                          const CloudFront* __restrict__ front, int tiles_cap, unsigned* __restrict__ hist) {
  __shared__ int sm[33];
  const int cloud = blockIdx.x, tid = threadIdx.x;
  const int m = n_valid[cloud];
  if (m <= 0 || pass >= vox_digits(bbox + cloud * 6, m, front[cloud].inv_leaf)) return;
  const int nt = (m + kVsTile - 1) / kVsTile;     // live tiles: the entries of the others were never written
  unsigned* __restrict__ H = hist + (size_t)cloud * 256 * tiles_cap;
  const int total = 256 * nt;                     // flattened (digit, live tile)
  int carry = 0;
  constexpr int kPer = 8;
  for (int base = 0; base < total; base += kPer * 1024) {
    const int e0 = base + kPer * tid;
    int v[kPer], s = 0;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int e = e0 + j;
      v[j] = e < total ? (int)H[(size_t)(e / nt) * tiles_cap + (e % nt)] : 0;
      s += v[j];
    }
    int tot;
    int run = carry + block_excl_scan(s, sm, &tot);
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int e = e0 + j;
      if (e < total) H[(size_t)(e / nt) * tiles_cap + (e % nt)] = (unsigned)run;
      run += v[j];
    }
    carry += tot;
  }
}

// stable scatter of one tile by digit `pass`.  Item order inside a tile = (warp, round, lane): warp w owns items [256 w, 256 w + 256).
__global__ void __launch_bounds__(kVsThreads) vsort_scatter_kernel(int pass, const uint64_t* __restrict__ a, const uint64_t* __restrict__ b,
                                                                   uint64_t* __restrict__ a_out, uint64_t* __restrict__ b_out,
                                                                   const int* __restrict__ raw_off, const int* __restrict__ bbox,
                                                                   const int* __restrict__ n_valid, const CloudFront* __restrict__ front,
                                                                   int idx_bits, int tiles_cap, const unsigned* __restrict__ offs) {
  __shared__ unsigned s_w[kVsThreads / 32][256];   // per warp: digit counts, then running output positions
  const int cloud = blockIdx.y, tile = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int m = n_valid[cloud];
  if (tile * kVsTile >= m || pass >= vox_digits(bbox + cloud * 6, m, front[cloud].inv_leaf)) return;
  const uint64_t* __restrict__ src = ((pass & 1) ? b : a) + raw_off[cloud];
  uint64_t* __restrict__ dst = ((pass & 1) ? a_out : b_out) + raw_off[cloud];
  const int shift = idx_bits + 8 * pass;
  const int t0 = tile * kVsTile + warp * 256;
#pragma unroll
  for (int k = 0; k < 8; ++k) s_w[warp][lane + 32 * k] = 0u;
  __syncwarp();
  uint64_t it[8];
  int dg[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int i = t0 + r * 32 + lane;
    dg[r] = -1 - lane;                                    // idle lanes match nobody
    it[r] = 0;
    if (i < m) { it[r] = src[i]; dg[r] = (int)((unsigned)(it[r] >> shift) & 255u); }
    const unsigned peers = __match_any_sync(0xffffffffu, dg[r]);
    if (dg[r] >= 0 && (peers & ((1u << lane) - 1u)) == 0u) s_w[warp][dg[r]] += (unsigned)__popc(peers);   // the lowest lane of a digit group
    __syncwarp();
  }
  __syncthreads();
  {  // digit tid: warp bases = tile offset of the digit + counts of the lower warps
    unsigned run = offs[((size_t)cloud * 256 + tid) * tiles_cap + tile];
#pragma unroll
    for (int w = 0; w < kVsThreads / 32; ++w) {
      const unsigned c = s_w[w][tid];
      s_w[w][tid] = run;
      run += c;
    }
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const unsigned peers = __match_any_sync(0xffffffffu, dg[r]);
    if (dg[r] >= 0) {
      const unsigned rank = (unsigned)__popc(peers & ((1u << lane) - 1u));
      const unsigned pos = s_w[warp][dg[r]] + rank;
      dst[pos] = it[r];
    }
    __syncwarp();
    if (dg[r] >= 0 && (peers & ((1u << lane) - 1u)) == 0u) s_w[warp][dg[r]] += (unsigned)__popc(peers);
    __syncwarp();
  }
}

// Sort the packed items of every cloud (A = key_a, B = key_b).  Afterwards cloud c's sorted segment starts at
// (vox_digits(c) odd ? B : A) + raw_off[c] and holds n_valid[c] items.  Every kernel takes cloud c's leaf from d_front[c], so all of
// them agree on its digit count.
int launch_voxel_sort(Lane* h, int n_clouds, int idx_bits) {
  const int tiles_cap = (h->R + kVsTile - 1) / kVsTile;
  unsigned* hist = reinterpret_cast<unsigned*>(h->val_a.get());        // [clouds][256][tiles_cap]  (alloc_all sizes val_a for it)
  const int* chunk_cnt = reinterpret_cast<const int*>(h->val_b.get()); // [clouds][64]
  const dim3 gp(kVsChunks, n_clouds), gt(tiles_cap, n_clouds);
  voxel_pack_kernel<<<gp, kVsThreads, 0, h->stream>>>(h->d_cloud_ptr, h->d_cloud_n, h->d_raw_off, h->d_front, h->ctr.bbox, h->ctr.n_valid,
                                                     chunk_cnt, idx_bits, h->key_a);
  for (int pass = 0; pass < 4; ++pass) {
    vsort_hist_kernel<<<gt, kVsThreads, 0, h->stream>>>(pass, h->key_a, h->key_b, h->d_raw_off, h->ctr.bbox, h->ctr.n_valid, h->d_front, idx_bits,
                                                       tiles_cap, hist);
    vsort_scan_kernel<<<n_clouds, 1024, 0, h->stream>>>(pass, h->ctr.bbox, h->ctr.n_valid, h->d_front, tiles_cap, hist);
    vsort_scatter_kernel<<<gt, kVsThreads, 0, h->stream>>>(pass, h->key_a, h->key_b, h->key_a, h->key_b, h->d_raw_off, h->ctr.bbox, h->ctr.n_valid,
                                                          h->d_front, idx_bits, tiles_cap, hist);
  }
  h->launches += 13;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

}  // namespace qb
