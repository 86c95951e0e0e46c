// frontend.cu -- K1..K5: voxel down-sampling, neighbour lattice, normals, SPFH, FPFH  (sm_90a)
//
// Replaces: voxelize<T>() (include/quatro.hpp:49-57 -> [EXT] pcl::VoxelGrid) and
// FPFHEstimation::computeFPFHFeatures (src/teaser_utils/fpfh.cc:44-75 -> [EXT] pcl::NormalEstimation,
// pcl::FPFHEstimationOMP, pcl::search::KdTree).
//
// Design: every cloud of a batch wave is processed by the same launches (grid.y = cloud); sizes
// stay on the device.  Voxelisation is a stable per-cloud radix sort of the (voxel | point index) items of the KEPT
// points (voxsort.cu) followed by a segmented, in-order centroid sum (bit-identical to the sequential CPU sum).  The kd-tree is
// replaced by a sorted-cell lattice: a point's neighbours are found by (2m+1)^2 binary searches for
// x-runs of cells, visited in ascending (cell, index) order -- the accumulation order the CPU oracle
// uses, so the single-pass float covariance matches bit for bit.
#include <cub/device/device_radix_sort.cuh>
#include <type_traits>

#include "fpfh_math.cuh"
#include "handle.cuh"

namespace qb {

// ------------------------------------------------------------------------------------------------
// sort plumbing
// ------------------------------------------------------------------------------------------------
size_t sort_temp_bytes(int max_items) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr,
                                  (uint32_t*)nullptr, max_items, 0, 64, (cudaStream_t)0);
  return bytes;
}

int sort_pairs(Lane* h, int n_items, int end_bit) {
  if (n_items <= 0) return QB200_OK;
  size_t bytes = h->cub_bytes;
  QB_CUDA_TRY(h, cub::DeviceRadixSort::SortPairs(h->cub_temp.get(), bytes, h->key_a.get(), h->key_b.get(), h->val_a.get(), h->val_b.get(), n_items, 0, end_bit,
                                                 h->stream));
  h->launches += 1 + (end_bit + 7) / 8;  // onesweep: histogram + one pass per 8 key bits
  return QB200_OK;
}

static int clog2(int n) {
  int b = 0;
  while ((1 << b) < n) ++b;
  return b;
}

// ------------------------------------------------------------------------------------------------
// K1a: bounding box and per-chunk counts of the kept raw points (one pass, 128-bit loads).  The voxel key that the pack pass
// (voxsort.cu) then builds is PCL's own linear index  (i - min_i) + (j - min_j) dx + (k - min_k) dx dy  ([EXT] pcl::VoxelGrid,
// called from include/quatro.hpp:49-57, each difference taken in float as PCL does), which the library requires to fit an int: at
// most 31 key bits, and for a given cloud only the bits of its largest index (vox_digits()).  The bbox alone decides whether a
// cloud is refused (vox_grid()), so this pass keeps no per-point range test.
// ------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(256) voxel_bbox_kernel(const float4* const* __restrict__ cloud_ptr, const int* __restrict__ cloud_n,
                                                         const CloudFront* __restrict__ front, int* __restrict__ bbox,
                                                         int* __restrict__ n_valid, int* __restrict__ chunk_cnt) {
  const int cloud = blockIdx.y;
  const int n = cloud_n[cloud];
  const int skip_flagged = front[cloud].skip_flagged;
  const float4* __restrict__ pts = cloud_ptr[cloud];
  int mn0 = INT_MAX, mn1 = INT_MAX, mn2 = INT_MAX, mx0 = INT_MIN, mx1 = INT_MIN, mx2 = INT_MIN, cnt = 0;
  // eight independent 16-byte loads in flight per thread and ~30 points per thread: this pass streams the raw scans (230 MB per
  // 64-pair wave) from HBM, and the reduction tail (shuffles, atomics) is paid once per 30 points instead of once per 7.
  // A CTA walks kVsChunks / gridDim.x CONTIGUOUS chunks of the scan and also reports how many points of each chunk are kept:
  // the pack pass (voxsort.cu) writes the kept points compacted, in scan order, from these counts.
  constexpr int kInFlight = 8;
  __shared__ int s_cc[kVsChunks];
  if (threadIdx.x < kVsChunks) s_cc[threadIdx.x] = 0;
  __syncthreads();
  const int cs = vox_chunk_size(n);
  const int per_cta = kVsChunks / gridDim.x;
  for (int cl = 0; cl < per_cta; ++cl) {
    const int ch = blockIdx.x * per_cta + cl;
    const int c0 = ch * cs, c1 = min(n, c0 + cs);
    int ccnt = 0;
    for (int i0 = c0 + threadIdx.x; i0 < c1; i0 += kInFlight * 256) {
      float4 pp[kInFlight];
#pragma unroll
      for (int j = 0; j < kInFlight; ++j) pp[j] = i0 + j * 256 < c1 ? __ldg(pts + i0 + j * 256) : make_float4(NAN, NAN, NAN, 0.f);  // NaN = not kept
#pragma unroll
      for (int j = 0; j < kInFlight; ++j) {
        const float4 p = pp[j];
        if (i0 + j * 256 >= c1 || !raw_point_kept(p, skip_flagged)) continue;
        const int ox = float_ordered(p.x), oy = float_ordered(p.y), oz = float_ordered(p.z);
        mn0 = min(mn0, ox); mn1 = min(mn1, oy); mn2 = min(mn2, oz);
        mx0 = max(mx0, ox); mx1 = max(mx1, oy); mx2 = max(mx2, oz);
        ++ccnt;
      }
    }
    cnt += ccnt;
    ccnt = __reduce_add_sync(0xffffffffu, ccnt);
    if (lane_id() == 0 && ccnt) atomicAdd(&s_cc[ch], ccnt);
  }
  __syncthreads();
  if ((int)threadIdx.x < per_cta) chunk_cnt[cloud * kVsChunks + blockIdx.x * per_cta + threadIdx.x] = s_cc[blockIdx.x * per_cta + threadIdx.x];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn0 = min(mn0, __shfl_xor_sync(0xffffffffu, mn0, o)); mn1 = min(mn1, __shfl_xor_sync(0xffffffffu, mn1, o));
    mn2 = min(mn2, __shfl_xor_sync(0xffffffffu, mn2, o)); mx0 = max(mx0, __shfl_xor_sync(0xffffffffu, mx0, o));
    mx1 = max(mx1, __shfl_xor_sync(0xffffffffu, mx1, o)); mx2 = max(mx2, __shfl_xor_sync(0xffffffffu, mx2, o));
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  // one set of global atomics per CTA
  __shared__ int s_red[7];
  if (threadIdx.x == 0) { s_red[0] = s_red[1] = s_red[2] = INT_MAX; s_red[3] = s_red[4] = s_red[5] = INT_MIN; s_red[6] = 0; }
  __syncthreads();
  if (lane_id() == 0 && cnt) {
    atomicMin(&s_red[0], mn0); atomicMin(&s_red[1], mn1); atomicMin(&s_red[2], mn2);
    atomicMax(&s_red[3], mx0); atomicMax(&s_red[4], mx1); atomicMax(&s_red[5], mx2);
    atomicAdd(&s_red[6], cnt);
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_red[6]) {
    int* b = bbox + cloud * 6;
    atomicMin(b + 0, s_red[0]); atomicMin(b + 1, s_red[1]); atomicMin(b + 2, s_red[2]);
    atomicMax(b + 3, s_red[3]); atomicMax(b + 4, s_red[4]); atomicMax(b + 5, s_red[5]);
    atomicAdd(n_valid + cloud, s_red[6]);
  }
}

// ------------------------------------------------------------------------------------------------
// K1b / K2b: run heads of the sorted keys of one cloud -> start position of every voxel / cell.
// One CTA per cloud walks its segment with a carried block scan (sizes never leave the device).
//   mode 0 (voxels): segment = [raw_off, raw_off + n_valid) of the voxel sort's A (keys) or B (keys_b) array, by the parity of
//                    the cloud's digit count (voxsort.cu); writes starts[], n_out = #voxels and digits_out = that digit count
//   mode 1 (cells):  segment = [cloud*V, cloud*V + V) of keys, writes starts[] and cell keys (front is not read)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) run_heads_kernel(int mode, const uint64_t* keys, const uint64_t* keys_b, const int* __restrict__ seg_off,
                                                         int V, int key_shift, const CloudFront* __restrict__ front, const int* __restrict__ bbox,
                                                         const int* __restrict__ n_valid_in, int* __restrict__ starts,
                                                         uint64_t* __restrict__ cell_keys, int* __restrict__ n_out, int* __restrict__ n_valid_out,
                                                         int* __restrict__ cloud_status, int* __restrict__ digits_out) {
  __shared__ int sm[33];
  __shared__ int s_overflow, s_valid;  // s_valid: thread 0's running count of valid keys (no register carried across the loop)
  const int cloud = blockIdx.x;
  const int off = mode == 0 ? seg_off[cloud] : cloud * V;
  const int n = mode == 0 ? n_valid_in[cloud] : V;
  const int digits = mode == 0 ? vox_digits(bbox + cloud * 6, n, front[cloud].inv_leaf) : 0;
  if (digits & 1) keys = keys_b;
  // [EXT] pcl::VoxelGrid: dx*dy*dz > INT_MAX -> "leaf size too small", input returned unfiltered; also every other case in which
  // PCL's int index would overflow (vox_grid())
  if (threadIdx.x == 0) {
    s_overflow = digits < 0 ? 1 : 0;
    s_valid = 0;
    if (digits_out) digits_out[cloud] = digits;
  }
  __syncthreads();
  if (s_overflow) {
    if (threadIdx.x == 0) {
      n_out[cloud] = 0;
      cloud_status[cloud] = QB200_ERR_VOXEL_OVERFLOW;
      starts[(size_t)cloud * (V + 1)] = 0;
    }
    return;
  }
  int carry = 0;
  // four consecutive keys per thread and round: a quarter of the block scans (three barriers each) of a key-per-thread loop
  constexpr int kPer = 4;
  for (int base = 0; base < n; base += kPer * blockDim.x) {
    const int p0 = base + kPer * threadIdx.x;
    uint64_t k[kPer];
    bool valid[kPer];
    int head[kPer], nh = 0, nv = 0;
    uint64_t kprev = (p0 > 0 && p0 < n) ? keys[off + p0 - 1] >> key_shift : 0;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int p = p0 + j;
      k[j] = 0; valid[j] = false; head[j] = 0;
      if (p < n) {
        k[j] = keys[off + p] >> key_shift;  // mode 0: the low bits carry the point index
        valid[j] = mode == 0 ? (k[j] & kVoxMask) != kVoxInvalid : (k[j] & kCellMask) != kCellInvalid;
        head[j] = (valid[j] && (p == 0 || k[j] != kprev)) ? 1 : 0;
        kprev = k[j];
      }
      nh += head[j]; nv += valid[j] ? 1 : 0;
    }
    // one scan for both counts: heads in the low half, valid points in the high half (<= 4096 each per round)
    int both;
    const int exb = block_excl_scan(nh | (nv << 16), sm, &both);
    int rank = carry + (exb & 0xFFFF);
    const int tot = both & 0xFFFF, vtot = both >> 16;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      if (head[j]) {
        if (rank <= V) {
          starts[(size_t)cloud * (V + 1) + rank] = p0 + j;
          if (mode == 1 && rank < V) cell_keys[(size_t)cloud * V + rank] = k[j] & kCellMask;
        }
        ++rank;
      }
    }
    carry += tot;
    if (threadIdx.x == 0) s_valid += vtot;
  }
  if (threadIdx.x == 0) {
    const int valid_total = s_valid;
    int nv = carry;
    if (nv > V) {
      nv = V;
      cloud_status[cloud] = QB200_CAPACITY_EXCEEDED;
    } else {
      starts[(size_t)cloud * (V + 1) + nv] = valid_total;  // end sentinel: valid points sort to the front
    }
    n_out[cloud] = nv;
    if (n_valid_out) n_valid_out[cloud] = valid_total;
  }
}

// K1c: centroid of each voxel, summed in original point order (stable sort) -> identical to the
// sequential CPU sum.  One thread per voxel; points are gathered through the sorted index.
__global__ void __launch_bounds__(128) voxel_centroid_kernel(const float4* const* __restrict__ cloud_ptr, const int* __restrict__ raw_off,
                                                             const uint64_t* sorted_keys, const uint64_t* keys_b, const int* __restrict__ vox_digits,
                                                             uint64_t idx_mask,
                                                             const int* __restrict__ starts, const int* __restrict__ n_vox, int V,
                                                             float4* __restrict__ vox_pts) {
  const int cloud = blockIdx.y;
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_vox[cloud]) return;
  // the cloud's sorted segment: B when run_heads_kernel found an odd digit count, else A
  const uint64_t* __restrict__ keys = ((vox_digits[cloud] & 1) ? keys_b : sorted_keys) + raw_off[cloud];
  const float4* __restrict__ pts = cloud_ptr[cloud];
  const int a = starts[(size_t)cloud * (V + 1) + r], b = starts[(size_t)cloud * (V + 1) + r + 1];
  float sx = 0.f, sy = 0.f, sz = 0.f;
  int t = a;
  for (; t + 4 <= b; t += 4) {  // four gathers in flight, summed in order
    const uint64_t k0 = keys[t], k1 = keys[t + 1], k2 = keys[t + 2], k3 = keys[t + 3];
    const float4 p0 = __ldg(pts + (k0 & idx_mask)), p1 = __ldg(pts + (k1 & idx_mask)), p2 = __ldg(pts + (k2 & idx_mask)),
                 p3 = __ldg(pts + (k3 & idx_mask));
    sx += p0.x; sy += p0.y; sz += p0.z;
    sx += p1.x; sy += p1.y; sz += p1.z;
    sx += p2.x; sy += p2.y; sz += p2.z;
    sx += p3.x; sy += p3.y; sz += p3.z;
  }
  for (; t < b; ++t) {
    const float4 p = __ldg(pts + (keys[t] & idx_mask));
    sx += p.x; sy += p.y; sz += p.z;
  }
  const float cnt = (float)(b - a);
  vox_pts[(size_t)cloud * V + r] = make_float4(sx / cnt, sy / cnt, sz / cnt, 1.0f);
}

// K2a: lattice keys of the (voxelised) clouds
__global__ void __launch_bounds__(256) lattice_keys_kernel(const float4* __restrict__ pts, const int* __restrict__ n_pts, int V,
                                                           const CloudFront* __restrict__ front, uint64_t* __restrict__ keys,
                                                           uint32_t* __restrict__ vals) {
  const int cloud = blockIdx.y;
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= V) return;
  uint64_t cell = kCellInvalid;
  if (r < n_pts[cloud]) {
    const float inv_cell = front[cloud].inv_cell;
    const float4 p = pts[(size_t)cloud * V + r];
    if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
      const int ci = (int)floorf(p.x * inv_cell), cj = (int)floorf(p.y * inv_cell), ck = (int)floorf(p.z * inv_cell);
      if (cell_ok(ci, cj, ck)) cell = cell_key(ci, cj, ck);
    }
  }
  keys[(size_t)cloud * V + r] = ((uint64_t)cloud << kCloudShift) | cell;
  vals[(size_t)cloud * V + r] = (uint32_t)r;
}

// ------------------------------------------------------------------------------------------------
// Neighbour walk (device): ascending (cell, index) order; set = {d2 < r2}, self included.
// ------------------------------------------------------------------------------------------------
struct LatticeView {
  const float4* pts;       // cloud's points
  const uint64_t* ckeys;   // occupied cells, ascending
  const int* cstart;       // n_cells + 1
  const uint32_t* order;   // point indices sorted by (cell, index)
  int n_cells;
  float inv;
};

// candidates of the occupied cells [c0, c1): loads are issued four points at a time (index -> point are dependent loads;
// independent candidates overlap their latency), tests and callbacks stay in (cell, index) order
template <class R2, class F>
__device__ __forceinline__ void walk_cells(const LatticeView& L, const float4 pq, const R2& r2_src, int c0, int c1, F&& f) {
  if (c0 >= c1) return;
  const float r2 = r2_src;  // once per cell range (see for_each_neighbor)
  const int t1 = L.cstart[c1];
  for (int t = L.cstart[c0]; t < t1; t += 4) {
    int p[4];
    float4 pp[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) p[e] = t + e < t1 ? (int)L.order[t + e] : -1;
#pragma unroll
    for (int e = 0; e < 4; ++e) pp[e] = p[e] >= 0 ? L.pts[p[e]] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (p[e] < 0) continue;
      const float dx = pq.x - pp[e].x, dy = pq.y - pp[e].y, dz = pq.z - pp[e].z;
      const float d2 = (dx * dx + dy * dy) + dz * dz;
      if (d2 < r2) f(p[e], d2, pp[e]);
    }
  }
}

// kLockstep = false: rows one after the other, in the same order; for callbacks too heavy to be repeated for nine unrolled rows.
// r2: the squared radius, a float or a volatile shared-memory copy that each cell range reads once, so that no register holds it
// across the binary searches.
template <bool kLockstep = true, class R2, class F>
__device__ __forceinline__ void for_each_neighbor(const LatticeView& L, const float4 pq, int m, const R2& r2, F&& f) {
  if (!(isfinite(pq.x) && isfinite(pq.y) && isfinite(pq.z))) return;
  const int ci = (int)floorf(pq.x * L.inv), cj = (int)floorf(pq.y * L.inv), ck = (int)floorf(pq.z * L.inv);
  if (!cell_ok(ci, cj, ck)) return;
  const int ilo = max(ci - m, -kOffIJ), ihi = min(ci + m, kOffIJ - 2);
  if (kLockstep && m == 1) {
    // the usual case (cell >= radius): the 9 (k, j) rows are located by 9 binary searches that advance in lockstep, so
    // their loads are independent (one round trip per step instead of nine), and each row is one contiguous cell range
    uint64_t lo[9], hi[9];
    int a[9], b[9], e[9];
#pragma unroll
    for (int r = 0; r < 9; ++r) {
      const int k = ck + r / 3 - 1, j = cj + r % 3 - 1;
      const bool ok = !(k < -kOffK || k >= kOffK - 1 || j < -kOffIJ || j >= kOffIJ - 1);
      lo[r] = ok ? cell_key(ilo, j, k) : 1;
      hi[r] = ok ? cell_key(ihi, j, k) : 0;
      a[r] = 0; b[r] = ok ? L.n_cells : 0;
      e[r] = 0;
    }
    const int steps = 33 - __clz(L.n_cells | 1);
    for (int s = 0; s < steps; ++s) {
#pragma unroll
      for (int r = 0; r < 9; ++r) {
        if (a[r] < b[r]) {
          const int mid = (a[r] + b[r]) >> 1;
          if (L.ckeys[mid] < lo[r]) a[r] = mid + 1; else b[r] = mid;
        }
      }
    }
    // end of each row's range: at most 3 cells (i - 1, i, i + 1)
#pragma unroll
    for (int r = 0; r < 9; ++r) {
      int c = a[r];
#pragma unroll
      for (int q = 0; q < 3; ++q)
        if (c < L.n_cells && hi[r] >= lo[r] && L.ckeys[c] <= hi[r]) ++c;
      e[r] = c;
    }
#pragma unroll
    for (int r = 0; r < 9; ++r) walk_cells(L, pq, r2, a[r], e[r], f);
    return;
  }
  for (int dk = -m; dk <= m; ++dk) {
    const int k = ck + dk;
    if (k < -kOffK || k >= kOffK - 1) continue;
    for (int dj = -m; dj <= m; ++dj) {
      const int j = cj + dj;
      if (j < -kOffIJ || j >= kOffIJ - 1) continue;
      const uint64_t lo = cell_key(ilo, j, k), hi = cell_key(ihi, j, k);
      int a = 0, b = L.n_cells;
      while (a < b) {
        const int mid = (a + b) >> 1;
        if (L.ckeys[mid] < lo) a = mid + 1; else b = mid;
      }
      int c = a;
      while (c < L.n_cells && L.ckeys[c] <= hi) ++c;
      walk_cells(L, pq, r2, a, c, f);
    }
  }
}

__device__ __forceinline__ LatticeView make_view(int cloud, int V, const float4* pts, const uint64_t* cell_key, const int* cell_start,
                                                 const uint32_t* order, const int* n_cells, float inv) {
  LatticeView L;
  L.pts = pts + (size_t)cloud * V;
  L.ckeys = cell_key + (size_t)cloud * V;
  L.cstart = cell_start + (size_t)cloud * (V + 1);
  L.order = order + (size_t)cloud * V;
  L.n_cells = n_cells[cloud];
  L.inv = inv;
  return L;
}

// K4 / K5 of a point with more than kNbrGlobalCap neighbours (the rare kernels) walk the lattice ONCE, in lattice order.  These
// points are rare in LiDAR scans, but a dense or degenerate cloud can give every point tens of thousands of neighbours, and a walk
// per window of neighbours would then cost O(k^2) per point.  fpfh_rare_kernel accumulates inside the walk.  spfh_kernel<true>
// collects up to kNbrCap neighbour indices at a time in shared memory (walk_chunk: the walk stops when the list is full and
// resumes where it stopped), then computes their pair features in a dense loop with no walk state live across the feature's
// division slow paths.
constexpr int kNbrThreads = 128;
constexpr int kNbrCap = 32;

struct WalkPos {
  int row = 0;   // (k, j) row of the walk, (dk + m) (2m + 1) + (dj + m)
  int t = -1;    // next candidate (position in the sorted index) of that row; -1: the row is not started
};

// the rows of for_each_neighbor<false> from `pos` on, in the same order: writes up to kNbrCap neighbours to nbr[][threadIdx.x],
// returns how many; pos.row == (2m + 1)^2 once the walk is complete
__device__ __forceinline__ int walk_chunk(const LatticeView& L, const float4 pq, int m, float r2, WalkPos& pos,
                                          uint32_t (*nbr)[kNbrThreads]) {
  const int w = 2 * m + 1;
  if (!(isfinite(pq.x) && isfinite(pq.y) && isfinite(pq.z))) { pos.row = w * w; return 0; }
  const int ci = (int)floorf(pq.x * L.inv), cj = (int)floorf(pq.y * L.inv), ck = (int)floorf(pq.z * L.inv);
  if (!cell_ok(ci, cj, ck)) { pos.row = w * w; return 0; }
  const int ilo = max(ci - m, -kOffIJ), ihi = min(ci + m, kOffIJ - 2);
  int n = 0;
  for (; pos.row < w * w; ++pos.row, pos.t = -1) {
    const int k = ck + pos.row / w - m, j = cj + pos.row % w - m;
    if (k < -kOffK || k >= kOffK - 1 || j < -kOffIJ || j >= kOffIJ - 1) continue;
    const uint64_t lo = cell_key(ilo, j, k), hi = cell_key(ihi, j, k);
    int a = 0, b = L.n_cells;
    while (a < b) {
      const int mid = (a + b) >> 1;
      if (L.ckeys[mid] < lo) a = mid + 1; else b = mid;
    }
    int c = a;
    while (c < L.n_cells && L.ckeys[c] <= hi) ++c;
    if (a >= c) continue;
    const int t1 = L.cstart[c];
    for (int t = pos.t >= 0 ? pos.t : L.cstart[a]; t < t1; ++t) {
      const int p = (int)L.order[t];
      const float4 pp = L.pts[p];
      const float dx = pq.x - pp.x, dy = pq.y - pp.y, dz = pq.z - pp.z;
      const float d2 = (dx * dx + dy * dy) + dz * dz;
      if (!(d2 < r2)) continue;
      if (n == kNbrCap) { pos.t = t; return n; }
      nbr[n++][threadIdx.x] = (uint32_t)p;
    }
  }
  return n;
}

// K2c: the fpfh_radius neighbourhood of every point, found ONCE: indices in lattice (cell, index) order, written
// [t][point] so that the stores of a CTA's points coalesce.  K3 (smaller radius: a subsequence of the same order), K4 and K5
// consume the list; a point with more than kNbrGlobalCap neighbours makes its consumers walk the lattice themselves.
__global__ void __launch_bounds__(kNbrThreads) nbr_list_kernel(const float4* __restrict__ pts, const int* __restrict__ n_pts, int V,
                                                               const uint64_t* __restrict__ cell_key, const int* __restrict__ cell_start,
                                                               const uint32_t* __restrict__ order, const int* __restrict__ n_cells,
                                                               const CloudFront* __restrict__ front, uint32_t* __restrict__ nbr_list,
                                                               int* __restrict__ nbr_cnt) {
  volatile __shared__ float s_r2;
  const int cloud = blockIdx.y;
  if (threadIdx.x == 0) s_r2 = front[cloud].rf2;
  __syncthreads();
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_pts[cloud]) return;
  const int m = front[cloud].mf;
  const LatticeView L = make_view(cloud, V, pts, cell_key, cell_start, order, n_cells, front[cloud].inv_cell);
  uint32_t* __restrict__ gl = nbr_list + (size_t)cloud * kNbrGlobalCap * V + q;
  int k = 0;
  for_each_neighbor(L, L.pts[q], m, s_r2, [&](int p, float, const float4) {
    if (k < kNbrGlobalCap) gl[(size_t)k * V] = (uint32_t)p;
    ++k;
  });
  nbr_cnt[(size_t)cloud * V + q] = k;
}

// K3: normals.  One thread per point, sequential float accumulation in lattice order over the points within
// normal_radius: the subsequence of the K2c list that passes the (bit-identical) distance test.
__global__ void __launch_bounds__(128) normals_kernel(const float4* __restrict__ pts, const int* __restrict__ n_pts, int V,
                                                      const uint64_t* __restrict__ cell_key, const int* __restrict__ cell_start,
                                                      const uint32_t* __restrict__ order, const int* __restrict__ n_cells,
                                                      const CloudFront* __restrict__ front, const uint32_t* __restrict__ nbr_list,
                                                      const int* __restrict__ nbr_cnt, float4* __restrict__ normals) {
  volatile __shared__ float s_r2;
  const int cloud = blockIdx.y;
  if (threadIdx.x == 0) s_r2 = front[cloud].rn2;
  __syncthreads();
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_pts[cloud]) return;
  const float4* __restrict__ P = pts + (size_t)cloud * V;
  const float4 pq = P[q];
  float accu[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  int cnt = 0;
  auto add = [&](const float4 pp) {
    accu[0] += pp.x * pp.x; accu[1] += pp.x * pp.y; accu[2] += pp.x * pp.z;
    accu[3] += pp.y * pp.y; accu[4] += pp.y * pp.z; accu[5] += pp.z * pp.z;
    accu[6] += pp.x; accu[7] += pp.y; accu[8] += pp.z;
    ++cnt;
  };
  const int kq = nbr_cnt[(size_t)cloud * V + q];
  if (front[cloud].list_usable && kq <= kNbrGlobalCap) {
    const uint32_t* __restrict__ gl = nbr_list + (size_t)cloud * kNbrGlobalCap * V + q;
    const float r2 = s_r2;
    for (int t = 0; t < kq; ++t) {
      const float4 pp = P[gl[(size_t)t * V]];
      const float dx = pq.x - pp.x, dy = pq.y - pp.y, dz = pq.z - pp.z;
      const float d2 = (dx * dx + dy * dy) + dz * dz;  // same expression as the lattice walk
      if (d2 < r2) add(pp);
    }
  } else {
    const LatticeView L = make_view(cloud, V, pts, cell_key, cell_start, order, n_cells, front[cloud].inv_cell);
    for_each_neighbor(L, pq, front[cloud].mn, s_r2, [&](int, float, const float4 pp) { add(pp); });
  }
  float out[4];
  qb_normal_from_accu(accu, cnt, pq.x, pq.y, pq.z, out);
  normals[(size_t)cloud * V + q] = make_float4(out[0], out[1], out[2], out[3]);
}

// K4: SPFH.  Bin COUNTS are order-free; the float histogram value is rebuilt by repeated addition
// of the same increment, which is what the sequential reference loop produces.
// kRare = false: the points whose neighbourhood is in the K2c list (all but a handful): no lattice walk compiled in, and at most
// kNbrGlobalCap pairs, so 16-bit bin counts.  kRare = true: only the points with more than kNbrGlobalCap neighbours, which walk
// the lattice; a bin can then collect every neighbour of the point (all pairs of a planar neighbourhood share their f2 and f3
// bins), so its counts are 32-bit: 16.5 KB of static shared memory, plus 16 KB of neighbour list (walk_chunk).
// SPFH rows are stored as three padded thirds [11 bins, 0][11 bins, 0][11 bins, 0] (36 floats): a third is three 16-byte loads.
constexpr int kSpfhThreads = kNbrThreads;
static_assert(kNbrGlobalCap < 65536, "spfh_kernel<false> counts in 16 bits");
constexpr int kSpfhRowStride = kDescPad + 1;  // floats per row staged in shared memory: odd, so a warp's row stores hit 32 banks
__device__ __forceinline__ int spfh_slot(int b) { return b + b / 11; }
template <bool kRare>
__global__ void __launch_bounds__(kSpfhThreads) spfh_kernel(const float4* __restrict__ pts, const float4* __restrict__ normals,
                                                            const int* __restrict__ n_pts, int V, const uint64_t* __restrict__ cell_key,
                                                            const int* __restrict__ cell_start, const uint32_t* __restrict__ order,
                                                            const int* __restrict__ n_cells, const CloudFront* __restrict__ front,
                                                            float* __restrict__ spfh, const uint32_t* __restrict__ nbr_list,
                                                            const int* __restrict__ nbr_cnt) {
  using Count = typename std::conditional<kRare, unsigned, unsigned short>::type;
  __shared__ Count cnts[kDescDim][kSpfhThreads];
  __shared__ uint32_t nbr[kRare ? kNbrCap : 1][kNbrThreads];
  __shared__ float staged[kRare ? 1 : kSpfhThreads * kSpfhRowStride];  // kRare = false: the CTA's rows, stored together at the end
  __shared__ bool listed[kRare ? 1 : kSpfhThreads];
  const int cloud = blockIdx.y;
  const int n_cloud = n_pts[cloud];
  const int q0 = blockIdx.x * blockDim.x;
  if (q0 >= n_cloud) return;  // the whole CTA
  const int q = q0 + threadIdx.x;
  int k = q < n_cloud ? nbr_cnt[(size_t)cloud * V + q] : 0;
  const bool mine = q < n_cloud && (k > kNbrGlobalCap) == kRare;
  if (!kRare) listed[threadIdx.x] = mine;
  if (mine) {
    const LatticeView L = make_view(cloud, V, pts, cell_key, cell_start, order, n_cells, front[cloud].inv_cell);
    const float4* __restrict__ nrm = normals + (size_t)cloud * V;
    const float4 pq = L.pts[q];
    const float4 nq = nrm[q];
#pragma unroll
    for (int b = 0; b < kDescDim; ++b) cnts[b][threadIdx.x] = 0;
    auto feature = [&](int p) {
      if (p == q) return;
      const float4 pp = L.pts[p];
      const float4 np = nrm[p];
      float f1, f2, f3;
      if (!qb_pair_features(pq.x, pq.y, pq.z, nq.x, nq.y, nq.z, pp.x, pp.y, pp.z, np.x, np.y, np.z, &f1, &f2, &f3)) return;
      int b1, b2, b3;
      qb_feature_bins(f1, f2, f3, &b1, &b2, &b3);
      cnts[b1][threadIdx.x]++;
      cnts[11 + b2][threadIdx.x]++;
      cnts[22 + b3][threadIdx.x]++;
    };
    if (!kRare) {
      const uint32_t* __restrict__ gl = nbr_list + (size_t)cloud * kNbrGlobalCap * V + q;
      for (int t = 0; t < k; ++t) feature((int)gl[(size_t)t * V]);
    } else {
      k = 0;
      WalkPos pos;
      const int m = front[cloud].mf;
      const float r2 = front[cloud].rf2;
      const int rows = (2 * m + 1) * (2 * m + 1);
      while (pos.row < rows) {
        const int n = walk_chunk(L, pq, m, r2, pos, nbr);
        for (int t = 0; t < n; ++t) feature((int)nbr[t][threadIdx.x]);
        k += n;
      }
    }
    // three padded thirds: 16-byte gathers in K5
    float* __restrict__ out = kRare ? spfh + ((size_t)cloud * V + q) * kDescPad : staged + threadIdx.x * kSpfhRowStride;
    const float incr = k >= 2 ? 100.0f / (float)(k - 1) : 0.0f;
    for (int b = 0; b < kDescDim; ++b) {
      const int c = (int)cnts[b][threadIdx.x];  // at most the neighbour count, which fits an int
      float v = 0.0f;
      for (int t = 0; t < c; ++t) v += incr;
      out[spfh_slot(b)] = v;
    }
    out[11] = 0.0f; out[23] = 0.0f; out[35] = 0.0f;
  }
  if (kRare) return;
  // The CTA's rows are one contiguous run of spfh.  Copied from shared memory by consecutive threads, every warp store writes 128
  // contiguous bytes; stored by their own threads, each of a warp's 36 row stores would write 4 bytes into each of 32 rows.  Rows
  // this launch does not own (points with more than kNbrGlobalCap neighbours, and beyond the cloud) are left alone.
  __syncthreads();
  const int m = min(kSpfhThreads, n_cloud - q0);
  float* __restrict__ dst = spfh + ((size_t)cloud * V + q0) * kDescPad;
  for (int i = threadIdx.x; i < m * kDescPad; i += kSpfhThreads) {
    const int r = i / kDescPad;
    if (listed[r]) dst[i] = staged[r * kSpfhRowStride + (i - r * kDescPad)];
  }
}

// K5: FPFH = per-third renormalised sum of neighbour SPFHs weighted by 1/d^2, neighbours in lattice
// order.  Output is written dimension-major (desc_t[d][q]) for the matching kernel's tile loads.
//
// fpfh_list_kernel (the points whose neighbourhood is in the K2c list): the three thirds of the signature are independent
// (own 11 accumulators, own fp64 normaliser), so a point is served by three threads in three different warps -- 11 accumulators
// and three 16-byte gathers per neighbour each instead of 33 and nine: 3x the warps at well under half the registers.
// Per-bin accumulation order (lattice order of the neighbours) is unchanged.
__global__ void __launch_bounds__(3 * kNbrThreads, 3) fpfh_list_kernel(const float4* __restrict__ pts, const int* __restrict__ n_pts, int V,
                                                                    const float* __restrict__ spfh, const uint32_t* __restrict__ nbr_list,
                                                                    const int* __restrict__ nbr_cnt, float* __restrict__ desc_t) {
  const int cloud = blockIdx.y;
  const int third = threadIdx.x / kNbrThreads;  // warp-uniform
  const int q = blockIdx.x * kNbrThreads + (threadIdx.x - third * kNbrThreads);
  if (q >= n_pts[cloud]) return;
  const int kq = nbr_cnt[(size_t)cloud * V + q];
  if (kq > kNbrGlobalCap) return;  // fpfh_rare_kernel
  const float4* __restrict__ P = pts + (size_t)cloud * V;
  const float4* __restrict__ sp = reinterpret_cast<const float4*>(spfh + (size_t)cloud * V * kDescPad) + 3 * third;
  const float4 pq = P[q];
  float o[11];
#pragma unroll
  for (int b = 0; b < 11; ++b) o[b] = 0.0f;
  double sum = 0.0;
  const uint32_t* __restrict__ gl = nbr_list + (size_t)cloud * kNbrGlobalCap * V + q;
  // Two-deep software pipeline: the index of neighbour t + 2 and the point / SPFH third of neighbour t + 1 are in flight while
  // neighbour t is accumulated (the chain index -> rows -> 11 dependent adds was one full L1/L2 latency per step: 66 % of the
  // scheduler cycles had no eligible warp).  The accumulation order is unchanged.
  int p_n = kq > 0 ? (int)gl[0] : 0;
  int p_nn = kq > 1 ? (int)gl[(size_t)V] : 0;
  float4 pp_n = P[p_n];
  float4 a0 = __ldg(sp + (size_t)p_n * (kDescPad / 4)), a1 = __ldg(sp + (size_t)p_n * (kDescPad / 4) + 1), a2 = __ldg(sp + (size_t)p_n * (kDescPad / 4) + 2);
  for (int t = 0; t < kq; ++t) {
    const float4 pp = pp_n, t0 = a0, t1 = a1, t2 = a2;
    if (t + 1 < kq) {
      const int pn = p_nn;
      if (t + 2 < kq) p_nn = (int)gl[(size_t)(t + 2) * V];
      pp_n = P[pn];
      a0 = __ldg(sp + (size_t)pn * (kDescPad / 4)); a1 = __ldg(sp + (size_t)pn * (kDescPad / 4) + 1); a2 = __ldg(sp + (size_t)pn * (kDescPad / 4) + 2);
    }
    const float dx = pq.x - pp.x, dy = pq.y - pp.y, dz = pq.z - pp.z;
    const float d2 = (dx * dx + dy * dy) + dz * dz;  // the same expression as the neighbour test: bit-identical
    if (d2 == 0.0f) continue;
    const float weight = 1.0f / d2;
    const float sv[11] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w, t2.x, t2.y, t2.z};
#pragma unroll
    for (int b = 0; b < 11; ++b) { const float v = sv[b] * weight; sum += v; o[b] += v; }
  }
  if (sum != 0.0) sum = 100.0 / sum;
  const float g = (float)sum;
  float* __restrict__ out = desc_t + (size_t)cloud * kDescK * V + (size_t)(11 * third) * V + q;
#pragma unroll
  for (int b = 0; b < 11; ++b) out[(size_t)b * V] = o[b] * g;
}

// the rare point with more than kNbrGlobalCap neighbours walks the lattice itself (one thread, all 33 bins, one walk)
__global__ void __launch_bounds__(kNbrThreads) fpfh_rare_kernel(const float4* __restrict__ pts, const int* __restrict__ n_pts, int V,
                                                                const uint64_t* __restrict__ cell_key, const int* __restrict__ cell_start,
                                                                const uint32_t* __restrict__ order, const int* __restrict__ n_cells,
                                                                const CloudFront* __restrict__ front, const float* __restrict__ spfh,
                                                                const int* __restrict__ nbr_cnt, float* __restrict__ desc_t) {
  const int cloud = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_pts[cloud]) return;
  if (nbr_cnt[(size_t)cloud * V + q] <= kNbrGlobalCap) return;  // fpfh_list_kernel
  const int m = front[cloud].mf;
  const float r2 = front[cloud].rf2;
  const LatticeView L = make_view(cloud, V, pts, cell_key, cell_start, order, n_cells, front[cloud].inv_cell);
  const float4* __restrict__ sp = reinterpret_cast<const float4*>(spfh + (size_t)cloud * V * kDescPad);
  const float4 pq = L.pts[q];
  float o[kDescDim];
#pragma unroll
  for (int b = 0; b < kDescDim; ++b) o[b] = 0.0f;
  double s0 = 0.0, s1 = 0.0, s2 = 0.0;
  // the walk's own d2: the expression the list kernel recomputes, bit-identical
  for_each_neighbor<false>(L, pq, m, r2, [&](int p, float d2, const float4) {
    if (d2 == 0.0f) return;
    const float weight = 1.0f / d2;
    float s[kDescPad];
#pragma unroll
    for (int v4 = 0; v4 < kDescPad / 4; ++v4) {
      const float4 t = __ldg(sp + (size_t)p * (kDescPad / 4) + v4);
      s[4 * v4] = t.x; s[4 * v4 + 1] = t.y; s[4 * v4 + 2] = t.z; s[4 * v4 + 3] = t.w;
    }
#pragma unroll
    for (int b = 0; b < 11; ++b) { const float v = s[b] * weight; s0 += v; o[b] += v; }
#pragma unroll
    for (int b = 0; b < 11; ++b) { const float v = s[12 + b] * weight; s1 += v; o[11 + b] += v; }
#pragma unroll
    for (int b = 0; b < 11; ++b) { const float v = s[24 + b] * weight; s2 += v; o[22 + b] += v; }
  });
  if (s0 != 0.0) s0 = 100.0 / s0;
  if (s1 != 0.0) s1 = 100.0 / s1;
  if (s2 != 0.0) s2 = 100.0 / s2;
  const float g0 = (float)s0, g1 = (float)s1, g2 = (float)s2;
  float* __restrict__ out = desc_t + (size_t)cloud * kDescK * V + q;
#pragma unroll
  for (int b = 0; b < 11; ++b) out[(size_t)b * V] = o[b] * g0;
#pragma unroll
  for (int b = 11; b < 22; ++b) out[(size_t)b * V] = o[b] * g1;
#pragma unroll
  for (int b = 22; b < 33; ++b) out[(size_t)b * V] = o[b] * g2;
}

constexpr int kExportTile = 128, kExportThreads = 256;

// Front-end results -> their destinations: cloud c's first m = min(n, cap) voxel points and normals, and its descriptors turned from
// the dimension-major rows of desc_t (or a cache slot) into m rows of 33 floats (pcl::FPFHSignature33).  One launch serves a whole
// describe wave (qb200_describe_batch_each) or the one cloud of qb200_compute_fpfh, qb200_get_last_features and qb200_cache_read.
// One CTA per tile of kExportTile points of a cloud: every dimension's row segment is read coalesced into shared memory (row stride 33
// floats: the transposed stores are free of bank conflicts), and the tile's output rows, one contiguous run of m * 132 bytes, are
// written coalesced from there.  A pure copy: every value arrives bit for bit.
__global__ void __launch_bounds__(kExportThreads) feature_export_kernel(ExportSrc s, int V, ExportDst d) {
  __shared__ float tile[kExportTile * kDescDim];
  const int cloud = blockIdx.y, q0 = blockIdx.x * kExportTile, tid = threadIdx.x;
  const int st = s.status ? s.status[cloud] : QB200_OK;
  // a refused cloud reports 0 and gets nothing; a voxelize wave (n_kept) refuses none: see ExportSrc
  const bool pass = s.n_kept && st == QB200_ERR_VOXEL_OVERFLOW;
  const int n = st == QB200_OK || (s.n_kept && st == QB200_CAPACITY_EXCEEDED) ? s.n[cloud] : pass ? s.n_kept[cloud] : 0;
  if (blockIdx.x == 0 && tid == 0) {
    if (d.counts) d.counts[cloud] = n;
    if (d.status) d.status[cloud] = st;
  }
  const int m_all = pass ? 0 : min(n, d.cap);
  if (q0 >= m_all) return;
  const int m = min(kExportTile, m_all - q0);
  const size_t from = (size_t)cloud * V + q0, to = (size_t)cloud * d.stride + q0;
  for (int i = tid; i < m; i += kExportThreads) {
    if (d.vox) d.vox[to + i] = __ldg(s.vox + from + i);
    if (d.nrm) d.nrm[to + i] = __ldg(s.nrm + from + i);
  }
  if (!d.desc) return;
  const float* __restrict__ col = s.desc + (size_t)cloud * kDescK * V + q0;
  for (int i = tid; i < kDescDim * kExportTile; i += kExportThreads) {
    const int dim = i / kExportTile, q = i % kExportTile;
    if (q < m) tile[q * kDescDim + dim] = __ldg(col + (size_t)dim * V + q);
  }
  __syncthreads();
  float* __restrict__ out = d.desc + to * kDescDim;
  for (int i = tid; i < m * kDescDim; i += kExportThreads) out[i] = tile[i];
}

constexpr int kPassThreads = 1024;

// K1d (voxelize waves): [EXT] pcl::VoxelGrid returns the input unfiltered when its int voxel index would overflow ("leaf size is too
// small"); qb200_voxelize hands back the kept points of such a cloud, in input order.  One CTA per cloud; a cloud that run_heads_kernel
// did not refuse with QB200_ERR_VOXEL_OVERFLOW exits at once.  The CTA walks the cloud one point per thread and round with the keep
// test voxel_bbox_kernel counts into n_valid, and places the kept points by a block scan carried across rounds, as run_heads_kernel
// does.  In place (host scans into their own raw_stage region) every point of a round is read before the scan's barriers and
// written at or before its own position, so no point is overwritten before it is read: the pointers are not __restrict__ and the
// loads do not go through the read-only cache.
__global__ void __launch_bounds__(kPassThreads) passthrough_kernel(const float4* const* __restrict__ cloud_ptr, const int* __restrict__ cloud_n,
                                                                   const CloudFront* __restrict__ front, const int* __restrict__ cloud_status,
                                                                   const int* __restrict__ raw_off, float4* stage, float4* dst,
                                                                   long long stride, int cap) {
  __shared__ int sm[33];
  const int cloud = blockIdx.x;
  if (cloud_status[cloud] != QB200_ERR_VOXEL_OVERFLOW) return;
  const int n = cloud_n[cloud], skip_flagged = front[cloud].skip_flagged;
  const float4* src = cloud_ptr[cloud];
  float4* out = dst ? dst + cloud * stride : stage + raw_off[cloud];
  const int lim = dst ? cap : n;
  int carry = 0;  // the same in every thread: the loop condition is uniform
  for (int base = 0; base < n && carry < lim; base += blockDim.x) {
    const int i = base + threadIdx.x;
    float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
    bool keep = false;
    if (i < n) {
      p = src[i];
      keep = raw_point_kept(p, skip_flagged);
    }
    int tot;
    const int pos = carry + block_excl_scan(keep ? 1 : 0, sm, &tot);
    if (keep && pos < lim) out[pos] = p;
    carry += tot;
  }
}

constexpr int kImportTile = 128, kImportThreads = 256;

// Caller features of a wave -> the matcher's inputs: cloud c's keypoints into vox_pts, the first `dim` floats of its n descriptor
// rows (`stride` floats apart: pcl::FPFHSignature33 is 33 of 33, pcl::SHOT352 352 of 361) into `dim` dimension-major rows at
// f.out, ld apart (desc_t for FPFH-33, dd_buf for other lengths), and n into n_vox and, for FPFH-33, n_fpfh.  One CTA per tile of
// kImportTile points of a cloud, 33 dimensions at a time: the tile's rows are read as runs of up to 33 floats into shared memory,
// and every dimension-major row segment is written coalesced from there (row pitch 33 floats: the column reads are free of bank
// conflicts).  A pure copy: every value, NaN payloads included, arrives bit for bit.  A cloud without descriptors (a keypoint wave
// of qb200_describe_points_each, which K2..K5 describe next) imports its keypoints and count only.
__global__ void __launch_bounds__(kImportThreads) feature_import_kernel(const FeatureSrc* __restrict__ table, int V, float4* __restrict__ vox_pts,
                                                                        int* __restrict__ n_vox, int* __restrict__ n_fpfh) {
  __shared__ float tile[kImportTile * kDescDim];
  const int cloud = blockIdx.y, q0 = blockIdx.x * kImportTile, tid = threadIdx.x;
  const FeatureSrc f = table[cloud];
  if (blockIdx.x == 0 && tid == 0) {
    n_vox[cloud] = f.n;
    n_fpfh[cloud] = f.dim == kDescDim ? f.n : 0;
  }
  if (q0 >= f.n) return;
  const int m = min(kImportTile, f.n - q0);
  if (f.pts)  // (qb200_debug_tc_distances imports descriptors only)
    for (int i = tid; i < m; i += kImportThreads) vox_pts[(size_t)cloud * V + q0 + i] = __ldg(f.pts + q0 + i);
  if (!f.desc) return;  // the same for every thread of the CTA: no thread waits at the barriers below
  const float* __restrict__ src = f.desc + (size_t)q0 * f.stride;
  for (int k0 = 0; k0 < f.dim; k0 += kDescDim) {
    const int kw = min(kDescDim, f.dim - k0);
    if (k0 > 0) __syncthreads();  // the previous chunk's column reads are done
    for (int i = tid; i < m * kDescDim; i += kImportThreads) {
      const int q = i / kDescDim, d = i % kDescDim;
      if (d < kw) tile[i] = __ldg(src + (size_t)q * f.stride + k0 + d);
    }
    __syncthreads();
    float* __restrict__ out = f.out + (size_t)k0 * f.ld + q0;
    for (int i = tid; i < kw * kImportTile; i += kImportThreads) {
      const int d = i / kImportTile, q = i % kImportTile;
      if (q < m) out[(size_t)d * f.ld + q] = tile[q * kDescDim + d];
    }
  }
}

// ------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------
void front_voxel(CloudFront* e, float leaf, int skip_flagged) {
  e->inv_leaf = 1.0f / leaf;
  e->skip_flagged = skip_flagged;
}

void front_lattice(CloudFront* e, float normal_radius, float fpfh_radius, float cell) {
  e->inv_cell = 1.0f / cell;
  e->mn = (int)ceilf(normal_radius * e->inv_cell + 1e-3f);
  e->mf = (int)ceilf(fpfh_radius * e->inv_cell + 1e-3f);
  e->rn2 = (float)((double)normal_radius * (double)normal_radius);
  e->rf2 = (float)((double)fpfh_radius * (double)fpfh_radius);
  // the list serves K3 when the normal neighbourhood is a subset visited in the same order: radius <= fpfh radius (checked
  // by the callers) and the same lattice reach for both walks
  e->list_usable = (e->mn <= e->mf && e->rn2 <= e->rf2) ? 1 : 0;
}

int upload_front(Lane* L, int n) {
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->d_front, L->h_front, (size_t)n * sizeof(CloudFront), cudaMemcpyHostToDevice, L->stream));
  return QB200_OK;
}

int launch_voxel(Lane* h, int n_clouds) {
  if (n_clouds <= 0) return QB200_OK;
  const dim3 gb(n_clouds >= 16 ? 16 : 64, n_clouds);  // ~30 points per thread when the batch fills the device on its own
  int* chunk_cnt = reinterpret_cast<int*>(h->val_b.get());   // [clouds][kVsChunks]
  voxel_bbox_kernel<<<gb, 256, 0, h->stream>>>(h->d_cloud_ptr, h->d_cloud_n, h->d_front, h->ctr.bbox, h->ctr.n_valid, chunk_cnt);
  h->launches += 1;
  const int idx_bits = clog2(h->R > 2 ? h->R : 2);  // point index inside its scan
  if (int rc = launch_voxel_sort(h, n_clouds, idx_bits)) return rc;
  run_heads_kernel<<<n_clouds, 1024, 0, h->stream>>>(0, h->key_a, h->key_b, h->d_raw_off, h->V, idx_bits, h->d_front, h->ctr.bbox, h->ctr.n_valid,
                                                     h->vox_start, nullptr, h->ctr.n_vox, nullptr, h->ctr.cloud_status, h->ctr.vox_digits);
  const dim3 gc((h->V + 127) / 128, n_clouds);
  voxel_centroid_kernel<<<gc, 128, 0, h->stream>>>(h->d_cloud_ptr, h->d_raw_off, h->key_a, h->key_b, h->ctr.vox_digits,
                                                   (1ull << idx_bits) - 1, h->vox_start, h->ctr.n_vox, h->V, h->vox_pts);
  h->launches += 2;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

int launch_fpfh(Lane* h, int n_clouds) {
  if (n_clouds <= 0) return QB200_OK;
  const int V = h->V;
  const dim3 gl((V + 255) / 256, n_clouds);
  lattice_keys_kernel<<<gl, 256, 0, h->stream>>>(h->vox_pts, h->ctr.n_vox, V, h->d_front, h->key_a, h->val_a);
  h->launches++;
  // per-cloud shared-memory sort (sort.cu); clouds too large for it go through the device-wide radix sort
  int rc = launch_cloud_sort(h, n_clouds, h->ctr.n_vox, 18, 36);  // fields of cell_key(): i | j | k
  if (rc == QB200_ERR_UNSUPPORTED) rc = sort_pairs(h, n_clouds * V, kCloudShift + clog2(n_clouds > 1 ? n_clouds : 2));
  if (rc) return rc;
  run_heads_kernel<<<n_clouds, 1024, 0, h->stream>>>(1, h->key_b, nullptr, nullptr, V, 0, nullptr, nullptr, nullptr, h->cell_start, h->cell_key,
                                                     h->ctr.n_cells, h->ctr.n_lat, h->ctr.cloud_status, nullptr);
  const dim3 gp((V + 127) / 128, n_clouds);
  nbr_list_kernel<<<gp, kNbrThreads, 0, h->stream>>>(h->vox_pts, h->ctr.n_vox, V, h->cell_key, h->cell_start, h->val_b, h->ctr.n_cells,
                                                     h->d_front, h->nbr_list, h->nbr_cnt);
  normals_kernel<<<gp, 128, 0, h->stream>>>(h->vox_pts, h->ctr.n_vox, V, h->cell_key, h->cell_start, h->val_b, h->ctr.n_cells, h->d_front,
                                            h->nbr_list, h->nbr_cnt, h->normals);
  // listed neighbourhoods (all but a handful of points) and the lattice-walking rest are separate launches: the common kernels
  // carry neither the walk's registers nor its list buffer
  spfh_kernel<false><<<gp, kSpfhThreads, 0, h->stream>>>(h->vox_pts, h->normals, h->ctr.n_vox, V, h->cell_key, h->cell_start, h->val_b,
                                                         h->ctr.n_cells, h->d_front, h->spfh, h->nbr_list, h->nbr_cnt);
  spfh_kernel<true><<<gp, kSpfhThreads, 0, h->stream>>>(h->vox_pts, h->normals, h->ctr.n_vox, V, h->cell_key, h->cell_start, h->val_b,
                                                        h->ctr.n_cells, h->d_front, h->spfh, h->nbr_list, h->nbr_cnt);
  fpfh_list_kernel<<<gp, 3 * kNbrThreads, 0, h->stream>>>(h->vox_pts, h->ctr.n_vox, V, h->spfh, h->nbr_list, h->nbr_cnt, h->desc_t);
  fpfh_rare_kernel<<<gp, kNbrThreads, 0, h->stream>>>(h->vox_pts, h->ctr.n_vox, V, h->cell_key, h->cell_start, h->val_b, h->ctr.n_cells,
                                                      h->d_front, h->spfh, h->nbr_cnt, h->desc_t);
  h->launches += 3;
  h->launches += 4;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

int launch_feature_export(Lane* h, int n_clouds, const ExportSrc& src, const ExportDst& dst, int max_n) {
  if (n_clouds <= 0) return QB200_OK;
  const int m = max_n < dst.cap ? max_n : dst.cap;
  const dim3 g(((m > 1 ? m : 1) + kExportTile - 1) / kExportTile, n_clouds);  // at least one tile: its first CTA reports the cloud
  feature_export_kernel<<<g, kExportThreads, 0, h->stream>>>(src, h->V, dst);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

int launch_passthrough(Lane* h, int n_clouds, float4* dst, long long stride, int cap) {
  if (n_clouds <= 0) return QB200_OK;
  passthrough_kernel<<<n_clouds, kPassThreads, 0, h->stream>>>(h->d_cloud_ptr, h->d_cloud_n, h->d_front, h->ctr.cloud_status, h->d_raw_off,
                                                               h->raw_stage, dst, stride, cap);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

int export_desc_rows(Lane* h, const float* desc, const int* n, int m) {
  ExportSrc s{nullptr, nullptr, desc, n, nullptr, nullptr};
  ExportDst d{nullptr, nullptr, h->aos_scratch, m, m, nullptr, nullptr};
  return launch_feature_export(h, 1, s, d, m);
}

ExportDst ExportDst::caller(const qb200_feature_out& o, long long first) {
  const long long c = o.cap_per_scan;
  ExportDst d;
  d.vox = o.vox4 ? reinterpret_cast<float4*>(o.vox4) + first * c : nullptr;
  d.nrm = o.normals4 ? reinterpret_cast<float4*>(o.normals4) + first * c : nullptr;
  d.desc = o.desc33 ? o.desc33 + first * c * kDescDim : nullptr;
  d.stride = c;
  d.cap = o.cap_per_scan;
  d.counts = d.status = nullptr;
  return d;
}

size_t ExportDst::carve(unsigned char* base, int n, int cap, const qb200_feature_out& o, ExportDst* d) {
  const size_t k = (size_t)n * cap;
  size_t off = 0;
  auto take = [&](size_t bytes, bool want) -> unsigned char* {
    if (!want) return nullptr;
    unsigned char* p = base ? base + off : nullptr;
    off += (bytes + 15) & ~(size_t)15;
    return p;
  };
  d->counts = reinterpret_cast<int*>(take((size_t)n * sizeof(int), true));
  d->status = reinterpret_cast<int*>(take((size_t)n * sizeof(int), true));
  d->vox = reinterpret_cast<float4*>(take(k * sizeof(float4), o.vox4));
  d->nrm = reinterpret_cast<float4*>(take(k * sizeof(float4), o.normals4));
  d->desc = reinterpret_cast<float*>(take(k * kDescDim * sizeof(float), o.desc33));
  d->stride = cap;
  d->cap = cap;
  return off;
}
int launch_feature_import(Lane* h, int n_clouds) {
  if (n_clouds <= 0) return QB200_OK;
  int n_max = 1;  // at least one tile per cloud: its first CTA writes n_vox, also for an empty cloud
  for (int c = 0; c < n_clouds; ++c) n_max = h->h_feat[c].n > n_max ? h->h_feat[c].n : n_max;
  const dim3 g((n_max + kImportTile - 1) / kImportTile, n_clouds);
  feature_import_kernel<<<g, kImportThreads, 0, h->stream>>>(h->d_feat, h->V, h->vox_pts, h->ctr.n_vox, h->ctr.n_fpfh);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

}  // namespace qb
