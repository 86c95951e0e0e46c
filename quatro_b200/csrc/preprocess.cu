// preprocess.cu -- ground removal BEFORE the registration path (SURVEY.md 8f-1), sm_90a.
//
// Replaces PatchWork<PointT>::estimate_ground (include/patchwork.hpp:329-455): concentric-zone binning (pc2czm, :512-543),
// per-patch z order (the global z sort of :348 only matters inside a patch), region-wise ground plane fitting
// (extract_initial_seeds_ :278-322, estimate_plane_ :264-276, extract_piecewiseground :548-590) and the ground likelihood
// estimation (:386-440).  The reference walks ~500 patches one after the other on one core; here every patch is one CTA:
//
//   pw_bin_kernel      point -> patch id (double radius / azimuth like the reference), per-patch counts
//   pw_scan_kernel     exclusive scan of the counts (one CTA)
//   pw_scatter_kernel  (ordered z bits | point index) keys into the patch's segment (arrival order, fixed by the sort below)
//   pw_patch_kernel    one CTA per patch: bitonic sort of the keys in shared memory (ascending z, ties by index), seeds from the
//                      lowest points, num_iter x { mean / covariance of the current ground set by a FIXED reduction tree (256
//                      interleaved partial sums, xor butterfly per warp, warps left to right), closed-form 3x3 eigen solve,
//                      signed-distance test }, likelihood tests, ranks of the ground / non-ground points inside the patch
//   pw_offsets_kernel  exclusive scans of the patches' output counts (one CTA)
//   pw_gather_kernel   points into the two outputs in the reference's order (patches zone -> ring -> sector, ascending z inside)
//
// Arithmetic: float sums and products in the order DESIGN.md 5.5 states (the library is built with -fmad=false, nothing is
// contracted), thresholds in double exactly where the reference compares a float with a double.
#include "fpfh_math.cuh"
#include "handle.cuh"

namespace qb {

constexpr int kPwThreads = 256;
constexpr int kPwMaxPatchPts = 16384;   // keys of one patch in shared memory (128 KB)
constexpr int kPwMaxPatches = 4096;

struct PwDev {   // device copy of the parameters + derived table
  qb200_patchwork_params p;
  int patch_base[QB200_PW_MAX_ZONES + 1];
  int n_patches;
};

__host__ __device__ inline bool pw_params_valid(const qb200_patchwork_params& pp) {  // check_input_parameters_are_correct, :592-616
  if (pp.num_zones != 4 || pp.num_thresholds < 0 || pp.num_thresholds > QB200_PW_MAX_THRESHOLDS) return false;
  if (pp.min_range != pp.min_ranges_each_zone[0]) return false;
  if (pp.num_iter < 1 || pp.num_lpr < 0 || pp.num_min_pts < 0 || !(pp.max_range > pp.min_ranges_each_zone[3])) return false;
  int tot = 0;
  for (int k = 0; k < 4; ++k) {
    if (pp.num_sectors_each_zone[k] < 1 || pp.num_rings_each_zone[k] < 1) return false;
    if (k > 0 && !(pp.min_ranges_each_zone[k] > pp.min_ranges_each_zone[k - 1])) return false;
    tot += pp.num_sectors_each_zone[k] * pp.num_rings_each_zone[k];
  }
  return tot <= kPwMaxPatches;
}

// pc2czm, patchwork.hpp:512-543 (xy2radius :505-508, xy2theta :491-502): patch index in traversal order, or -1
__device__ __forceinline__ int pw_patch_of(const float4 pt, const PwDev& c) {
  const qb200_patchwork_params& pp = c.p;
  const double x = (double)pt.x, y = (double)pt.y;
  const double r = sqrt(x * x + y * y);
  if (!(r <= pp.max_range && r > pp.min_range)) return -1;
  const double at = atan2(y, x);
  const double theta = at > 0 ? at : at + 2 * 3.14159265358979323846;
  int k = 3;
  if (r < pp.min_ranges_each_zone[1]) k = 0;
  else if (r < pp.min_ranges_each_zone[2]) k = 1;
  else if (r < pp.min_ranges_each_zone[3]) k = 2;
  const double zmin = pp.min_ranges_each_zone[k];
  const double zmax = k < 3 ? pp.min_ranges_each_zone[k + 1] : pp.max_range;
  const double ring_size = (zmax - zmin) / pp.num_rings_each_zone[k];
  const double sector_size = 2 * 3.14159265358979323846 / pp.num_sectors_each_zone[k];
  const int ring = min((int)((r - zmin) / ring_size), pp.num_rings_each_zone[k] - 1);
  const int sector = min((int)(theta / sector_size), pp.num_sectors_each_zone[k] - 1);
  return c.patch_base[k] + ring * pp.num_sectors_each_zone[k] + sector;
}

__global__ void __launch_bounds__(256) pw_bin_kernel(const float4* __restrict__ pts, int n, PwDev c, int* __restrict__ patch_of,
                                                     int* __restrict__ count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = pts[i];
  int pid = -1;
  // non-finite points never enter (D11); :356-368 drops everything below -1.8 sensor_height
  if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && !((double)p.z < -1.8 * c.p.sensor_height)) pid = pw_patch_of(p, c);
  patch_of[i] = pid;
  if (pid >= 0) atomicAdd(&count[pid], 1);
}

// start[] = exclusive scan of count[0..np), start[np] = total; cursor = copy of start
__global__ void __launch_bounds__(1024) pw_scan_kernel(const int* __restrict__ count, int np, int* __restrict__ start, int* __restrict__ cursor) {
  __shared__ int sm[33];
  int carry = 0;
  for (int base = 0; base < np; base += 1024) {
    const int q = base + threadIdx.x;
    const int v = q < np ? count[q] : 0;
    int tot;
    const int ex = block_excl_scan(v, sm, &tot);
    if (q < np) { start[q] = carry + ex; cursor[q] = carry + ex; }
    carry += tot;
  }
  if (threadIdx.x == 0) start[np] = carry;
}

__global__ void __launch_bounds__(256) pw_scatter_kernel(const float4* __restrict__ pts, int n, const int* __restrict__ patch_of,
                                                         int* __restrict__ cursor, unsigned long long* __restrict__ items) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int pid = patch_of[i];
  if (pid < 0) return;
  const float z = pts[i].z + 0.0f;  // -0 -> +0: the comparator z_a < z_b does not tell them apart
  unsigned zb = __float_as_uint(z);
  zb = (zb & 0x80000000u) ? ~zb : (zb | 0x80000000u);  // order-preserving
  const int pos = atomicAdd(&cursor[pid], 1);
  items[pos] = ((unsigned long long)zb << 32) | (unsigned)i;
}

__device__ __forceinline__ void pw_plane_from_accu(float accu[9], int cnt, float n[3], float mean[3], float* surf) {
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
  qb_eigen33_smallest(cov, &ev, e);   // [EXT] Eigen::JacobiSVD in the reference (:267-271): closed form, oriented n_z >= 0
  if (e[2] < 0.0f) { e[0] = -e[0]; e[1] = -e[1]; e[2] = -e[2]; }
  const float tr = cov[0] + cov[4] + cov[8];
  *surf = (tr != 0.0f) ? fabsf(ev / tr) : 0.0f;
  n[0] = e[0]; n[1] = e[1]; n[2] = e[2];
  mean[0] = accu[6]; mean[1] = accu[7]; mean[2] = accu[8];
}

// One CTA per patch.  keys: sorted (z | index); flag[p] = sorted position p belongs to the current ground set.
__global__ void __launch_bounds__(kPwThreads) pw_patch_kernel(const float4* __restrict__ pts, PwDev c, const int* __restrict__ start,
                                                              unsigned long long* __restrict__ items, int cap_pow2,
                                                              int* __restrict__ n_ground, int* __restrict__ n_nonground,
                                                              int* __restrict__ rank_out, int* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char pw_smem[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(pw_smem);   // [cap_pow2]
  unsigned char* flag = reinterpret_cast<unsigned char*>(keys + cap_pow2);     // [cap_pow2]
  __shared__ float s_part[kPwThreads / 32][9];
  __shared__ int s_cnt[kPwThreads / 32];
  __shared__ float s_plane[8];   // n[3], mean[3], surf, th_dist_d
  __shared__ double s_lpr;
  __shared__ int s_init, s_keep, s_scan[33];
  const qb200_patchwork_params& pp = c.p;
  const int pid = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int s0 = start[pid], m = start[pid + 1] - s0;
  if (!(m > pp.num_min_pts) || m > kPwMaxPatchPts) {   // :382 -- small patches are dropped altogether
    if (tid == 0) {
      n_ground[pid] = 0; n_nonground[pid] = 0;
      if (m > kPwMaxPatchPts) *status = QB200_CAPACITY_EXCEEDED;
    }
    return;
  }
  int zone = 0;
  while (zone < 3 && pid >= c.patch_base[zone + 1]) ++zone;
  const int ring = (pid - c.patch_base[zone]) / pp.num_sectors_each_zone[zone];
  int concentric_idx = ring;
  for (int k = 0; k < zone; ++k) concentric_idx += pp.num_rings_each_zone[k];

  // ---- ascending (z, index): bitonic sort over the next power of two (padding = all ones)
  int N = 1;
  while (N < m) N <<= 1;
  for (int p = tid; p < N; p += kPwThreads) keys[p] = p < m ? items[s0 + p] : ~0ull;
  if (tid == 0) s_init = 0;
  __syncthreads();
  for (int k = 2; k <= N; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < N; i += kPwThreads) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = keys[i], b = keys[ixj];
          const bool asc = (i & k) == 0;
          if ((a > b) == asc) { keys[i] = b; keys[ixj] = a; }
        }
      }
      __syncthreads();
    }
  }
  // ---- extract_initial_seeds_, :278-322
  const double low_margin = pp.sensor_height == 0.0 ? -0.1 : pp.adaptive_seed_selection_margin * pp.sensor_height;
  if (zone == 0) {  // leading points below the margin (the positions are sorted by z: a count is the prefix length)
    int below = 0;
    for (int p = tid; p < m; p += kPwThreads) below += ((double)pts[(unsigned)keys[p]].z < low_margin) ? 1 : 0;
    below = __reduce_add_sync(0xffffffffu, below);
    if (lane == 0 && below) atomicAdd(&s_init, below);
  }
  __syncthreads();
  if (tid == 0) {
    double sum = 0;
    int cnt = 0;
    for (int i = s_init; i < m && cnt < pp.num_lpr; ++i) { sum += (double)pts[(unsigned)keys[i]].z; ++cnt; }
    s_lpr = cnt != 0 ? sum / cnt : 0;
    s_plane[0] = 0.f; s_plane[1] = 0.f; s_plane[2] = 1.f; s_plane[3] = 0.f; s_plane[4] = 0.f; s_plane[5] = 0.f; s_plane[6] = 0.f;
  }
  __syncthreads();
  {
    const double thr = s_lpr + pp.th_seeds;
    for (int p = tid; p < m; p += kPwThreads) flag[p] = ((double)pts[(unsigned)keys[p]].z < thr) ? 1 : 0;
  }
  __syncthreads();
  // ---- extract_piecewiseground, :548-590
  for (int it = 0; it < pp.num_iter; ++it) {
    float a[9];
#pragma unroll
    for (int e = 0; e < 9; ++e) a[e] = 0.0f;
    int gc = 0;
    for (int p = tid; p < m; p += kPwThreads) {
      if (!flag[p]) continue;
      const float4 q = pts[(unsigned)keys[p]];
      a[0] += q.x * q.x; a[1] += q.x * q.y; a[2] += q.x * q.z;
      a[3] += q.y * q.y; a[4] += q.y * q.z; a[5] += q.z * q.z;
      a[6] += q.x; a[7] += q.y; a[8] += q.z;
      ++gc;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int e = 0; e < 9; ++e) a[e] = a[e] + __shfl_xor_sync(0xffffffffu, a[e], o);
    }
    gc = __reduce_add_sync(0xffffffffu, gc);
    if (lane == 0) {
#pragma unroll
      for (int e = 0; e < 9; ++e) s_part[warp][e] = a[e];
      s_cnt[warp] = gc;
    }
    __syncthreads();
    if (tid == 0) {
      float accu[9];
      int tot = 0;
      for (int e = 0; e < 9; ++e) {
        float t = s_part[0][e];
        for (int g = 1; g < kPwThreads / 32; ++g) t = t + s_part[g][e];
        accu[e] = t;
      }
      for (int g = 0; g < kPwThreads / 32; ++g) tot += s_cnt[g];
      float nrm[3] = {s_plane[0], s_plane[1], s_plane[2]}, mean[3] = {s_plane[3], s_plane[4], s_plane[5]}, surf = s_plane[6];
      if (tot > 0) pw_plane_from_accu(accu, tot, nrm, mean, &surf);   // estimate_plane_, :264-276
      const float d = -((nrm[0] * mean[0] + nrm[1] * mean[1]) + nrm[2] * mean[2]);
      s_plane[0] = nrm[0]; s_plane[1] = nrm[1]; s_plane[2] = nrm[2];
      s_plane[3] = mean[0]; s_plane[4] = mean[1]; s_plane[5] = mean[2];
      s_plane[6] = surf;
      s_plane[7] = (float)(pp.th_dist - (double)d);
    }
    __syncthreads();
    const float n0 = s_plane[0], n1 = s_plane[1], n2 = s_plane[2], thd = s_plane[7];
    for (int p = tid; p < m; p += kPwThreads) {
      const float4 q = pts[(unsigned)keys[p]];
      const float res = (q.x * n0 + q.y * n1) + q.z * n2;
      flag[p] = res < thd ? 1 : 0;
    }
    __syncthreads();
  }
  // ---- ground likelihood estimation, :386-440
  if (tid == 0) {
    const double ground_z_vec = fabs((double)s_plane[2]);
    const double ground_z_elevation = (double)s_plane[5];
    const double surface_variable = (double)s_plane[6];
    int keep;
    if (ground_z_vec < pp.uprightness_thr) keep = 0;
    else if (concentric_idx < pp.num_thresholds) {
      const int ti = ring + 2 * zone;
      const double et = ti < pp.num_thresholds ? pp.elevation_thresholds[ti] : pp.elevation_thresholds[pp.num_thresholds - 1];
      const double ft = ti < pp.num_thresholds ? pp.flatness_thresholds[ti] : pp.flatness_thresholds[pp.num_thresholds - 1];
      if (ground_z_elevation > et) keep = ft > surface_variable ? 1 : 0;
      else keep = 1;
    } else {
      keep = !(pp.using_global_elevation && ground_z_elevation > pp.global_elevation_threshold) ? 1 : 0;
    }
    s_keep = keep;
  }
  __syncthreads();
  // ---- ranks inside the patch: rank_out[s0 + p] = (point index, output, position in the patch's part of that output)
  //      encoded as  rank | (1 << 30 if the point goes to the GROUND output); the gather pass reads the point index from items
  const int keep = s_keep;
  int carry_f = 0, carry_u = 0;
  int nf_total = 0;
  for (int p = tid; p < m; p += kPwThreads) nf_total += flag[p];
  nf_total = __reduce_add_sync(0xffffffffu, nf_total);
  if (lane == 0) s_cnt[warp] = nf_total;
  __syncthreads();
  nf_total = 0;
  for (int g = 0; g < kPwThreads / 32; ++g) nf_total += s_cnt[g];
  for (int base = 0; base < m; base += kPwThreads) {
    const int p = base + tid;
    const int f = (p < m && flag[p]) ? 1 : 0, u = (p < m && !flag[p]) ? 1 : 0;
    int both;
    const int ex = block_excl_scan(f | (u << 16), s_scan, &both);
    if (p < m) {
      int code;
      if (f) code = keep ? ((carry_f + (ex & 0xFFFF)) | (1 << 30)) : (carry_f + (ex & 0xFFFF));
      else code = keep ? (carry_u + (ex >> 16)) : (nf_total + carry_u + (ex >> 16));   // a rejected patch: ground part first
      rank_out[s0 + p] = code;
      // the sorted key goes back so that the gather pass finds the point of sorted position p
      items[s0 + p] = keys[p];
    }
    carry_f += both & 0xFFFF;
    carry_u += both >> 16;
  }
  if (tid == 0) {
    n_ground[pid] = keep ? nf_total : 0;
    n_nonground[pid] = keep ? m - nf_total : m;
  }
}

// exclusive scans of the per-patch output counts; totals -> out_n[0] (ground), out_n[1] (non-ground)
__global__ void __launch_bounds__(1024) pw_offsets_kernel(const int* __restrict__ n_ground, const int* __restrict__ n_nonground, int np,
                                                          int* __restrict__ goff, int* __restrict__ ngoff, int* __restrict__ out_n) {
  __shared__ int sm[33];
  int cg = 0, cn = 0;
  for (int base = 0; base < np; base += 1024) {
    const int q = base + threadIdx.x;
    int tot;
    int ex = block_excl_scan(q < np ? n_ground[q] : 0, sm, &tot);
    if (q < np) goff[q] = cg + ex;
    cg += tot;
    ex = block_excl_scan(q < np ? n_nonground[q] : 0, sm, &tot);
    if (q < np) ngoff[q] = cn + ex;
    cn += tot;
  }
  if (threadIdx.x == 0) { out_n[0] = cg; out_n[1] = cn; }
}

__global__ void __launch_bounds__(256) pw_gather_kernel(const float4* __restrict__ pts, const int* __restrict__ start, const int* __restrict__ n_ground,
                                                        const int* __restrict__ n_nonground, const unsigned long long* __restrict__ items,
                                                        const int* __restrict__ rank, const int* __restrict__ goff, const int* __restrict__ ngoff,
                                                        float4* __restrict__ ground, float4* __restrict__ nonground) {
  const int pid = blockIdx.x;
  if (n_ground[pid] + n_nonground[pid] == 0) return;
  const int s0 = start[pid], m = start[pid + 1] - s0;
  for (int p = threadIdx.x; p < m; p += blockDim.x) {
    const int code = rank[s0 + p];
    const float4 q = pts[(unsigned)items[s0 + p]];
    if (code & (1 << 30)) ground[goff[pid] + (code & ~(1 << 30))] = q;
    else nonground[ngoff[pid] + code] = q;
  }
}

// allocated on the first call of a lane: both buffers or neither
static int ensure_pw_scratch(Lane* h) {
  if (h->pw_ints) return QB200_OK;
  const size_t R = h->R;
  DeviceMem<int> ints;
  DeviceMem<float4> out;
  // ints: patch_of [R] | rank [R] | count, start(+1), cursor, n_ground, n_nonground, goff, ngoff [each 4096+1] | out_n [2] | status [1]
  QB_CUDA_TRY(h, ints.alloc(2 * R + 7 * (kPwMaxPatches + 1) + 4));
  QB_CUDA_TRY(h, out.alloc(2 * R));
  h->pw_ints = std::move(ints);
  h->pw_out = std::move(out);
  return QB200_OK;
}

// pts: n points on the device.  Leaves the two outputs in h->pw_out ([0, R) ground, [R, 2R) non-ground) and returns their sizes.
int launch_patchwork(Lane* h, const float4* pts, int n, const qb200_patchwork_params& pp, int* n_ground, int* n_nonground, int* status) {
  *n_ground = *n_nonground = 0;
  *status = QB200_OK;
  if (!pw_params_valid(pp)) return QB200_ERR_BAD_ARG;
  if (n <= 0) return QB200_OK;
  if (int rc = ensure_pw_scratch(h)) return rc;
  PwDev c;
  c.p = pp;
  c.patch_base[0] = 0;
  for (int k = 0; k < 4; ++k) c.patch_base[k + 1] = c.patch_base[k] + pp.num_sectors_each_zone[k] * pp.num_rings_each_zone[k];
  c.n_patches = c.patch_base[4];
  const int NP = c.n_patches;
  const size_t R = h->R;
  int* patch_of = h->pw_ints;
  int* rank = patch_of + R;
  int* count = rank + R;
  int* start = count + (kPwMaxPatches + 1);
  int* cursor = start + (kPwMaxPatches + 1);
  int* ng_ground = cursor + (kPwMaxPatches + 1);
  int* ng_non = ng_ground + (kPwMaxPatches + 1);
  int* goff = ng_non + (kPwMaxPatches + 1);
  int* ngoff = goff + (kPwMaxPatches + 1);
  int* out_n = ngoff + (kPwMaxPatches + 1);   // [0] ground, [1] non-ground, [2] status
  unsigned long long* items = reinterpret_cast<unsigned long long*>(h->key_a.get());   // [>= R]
  QB_CUDA_TRY(h, cudaMemsetAsync(count, 0, (kPwMaxPatches + 1) * sizeof(int), h->stream));
  QB_CUDA_TRY(h, cudaMemsetAsync(out_n, 0, 4 * sizeof(int), h->stream));
  const int nb = (n + 255) / 256;
  pw_bin_kernel<<<nb, 256, 0, h->stream>>>(pts, n, c, patch_of, count);
  pw_scan_kernel<<<1, 1024, 0, h->stream>>>(count, NP, start, cursor);
  pw_scatter_kernel<<<nb, 256, 0, h->stream>>>(pts, n, patch_of, cursor, items);
  const size_t smem = (size_t)kPwMaxPatchPts * 9;
  QB_CUDA_TRY(h, ensure_dyn_smem(h->device, (const void*)pw_patch_kernel, smem));
  pw_patch_kernel<<<NP, kPwThreads, smem, h->stream>>>(pts, c, start, items, kPwMaxPatchPts, ng_ground, ng_non, rank, out_n + 2);
  pw_offsets_kernel<<<1, 1024, 0, h->stream>>>(ng_ground, ng_non, NP, goff, ngoff, out_n);
  pw_gather_kernel<<<NP, 256, 0, h->stream>>>(pts, start, ng_ground, ng_non, items, rank, goff, ngoff, h->pw_out, h->pw_out + R);
  h->launches += 6;
  QB_CUDA_TRY(h, cudaGetLastError());
  int host_n[3];
  QB_CUDA_TRY(h, cudaMemcpyAsync(host_n, out_n, 3 * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  QB_CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  *n_ground = host_n[0];
  *n_nonground = host_n[1];
  *status = host_n[2];
  return QB200_OK;
}


// ------------------------------------------------------------------------------------------------
// Range-image sub-cluster removal: ImageProjection::segmentCloud in "Patchwork" mode (include/imageProjection.hpp:273-294).
// The reference grows one segment at a time with a breadth-first queue (labelComponents, :483-579); the pair criterion
// (angle between neighbouring range pixels, :530-541) is symmetric, so its segments are the connected components of the pixel
// graph -- built here with a lock-free union-find (roots = lowest pixel index = the reference's seed pixel in its row-major
// sweep, :427-430), followed by per-component statistics and an ordered extraction.
//   ip_project_kernel  point -> pixel (:308-352); the LAST input point of a pixel wins (atomicMax on the input index)
//   ip_range_kernel    winner -> range image, parent = own pixel (or -1: nothing projected, maskGround :354-363)
//   ip_union_kernel    one thread per pixel and forward neighbour: union when the angle criterion holds
//   ip_stats_kernel    flatten; component size and the set of rows touched by its pixels other than the seed (lineCountFlag, :545)
//   ip_kind_kernel     feasibility of every pixel's segment (:559-571), counts per block of 1024 pixels
//   ip_extract_kernel  the two outputs in row-major order (:424-481): block base from the counts, one block scan inside
// ------------------------------------------------------------------------------------------------
struct IpDev {
  qb200_segment_params p;
  float sin_x, cos_x, sin_y, cos_y;
  int nnb;
  int nb[8][2];
};

__device__ __forceinline__ bool ip_project(const float4 pt, const qb200_segment_params& sp, int* row, int* col, float* range) {
  const float vert = (float)((double)(qb_atan2f(pt.z, sqrtf(pt.x * pt.x + pt.y * pt.y)) * 180.0f) / 3.14159265358979323846);
  const float rf = (vert + sp.ang_bottom) / sp.ang_res_y;
  if (!(rf > -1.0f) || !(rf < (float)sp.n_scan)) return false;
  const int r = (int)rf;
  if (r < 0 || r >= sp.n_scan) return false;
  const float hor = (float)((double)(qb_atan2f(pt.x, pt.y) * 180.0f) / 3.14159265358979323846);
  const double cd = -round(((double)hor - 90.0) / (double)sp.ang_res_x) + (double)(sp.horizon_scan / 2);
  if (!(cd >= 0.0) || !(cd < 4.0e9)) return false;
  long long c = (long long)cd;
  if (c >= sp.horizon_scan) c -= sp.horizon_scan;
  if (c < 0 || c >= sp.horizon_scan) return false;
  const float rg = sqrtf(pt.x * pt.x + pt.y * pt.y + pt.z * pt.z);
  if (rg < 0.1f) return false;
  *row = r; *col = (int)c; *range = rg;
  return true;
}

__global__ void __launch_bounds__(256) ip_project_kernel(const float4* __restrict__ pts, int n, IpDev c, int* __restrict__ winner) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = pts[i];
  if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return;   // copyPointCloud, :260-266
  int r, col; float rg;
  if (!ip_project(p, c.p, &r, &col, &rg)) return;
  atomicMax(&winner[r * c.p.horizon_scan + col], i);
}

__global__ void __launch_bounds__(256) ip_range_kernel(const float4* __restrict__ pts, int npix, const int* __restrict__ winner,
                                                       float* __restrict__ range, int* __restrict__ parent, int* __restrict__ size,
                                                       unsigned long long* __restrict__ rows) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= npix) return;
  const int w = winner[q];
  float rg = FLT_MAX;
  if (w >= 0) {
    const float4 p = pts[w];
    rg = sqrtf(p.x * p.x + p.y * p.y + p.z * p.z);
  }
  range[q] = rg;
  parent[q] = w >= 0 ? q : -1;
  size[q] = 0;
  rows[q] = 0ull;
}

__device__ __forceinline__ int ip_find(const int* parent, int a) {
  for (;;) {
    const int pa = ((volatile const int*)parent)[a];
    if (pa == a) return a;
    a = pa;
  }
}

__global__ void __launch_bounds__(256) ip_union_kernel(int npix, IpDev c, const float* __restrict__ range, int* parent) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= npix) return;
  const float ra = range[q];
  if (ra == FLT_MAX) return;
  const int H = c.p.n_scan, Wd = c.p.horizon_scan;
  const int fx = q / Wd, fy = q - fx * Wd;
  for (int t = 0; t < c.nnb; ++t) {
    const int tx = fx + c.nb[t][0];
    int ty = fy + c.nb[t][1];
    if (tx < 0 || tx >= H) continue;
    if (ty < 0) ty = Wd - 1;
    if (ty >= Wd) ty = 0;
    const int o = tx * Wd + ty;
    if (o <= q) continue;             // every pixel pair once (the criterion is symmetric); o == q: Wd wrap of a 1-column image
    const float rb = range[o];
    if (rb == FLT_MAX) continue;
    const float d1 = fmaxf(ra, rb), d2 = fminf(ra, rb);
    const bool same_row = c.nb[t][0] == 0;
    const float angle = qb_atan2f(d2 * (same_row ? c.sin_x : c.sin_y), d1 - d2 * (same_row ? c.cos_x : c.cos_y));
    if (!(angle > c.p.segment_theta)) continue;
    int a = q, b = o;
    for (;;) {   // link the larger root under the smaller one
      a = ip_find(parent, a);
      b = ip_find(parent, b);
      if (a == b) break;
      if (a < b) { const int tmp = a; a = b; b = tmp; }
      const int old = atomicMin(&parent[a], b);
      if (old == a) break;
      a = old;
    }
  }
}

__global__ void __launch_bounds__(256) ip_stats_kernel(int npix, int Wd, int* parent, int* __restrict__ size, unsigned long long* __restrict__ rows) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= npix) return;
  if (((volatile int*)parent)[q] < 0) return;
  const int root = ip_find(parent, q);
  atomicAdd(&size[root], 1);
  if (q != root) atomicOr(&rows[root], 1ull << (q / Wd));
}

// feasibility of every occupied pixel's segment (:559-571) -> kind[] (0 empty, 1 valid segment, 2 outlier) and the two counts of
// every block of 1024 pixels
__global__ void __launch_bounds__(1024) ip_kind_kernel(int npix, IpDev c, const int* __restrict__ winner, const int* parent, const int* __restrict__ size,
                                                       const unsigned long long* __restrict__ rows, unsigned char* __restrict__ kind_out,
                                                       int* __restrict__ blk_cnt) {
  __shared__ int s_v, s_o;
  if (threadIdx.x == 0) { s_v = 0; s_o = 0; }
  __syncthreads();
  const int q = blockIdx.x * 1024 + threadIdx.x;
  int kind = 0;
  if (q < npix && winner[q] >= 0) {
    const int root = ip_find(parent, q);
    const int sz = size[root];
    bool feasible = sz >= c.p.min_pts_for_subclustering;
    if (!feasible && sz >= c.p.segment_valid_point_num) feasible = __popcll(rows[root]) >= c.p.segment_valid_line_num;
    kind = feasible ? 1 : 2;
  }
  if (q < npix) kind_out[q] = (unsigned char)kind;
  const unsigned bv = __ballot_sync(0xffffffffu, kind == 1), bo = __ballot_sync(0xffffffffu, kind == 2);
  if ((threadIdx.x & 31) == 0) {
    if (bv) atomicAdd(&s_v, __popc(bv));
    if (bo) atomicAdd(&s_o, __popc(bo));
  }
  __syncthreads();
  if (threadIdx.x == 0) { blk_cnt[2 * blockIdx.x] = s_v; blk_cnt[2 * blockIdx.x + 1] = s_o; }
}

// ordered extraction (row-major, :424-481): block base = counts of the preceding blocks, one block scan inside
__global__ void __launch_bounds__(1024) ip_extract_kernel(const float4* __restrict__ pts, int npix, const int* __restrict__ winner,
                                                          const unsigned char* __restrict__ kind_in, const int* __restrict__ blk_cnt,
                                                          float4* __restrict__ valid, float4* __restrict__ outlier, int* __restrict__ out_n) {
  __shared__ int sm[33];
  __shared__ int s_base[2];
  int bv = 0, bo = 0;
  for (int b = threadIdx.x; b < (int)blockIdx.x; b += 1024) { bv += blk_cnt[2 * b]; bo += blk_cnt[2 * b + 1]; }
  int tot;
  block_excl_scan(bv, sm, &tot);
  if (threadIdx.x == 0) s_base[0] = tot;
  block_excl_scan(bo, sm, &tot);
  if (threadIdx.x == 0) s_base[1] = tot;
  __syncthreads();
  const int q = blockIdx.x * 1024 + threadIdx.x;
  const int kind = q < npix ? (int)kind_in[q] : 0;
  int both;
  const int ex = block_excl_scan((kind == 1 ? 1 : 0) | ((kind == 2 ? 1 : 0) << 16), sm, &both);
  if (kind) {
    float4 p = pts[winner[q]];
    p.w = 1.0f;
    if (kind == 1) valid[s_base[0] + (ex & 0xFFFF)] = p;
    else outlier[s_base[1] + (ex >> 16)] = p;
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) { out_n[0] = s_base[0] + (both & 0xFFFF); out_n[1] = s_base[1] + (both >> 16); }
}

// grown to the largest image of the lane so far; a failed call keeps the old buffer
static int ensure_ip_scratch(Lane* h, int npix) {
  if (h->ip_buf && h->ip_npix >= npix) return QB200_OK;
  DeviceMem<void> buf;
  // per pixel: rows u64 | valid float4 | outlier float4 | winner, parent, size int | range float | kind u8 ; + out_n [2] + block counts
  QB_CUDA_TRY(h, buf.alloc_bytes((size_t)npix * (8 + 16 + 16 + 4 * 4 + 1) + 16 + 8 * (size_t)((npix + 1023) / 1024) + 64));
  h->ip_buf = std::move(buf);
  h->ip_npix = npix;
  return QB200_OK;
}

static bool ip_params_valid(const qb200_segment_params& sp) {
  return sp.n_scan >= 1 && sp.n_scan <= 64 && sp.horizon_scan >= 8 && sp.horizon_scan <= 8192 && sp.ang_res_x > 0 && sp.ang_res_y > 0 &&
         sp.neighbor_mode >= 0 && sp.neighbor_mode <= 2 && sp.min_pts_for_subclustering >= 0 && sp.segment_valid_point_num >= 0 &&
         sp.segment_valid_line_num >= 0;
}

// pts: n device points.  Leaves the outputs in the handle's scratch; *valid_dev / *outlier_dev point at them.
int launch_segment_cloud(Lane* h, const float4* pts, int n, const qb200_segment_params& sp, int* n_valid, int* n_outlier,
                         const float4** valid_dev, const float4** outlier_dev) {
  *n_valid = *n_outlier = 0;
  if (!ip_params_valid(sp)) return QB200_ERR_BAD_ARG;
  const int npix = sp.n_scan * sp.horizon_scan;
  if (int rc = ensure_ip_scratch(h, npix)) return rc;
  unsigned char* b = reinterpret_cast<unsigned char*>(h->ip_buf.get());
  float4* valid = reinterpret_cast<float4*>(b); b += (size_t)npix * 16;      // 16-byte records first: aligned for any image size
  float4* outlier = reinterpret_cast<float4*>(b); b += (size_t)npix * 16;
  unsigned long long* rows = reinterpret_cast<unsigned long long*>(b); b += (size_t)npix * 8;
  int* winner = reinterpret_cast<int*>(b); b += (size_t)npix * 4;
  int* parent = reinterpret_cast<int*>(b); b += (size_t)npix * 4;
  int* size = reinterpret_cast<int*>(b); b += (size_t)npix * 4;
  float* range = reinterpret_cast<float*>(b); b += (size_t)npix * 4;
  int* out_n = reinterpret_cast<int*>(b); b += 16;
  int* blk_cnt = reinterpret_cast<int*>(b); b += 8 * (size_t)((npix + 1023) / 1024);
  unsigned char* kind = b;
  *valid_dev = valid; *outlier_dev = outlier;
  IpDev c;
  c.p = sp;
  // segmentAlphaX / segmentAlphaY and their sine / cosine (:132-133, :535-541): constants of the call, evaluated on the host
  const float alpha_x = (float)((double)sp.ang_res_x / 180.0 * 3.14159265358979323846), alpha_y = (float)((double)sp.ang_res_y / 180.0 * 3.14159265358979323846);
  c.sin_x = sinf(alpha_x); c.cos_x = cosf(alpha_x); c.sin_y = sinf(alpha_y); c.cos_y = cosf(alpha_y);
  static const int n4[4][2] = {{-1, 0}, {0, 1}, {0, -1}, {1, 0}};
  static const int n8[8][2] = {{-1, 0}, {0, 1}, {0, -1}, {1, 0}, {-1, -1}, {-1, 1}, {1, 1}, {1, -1}};
  static const int nx[4][2] = {{-1, -1}, {-1, 1}, {1, 1}, {1, -1}};
  c.nnb = sp.neighbor_mode == QB200_NEIGHBORS_8 ? 8 : 4;
  for (int i = 0; i < 8; ++i) { c.nb[i][0] = 0; c.nb[i][1] = 0; }
  for (int i = 0; i < c.nnb; ++i) {
    const int(*src)[2] = sp.neighbor_mode == QB200_NEIGHBORS_4 ? n4 : (sp.neighbor_mode == QB200_NEIGHBORS_8 ? n8 : nx);
    c.nb[i][0] = src[i][0]; c.nb[i][1] = src[i][1];
  }
  QB_CUDA_TRY(h, cudaMemsetAsync(winner, 0xFF, (size_t)npix * sizeof(int), h->stream));   // -1
  const int gp = (npix + 255) / 256;
  if (n > 0) ip_project_kernel<<<(n + 255) / 256, 256, 0, h->stream>>>(pts, n, c, winner);
  ip_range_kernel<<<gp, 256, 0, h->stream>>>(pts, npix, winner, range, parent, size, rows);
  ip_union_kernel<<<gp, 256, 0, h->stream>>>(npix, c, range, parent);
  ip_stats_kernel<<<gp, 256, 0, h->stream>>>(npix, sp.horizon_scan, parent, size, rows);
  const int nblk = (npix + 1023) / 1024;
  ip_kind_kernel<<<nblk, 1024, 0, h->stream>>>(npix, c, winner, parent, size, rows, kind, blk_cnt);
  ip_extract_kernel<<<nblk, 1024, 0, h->stream>>>(pts, npix, winner, kind, blk_cnt, valid, outlier, out_n);
  h->launches += 6;
  QB_CUDA_TRY(h, cudaGetLastError());
  int host_n[2];
  QB_CUDA_TRY(h, cudaMemcpyAsync(host_n, out_n, 2 * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  QB_CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  *n_valid = host_n[0];
  *n_outlier = host_n[1];
  return QB200_OK;
}

}  // namespace qb

extern "C" void qb200_default_patchwork_params(qb200_patchwork_params* p) {  // config/patchwork_params.yaml:1-48
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->sensor_height = 1.723;
  p->th_seeds = 0.25;
  p->th_dist = 0.125;
  p->max_range = 80.0;
  p->min_range = 2.7;
  p->uprightness_thr = 0.707;
  p->adaptive_seed_selection_margin = -1.1;
  p->global_elevation_threshold = -0.5;
  const double mr[4] = {2.7, 12.3625, 22.025, 41.35};
  const double et[4] = {-1.2, -0.9984, -0.851, -0.605};
  const double ft[4] = {0.0001, 0.000125, 0.000185, 0.000185};
  const int ns[4] = {16, 32, 54, 32}, nr[4] = {2, 4, 4, 4};
  for (int k = 0; k < 4; ++k) {
    p->min_ranges_each_zone[k] = mr[k]; p->elevation_thresholds[k] = et[k]; p->flatness_thresholds[k] = ft[k];
    p->num_sectors_each_zone[k] = ns[k]; p->num_rings_each_zone[k] = nr[k];
  }
  p->num_iter = 3;
  p->num_lpr = 20;
  p->num_min_pts = 80;
  p->using_global_elevation = 0;
  p->num_zones = 4;
  p->num_thresholds = 4;
}

extern "C" void qb200_default_segment_params(qb200_segment_params* p) {  // "Velodyne-64-HDE", imageProjection.hpp:87-94; "4CrossNeighbor"
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->n_scan = 64;
  p->horizon_scan = 1800;
  p->ang_res_x = (float)(360.0 / (double)(float)1800);
  p->ang_res_y = (float)(26.9 / (double)(float)63);
  p->ang_bottom = 25.0f;
  p->segment_theta = (float)(60.0 / 180.0 * 3.14159265358979323846);
  p->neighbor_mode = QB200_NEIGHBORS_4_CROSS;
  p->min_pts_for_subclustering = 30;
  p->segment_valid_point_num = 5;
  p->segment_valid_line_num = 3;
}
