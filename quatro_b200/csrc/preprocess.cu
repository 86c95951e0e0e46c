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
constexpr int kPwStride = kPwMaxPatches + 1;   // per-scan entries of every per-patch array
// per-scan count block of a wave, [scan][kPpCnt]: ground, non-ground, patchwork status, valid, outlier (+ 3 spare)
constexpr int kPpCnt = 8;

struct PwDev {   // one scan's parameters + the derived patch table
  qb200_patchwork_params p;
  int patch_base[QB200_PW_MAX_ZONES + 1];
  int n_patches;
};

struct IpDev {   // one scan's range-image parameters + the constants the host derives from them
  qb200_segment_params p;
  float sin_x, cos_x, sin_y, cos_y;
  int nnb;
  int nb[8][2];
};

// One scan's entry of a lane's pre-processing table (h_pp / d_pp, [2S]): what every kernel of the wave reads for its scan.  The range
// image of scan s sits at pixel pix0 of the wave's per-pixel arrays (a prefix sum of n_scan * horizon_scan over the wave) and its
// counts per block of 1024 pixels at block blk0, so a wave of small images reserves only what they need.
struct PpScan {
  PwDev pw;         // unused by qb200_segment_cloud
  IpDev ip;         // unused without sub-cluster removal
  long long pix0;
  int blk0, npix;   // npix = n_scan * horizon_scan (0 without sub-cluster removal)
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

// Every kernel serves a wave of scans: blockIdx.y (or the one CTA of the per-scan scans) is the scan s, it reads scan s's entry of the
// table, and scan s's scratch sits at fixed strides -- R points (patch_of, rank, items, the two outputs) and kPwStride patches
// (counts, starts, offsets) -- so that a scan's results never depend on the wave it rides in.  The per-patch grids cover the wave's
// largest patch count; CTAs past their scan's count exit.
__global__ void __launch_bounds__(256) pw_bin_kernel(const float4* const* __restrict__ pts_of, const int* __restrict__ n_of,
                                                     const PpScan* __restrict__ tab, int R, int* __restrict__ patch_of, int* __restrict__ count) {
  const int s = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_of[s]) return;
  const PwDev& c = tab[s].pw;
  const float4 p = pts_of[s][i];
  int pid = -1;
  // non-finite points never enter (D11); :356-368 drops everything below -1.8 sensor_height
  if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && !((double)p.z < -1.8 * c.p.sensor_height)) pid = pw_patch_of(p, c);
  patch_of[(size_t)s * R + i] = pid;
  if (pid >= 0) atomicAdd(&count[(size_t)s * kPwStride + pid], 1);
}

// one CTA per scan: start[] = exclusive scan of count[0..np), start[np] = total; cursor = copy of start
__global__ void __launch_bounds__(1024) pw_scan_kernel(const int* __restrict__ count, const PpScan* __restrict__ tab, int* __restrict__ start,
                                                       int* __restrict__ cursor) {
  __shared__ int sm[33];
  const int np = tab[blockIdx.x].pw.n_patches;
  const size_t o = (size_t)blockIdx.x * kPwStride;
  count += o; start += o; cursor += o;
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

__global__ void __launch_bounds__(256) pw_scatter_kernel(const float4* const* __restrict__ pts_of, const int* __restrict__ n_of, int R,
                                                         const int* __restrict__ patch_of, int* __restrict__ cursor,
                                                         unsigned long long* __restrict__ items) {
  const int s = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_of[s]) return;
  const int pid = patch_of[(size_t)s * R + i];
  if (pid < 0) return;
  const float z = pts_of[s][i].z + 0.0f;  // -0 -> +0: the comparator z_a < z_b does not tell them apart
  unsigned zb = __float_as_uint(z);
  zb = (zb & 0x80000000u) ? ~zb : (zb | 0x80000000u);  // order-preserving
  const int pos = atomicAdd(&cursor[(size_t)s * kPwStride + pid], 1);
  items[(size_t)s * R + pos] = ((unsigned long long)zb << 32) | (unsigned)i;
}

// D17 (oracle/preprocess_oracle.inc): unit vector of the smallest eigenvalue's eigenspace when the closed form's eigenvector is
// undefined -- all points identical or on one line, every row of cov - lambda I parallel to one direction u.  (0,0,1) when it lies
// in that eigenspace, else (u_y, -u_x, 0) normalised, or (1,0,0) for a vertical u.
__device__ __forceinline__ void pw_degenerate_normal(const float cov[9], float ev, float e[3]) {
  float m[9];
  for (int i = 0; i < 9; ++i) m[i] = cov[i];
  m[0] -= ev; m[4] -= ev; m[8] -= ev;
  if (m[2] == 0.0f && m[5] == 0.0f && m[8] == 0.0f) { e[0] = 0.0f; e[1] = 0.0f; e[2] = 1.0f; return; }
  const float l0 = qb_dot3(&m[0], &m[0]), l1 = qb_dot3(&m[3], &m[3]), l2 = qb_dot3(&m[6], &m[6]);
  const float* u = (l0 >= l1 && l0 >= l2) ? &m[0] : (l1 >= l2 ? &m[3] : &m[6]);
  const float h = sqrtf(u[0] * u[0] + u[1] * u[1]);
  if (h > 0.0f) { e[0] = u[1] / h; e[1] = -u[0] / h; e[2] = 0.0f; }
  else { e[0] = 1.0f; e[1] = 0.0f; e[2] = 0.0f; }
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
  if (!(isfinite(e[0]) && isfinite(e[1]) && isfinite(e[2]))) pw_degenerate_normal(cov, ev, e);   // D17
  if (e[2] < 0.0f) { e[0] = -e[0]; e[1] = -e[1]; e[2] = -e[2]; }
  const float tr = cov[0] + cov[4] + cov[8];
  *surf = (tr != 0.0f) ? fabsf(ev / tr) : 0.0f;
  n[0] = e[0]; n[1] = e[1]; n[2] = e[2];
  mean[0] = accu[6]; mean[1] = accu[7]; mean[2] = accu[8];
}

// One CTA per (patch, scan).  keys: sorted (z | index); flag[p] = sorted position p belongs to the current ground set.
__global__ void __launch_bounds__(kPwThreads) pw_patch_kernel(const float4* const* __restrict__ pts_of, const PpScan* __restrict__ tab, int R,
                                                              const int* __restrict__ start, unsigned long long* __restrict__ items,
                                                              int cap_pow2, int* __restrict__ n_ground, int* __restrict__ n_nonground,
                                                              int* __restrict__ rank_out, int* __restrict__ cnt) {
  if ((int)blockIdx.x >= tab[blockIdx.y].pw.n_patches) return;
  // the scan's entry in shared memory: the serial sections below (one thread) read it where they use it, at shared-memory latency
  __shared__ PwDev s_entry;
  for (int w = threadIdx.x; w < (int)(sizeof(PwDev) / 4); w += blockDim.x)
    reinterpret_cast<int*>(&s_entry)[w] = reinterpret_cast<const int*>(&tab[blockIdx.y].pw)[w];
  __syncthreads();
  const PwDev& c = s_entry;
  extern __shared__ __align__(16) unsigned char pw_smem[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(pw_smem);   // [cap_pow2]
  unsigned char* flag = reinterpret_cast<unsigned char*>(keys + cap_pow2);     // [cap_pow2]
  __shared__ float s_part[kPwThreads / 32][9];
  __shared__ int s_cnt[kPwThreads / 32];
  __shared__ float s_plane[8];   // n[3], mean[3], surf, th_dist_d
  __shared__ double s_lpr;
  __shared__ int s_init, s_keep, s_scan[33];
  const qb200_patchwork_params& pp = c.p;
  const int pid = blockIdx.x, scan = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float4* __restrict__ pts = pts_of[scan];
  start += (size_t)scan * kPwStride; n_ground += (size_t)scan * kPwStride; n_nonground += (size_t)scan * kPwStride;
  items += (size_t)scan * R; rank_out += (size_t)scan * R;
  const int s0 = start[pid], m = start[pid + 1] - s0;
  if (!(m > pp.num_min_pts) || m > kPwMaxPatchPts) {   // :382 -- small patches are dropped altogether
    if (tid == 0) {
      n_ground[pid] = 0; n_nonground[pid] = 0;
      if (m > kPwMaxPatchPts) cnt[(size_t)scan * kPpCnt + 2] = QB200_CAPACITY_EXCEEDED;
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

// one CTA per scan: exclusive scans of the per-patch output counts; totals -> cnt[0] (ground), cnt[1] (non-ground)
__global__ void __launch_bounds__(1024) pw_offsets_kernel(const int* __restrict__ n_ground, const int* __restrict__ n_nonground,
                                                          const PpScan* __restrict__ tab, int* __restrict__ goff, int* __restrict__ ngoff,
                                                          int* __restrict__ cnt) {
  __shared__ int sm[33];
  const int np = tab[blockIdx.x].pw.n_patches;
  const size_t o = (size_t)blockIdx.x * kPwStride;
  n_ground += o; n_nonground += o; goff += o; ngoff += o;
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
  if (threadIdx.x == 0) { cnt[(size_t)blockIdx.x * kPpCnt] = cg; cnt[(size_t)blockIdx.x * kPpCnt + 1] = cn; }
}

// The caller's device arrays of a wave (ground, non-ground, valid, outlier): scan s's entries start at s * cap, entries at or past cap
// are not written; nullptr = not asked for.  The kernels write them next to the lane's scratch copy.
struct PpDev {
  float4* arr[4];
  long long cap;
};

// one CTA per (patch, scan): scan s's outputs go to out[s * R ...]: ground at [0, n_ground), non-ground at [n_ground, n_ground + n_nonground)
__global__ void __launch_bounds__(256) pw_gather_kernel(const float4* const* __restrict__ pts_of, const PpScan* __restrict__ tab, int R,
                                                        const int* __restrict__ start, const int* __restrict__ n_ground,
                                                        const int* __restrict__ n_nonground, const unsigned long long* __restrict__ items,
                                                        const int* __restrict__ rank, const int* __restrict__ goff, const int* __restrict__ ngoff,
                                                        const int* __restrict__ cnt, float4* __restrict__ out, PpDev dst) {
  const int pid = blockIdx.x, scan = blockIdx.y;
  if (pid >= tab[scan].pw.n_patches) return;
  const size_t po = (size_t)scan * kPwStride + pid, ro = (size_t)scan * R;
  if (n_ground[po] + n_nonground[po] == 0) return;
  const float4* __restrict__ pts = pts_of[scan];
  const int s0 = start[po], m = start[po + 1] - s0;
  const int g0 = goff[po], n0 = cnt[(size_t)scan * kPpCnt] + ngoff[po];   // non-ground part of out follows the ground part
  const int nn0 = ngoff[po];
  for (int p = threadIdx.x; p < m; p += blockDim.x) {
    const int code = rank[ro + s0 + p];
    const float4 q = pts[(unsigned)items[ro + s0 + p]];
    if (code & (1 << 30)) {
      const int pos = g0 + (code & ~(1 << 30));
      out[ro + pos] = q;
      if (dst.arr[0] && pos < dst.cap) dst.arr[0][scan * dst.cap + pos] = q;
    } else {
      out[ro + n0 + code] = q;
      const int pos = nn0 + code;
      if (dst.arr[1] && pos < dst.cap) dst.arr[1][scan * dst.cap + pos] = q;
    }
  }
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

// Scan s of a wave: the cloud tables of stage_raw (ptr[s], n[s]), or the non-ground part of the patchwork output (base != nullptr:
// base + s * R from cnt[s][0] on, cnt[s][1] points).
struct IpIn {
  const float4* const* ptr;
  const int* n;
  const float4* base;
  const int* cnt;
  int R;
};

__device__ __forceinline__ const float4* ip_input(const IpIn& in, int s, int* n) {
  if (in.base) {
    *n = in.cnt[(size_t)s * kPpCnt + 1];
    return in.base + (size_t)s * in.R + in.cnt[(size_t)s * kPpCnt];
  }
  *n = in.n[s];
  return in.ptr[s];
}

// blockIdx.y = scan; scan s's per-pixel entries are [tab[s].pix0, tab[s].pix0 + tab[s].npix) of every per-pixel array.  The
// per-pixel grids cover the wave's largest image; threads past their scan's image exit.
__global__ void __launch_bounds__(256) ip_project_kernel(IpIn in, const PpScan* __restrict__ tab, int* __restrict__ winner) {
  const int s = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  int n;
  const float4* pts = ip_input(in, s, &n);
  if (i >= n) return;
  const float4 p = pts[i];
  if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return;   // copyPointCloud, :260-266
  const PpScan& e = tab[s];
  int r, col; float rg;
  if (!ip_project(p, e.ip.p, &r, &col, &rg)) return;
  atomicMax(&winner[(size_t)e.pix0 + r * e.ip.p.horizon_scan + col], i);
}

__global__ void __launch_bounds__(256) ip_range_kernel(IpIn in, const PpScan* __restrict__ tab, const int* __restrict__ winner,
                                                       float* __restrict__ range, int* __restrict__ parent, int* __restrict__ size,
                                                       unsigned long long* __restrict__ rows) {
  const int s = blockIdx.y, q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= tab[s].npix) return;
  const size_t o = (size_t)tab[s].pix0 + q;
  const int w = winner[o];
  float rg = FLT_MAX;
  if (w >= 0) {
    int n;
    const float4 p = ip_input(in, s, &n)[w];
    rg = sqrtf(p.x * p.x + p.y * p.y + p.z * p.z);
  }
  range[o] = rg;
  parent[o] = w >= 0 ? q : -1;
  size[o] = 0;
  rows[o] = 0ull;
}

__device__ __forceinline__ int ip_find(const int* parent, int a) {
  for (;;) {
    const int pa = ((volatile const int*)parent)[a];
    if (pa == a) return a;
    a = pa;
  }
}

__global__ void __launch_bounds__(256) ip_union_kernel(const PpScan* __restrict__ tab, const float* __restrict__ range, int* parent) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= tab[blockIdx.y].npix) return;
  const IpDev& c = tab[blockIdx.y].ip;
  range += (size_t)tab[blockIdx.y].pix0;
  parent += (size_t)tab[blockIdx.y].pix0;
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

__global__ void __launch_bounds__(256) ip_stats_kernel(const PpScan* __restrict__ tab, int* parent, int* __restrict__ size,
                                                       unsigned long long* __restrict__ rows) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= tab[blockIdx.y].npix) return;
  const int Wd = tab[blockIdx.y].ip.p.horizon_scan;
  const size_t o = (size_t)tab[blockIdx.y].pix0;
  parent += o; size += o; rows += o;
  if (((volatile int*)parent)[q] < 0) return;
  const int root = ip_find(parent, q);
  atomicAdd(&size[root], 1);
  if (q != root) atomicOr(&rows[root], 1ull << (q / Wd));
}

// feasibility of every occupied pixel's segment (:559-571) -> kind[] (0 empty, 1 valid segment, 2 outlier) and the two counts of
// every block of 1024 pixels (blk_cnt: 2 entries per block, scan s's blocks from tab[s].blk0 on)
__global__ void __launch_bounds__(1024) ip_kind_kernel(const PpScan* __restrict__ tab, const int* __restrict__ winner, const int* parent,
                                                       const int* __restrict__ size, const unsigned long long* __restrict__ rows,
                                                       unsigned char* __restrict__ kind_out, int* __restrict__ blk_cnt) {
  const PpScan& e = tab[blockIdx.y];
  const int npix = e.npix;
  if ((int)blockIdx.x * 1024 >= npix) return;   // past the scan's image: the whole CTA
  __shared__ int s_v, s_o;
  if (threadIdx.x == 0) { s_v = 0; s_o = 0; }
  __syncthreads();
  const size_t o = (size_t)e.pix0;
  winner += o; parent += o; size += o; rows += o; kind_out += o;
  blk_cnt += (size_t)2 * e.blk0;
  const int q = blockIdx.x * 1024 + threadIdx.x;
  int kind = 0;
  if (q < npix && winner[q] >= 0) {
    const int root = ip_find(parent, q);
    const int sz = size[root];
    bool feasible = sz >= e.ip.p.min_pts_for_subclustering;
    if (!feasible && sz >= e.ip.p.segment_valid_point_num) feasible = __popcll(rows[root]) >= e.ip.p.segment_valid_line_num;
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

// ordered extraction (row-major, :424-481): block base = counts of the preceding blocks, one block scan inside.  Scan s's outputs go
// to out[pix0 ...]: valid segments at [0, n_valid), outliers at [n_valid, n_valid + n_outlier); counts -> cnt[s][3], cnt[s][4].
__global__ void __launch_bounds__(1024) ip_extract_kernel(IpIn in, const PpScan* __restrict__ tab, const int* __restrict__ winner,
                                                          const unsigned char* __restrict__ kind_in, const int* __restrict__ blk_cnt,
                                                          float4* __restrict__ out, int* __restrict__ cnt, PpDev dst) {
  __shared__ int sm[33];
  __shared__ int s_base[3];
  const int scan = blockIdx.y;
  const int npix = tab[scan].npix, nblk = (npix + 1023) / 1024;
  if ((int)blockIdx.x >= nblk) return;   // past the scan's image: the whole CTA
  const size_t o = (size_t)tab[scan].pix0;
  winner += o; kind_in += o; out += o;
  blk_cnt += (size_t)2 * tab[scan].blk0;
  int bv = 0, bo = 0, tv = 0;
  for (int b = threadIdx.x; b < nblk; b += 1024) {
    if (b < (int)blockIdx.x) { bv += blk_cnt[2 * b]; bo += blk_cnt[2 * b + 1]; }
    tv += blk_cnt[2 * b];
  }
  int tot;
  block_excl_scan(bv, sm, &tot);
  if (threadIdx.x == 0) s_base[0] = tot;
  block_excl_scan(bo, sm, &tot);
  if (threadIdx.x == 0) s_base[1] = tot;
  block_excl_scan(tv, sm, &tot);
  if (threadIdx.x == 0) s_base[2] = tot;
  __syncthreads();
  const int q = blockIdx.x * 1024 + threadIdx.x;
  const int kind = q < npix ? (int)kind_in[q] : 0;
  int both;
  const int ex = block_excl_scan((kind == 1 ? 1 : 0) | ((kind == 2 ? 1 : 0) << 16), sm, &both);
  if (kind) {
    int n;
    float4 p = ip_input(in, scan, &n)[winner[q]];
    p.w = 1.0f;
    const int pos = kind == 1 ? s_base[0] + (ex & 0xFFFF) : s_base[1] + (ex >> 16);
    out[kind == 1 ? pos : s_base[2] + pos] = p;
    float4* d = kind == 1 ? dst.arr[2] : dst.arr[3];
    if (d && pos < dst.cap) d[scan * dst.cap + pos] = p;
  }
  if ((int)blockIdx.x == nblk - 1 && threadIdx.x == 0) {
    cnt[(size_t)scan * kPpCnt + 3] = s_base[0] + (both & 0xFFFF);
    cnt[(size_t)scan * kPpCnt + 4] = s_base[1] + (both >> 16);
  }
}

static bool ip_params_valid(const qb200_segment_params& sp) {
  return sp.n_scan >= 1 && sp.n_scan <= 64 && sp.horizon_scan >= 8 && sp.horizon_scan <= 8192 && sp.ang_res_x > 0 && sp.ang_res_y > 0 &&
         sp.neighbor_mode >= 0 && sp.neighbor_mode <= 2 && sp.min_pts_for_subclustering >= 0 && sp.segment_valid_point_num >= 0 &&
         sp.segment_valid_line_num >= 0;
}

// ------------------------------------------------------------------------------------------------
// Waves.  One launch sequence serves up to 2S scans; the four entry points below run their scans through it on lane 0.
// ------------------------------------------------------------------------------------------------
// range-image scratch of a wave whose images have pix pixels and blk blocks of 1024 pixels in all: per pixel the output (float4), the
// row set (u64), winner, parent, size (int), range (float), kind (u8); per block its two counts
static size_t ip_bytes(long long pix, long long blk) { return (size_t)pix * (16 + 8 + 4 * 4 + 1) + 8 * (size_t)blk + 64; }

// Scratch of a wave of ns scans, grown on demand (a lane that never pre-processes holds none).  Each group -- the count block, the
// parameter table and their pinned mirrors, the patchwork buffers, the range-image buffer (ipb bytes, 0 = none) -- is allocated whole
// or not at all: a failed call leaves a group either as it was or empty, and the next call allocates it again.
static int ensure_pp_scratch(Lane* L, int ns, bool pw, size_t ipb) {
  const int C = 2 * L->S;
  const bool grow_pw = pw && ns > L->pw_scans, grow_ip = ipb > L->ip_cap;
  DeviceMem<int> cnt, ints;
  PinnedMem<int> hcnt;
  DeviceMem<PpScan> tab;
  PinnedMem<PpScan> htab;
  DeviceMem<float4> out;
  DeviceMem<void> ip;
  if (!L->pp_cnt) {
    QB_CUDA_TRY(L, cnt.alloc((size_t)C * kPpCnt));
    QB_CUDA_TRY(L, hcnt.alloc((size_t)C * kPpCnt));
    QB_CUDA_TRY(L, tab.alloc(C));
    QB_CUDA_TRY(L, htab.alloc(C));
  }
  if (grow_pw) {
    // the old buffers are idle (every wave ends in a sync): they go first, so the device never holds both
    L->pw_ints.reset(); L->pw_out.reset();
    L->pw_scans = 0;
    // patch_of [ns*R] | rank [ns*R] | count, start(+1), cursor, n_ground, n_nonground, goff, ngoff [ns*kPwStride each]
    QB_CUDA_TRY(L, ints.alloc((size_t)ns * (2 * (size_t)L->R + 7 * (size_t)kPwStride)));
    QB_CUDA_TRY(L, out.alloc((size_t)ns * L->R));
  }
  if (grow_ip) {
    L->ip_buf.reset();
    L->ip_cap = 0;
    QB_CUDA_TRY(L, ip.alloc_bytes(ipb));
  }
  if (!L->pp_cnt) { L->pp_cnt = std::move(cnt); L->pp_hcnt = std::move(hcnt); L->d_pp = std::move(tab); L->h_pp = std::move(htab); }
  if (grow_pw) { L->pw_ints = std::move(ints); L->pw_out = std::move(out); L->pw_scans = ns; }
  if (grow_ip) { L->ip_buf = std::move(ip); L->ip_cap = ipb; }
  return QB200_OK;
}

// a scan's Patchwork entry: its parameters and the first patch of every zone
static PwDev pw_entry(const qb200_patchwork_params& pp) {
  PwDev c;
  c.p = pp;
  c.patch_base[0] = 0;
  for (int k = 0; k < 4; ++k) c.patch_base[k + 1] = c.patch_base[k] + pp.num_sectors_each_zone[k] * pp.num_rings_each_zone[k];
  c.n_patches = c.patch_base[4];
  return c;
}

// a scan's range-image entry: its parameters, segmentAlphaX / segmentAlphaY's sine and cosine (:132-133, :535-541, evaluated on the
// host) and the neighbour offsets of its mode
static IpDev ip_entry(const qb200_segment_params& sp) {
  IpDev c;
  c.p = sp;
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
  return c;
}

// Enqueue ground removal of the wave's scans [0, ns) (cloud tables of stage_raw, entries d_pp[s]); scan s's outputs -> pw_out + s * R,
// its counts and status -> pp_cnt[s].  max_np = the wave's largest patch count.  Launches do not depend on ns or on the scans.
static int launch_patchwork_wave(Lane* L, int ns, int max_n, int max_np, const PpDev& dst) {
  const int R = L->R;
  const size_t P = (size_t)L->pw_scans * kPwStride;
  int* patch_of = L->pw_ints;
  int* rank = patch_of + (size_t)L->pw_scans * R;
  int* count = rank + (size_t)L->pw_scans * R;
  int* start = count + P;
  int* cursor = start + P;
  int* ng_ground = cursor + P;
  int* ng_non = ng_ground + P;
  int* goff = ng_non + P;
  int* ngoff = goff + P;
  unsigned long long* items = reinterpret_cast<unsigned long long*>(L->key_a.get());   // [2S * R] >= [ns * R]
  const PpScan* tab = L->d_pp;
  QB_CUDA_TRY(L, cudaMemsetAsync(count, 0, (size_t)ns * kPwStride * sizeof(int), L->stream));
  const dim3 gp((max_n + 255) / 256 > 0 ? (max_n + 255) / 256 : 1, ns);
  pw_bin_kernel<<<gp, 256, 0, L->stream>>>(L->d_cloud_ptr, L->d_cloud_n, tab, R, patch_of, count);
  pw_scan_kernel<<<ns, 1024, 0, L->stream>>>(count, tab, start, cursor);
  pw_scatter_kernel<<<gp, 256, 0, L->stream>>>(L->d_cloud_ptr, L->d_cloud_n, R, patch_of, cursor, items);
  const size_t smem = (size_t)kPwMaxPatchPts * 9;
  QB_CUDA_TRY(L, ensure_dyn_smem(L->device, (const void*)pw_patch_kernel, smem));
  pw_patch_kernel<<<dim3(max_np, ns), kPwThreads, smem, L->stream>>>(L->d_cloud_ptr, tab, R, start, items, kPwMaxPatchPts, ng_ground, ng_non,
                                                                     rank, L->pp_cnt);
  pw_offsets_kernel<<<ns, 1024, 0, L->stream>>>(ng_ground, ng_non, tab, goff, ngoff, L->pp_cnt);
  pw_gather_kernel<<<dim3(max_np, ns), 256, 0, L->stream>>>(L->d_cloud_ptr, tab, R, start, ng_ground, ng_non, items, rank, goff, ngoff,
                                                            L->pp_cnt, L->pw_out, dst);
  L->launches += 6;
  QB_CUDA_TRY(L, cudaGetLastError());
  return QB200_OK;
}

// Enqueue sub-cluster removal of the wave's scans [0, ns) read through `in` (entries d_pp[s]); scan s's outputs -> the range-image
// scratch + d_pp[s].pix0, its counts -> pp_cnt[s].  max_n bounds every scan's point count; the wave's images have pix pixels and blk
// blocks in all, max_npix pixels at most.
static int launch_segment_wave(Lane* L, int ns, int max_n, const IpIn& in, long long pix, long long blk, int max_npix, const PpDev& dst) {
  const size_t NPX = (size_t)pix;
  unsigned char* b = reinterpret_cast<unsigned char*>(L->ip_buf.get());
  float4* out = reinterpret_cast<float4*>(b); b += NPX * 16;      // 16-byte records first: aligned for any image size
  unsigned long long* rows = reinterpret_cast<unsigned long long*>(b); b += NPX * 8;
  int* winner = reinterpret_cast<int*>(b); b += NPX * 4;
  int* parent = reinterpret_cast<int*>(b); b += NPX * 4;
  int* size = reinterpret_cast<int*>(b); b += NPX * 4;
  float* range = reinterpret_cast<float*>(b); b += NPX * 4;
  int* blk_cnt = reinterpret_cast<int*>(b); b += 8 * (size_t)blk;
  unsigned char* kind = b;
  const PpScan* tab = L->d_pp;
  QB_CUDA_TRY(L, cudaMemsetAsync(winner, 0xFF, NPX * sizeof(int), L->stream));   // -1
  const dim3 gpt((max_n + 255) / 256 > 0 ? (max_n + 255) / 256 : 1, ns), gpx((max_npix + 255) / 256, ns), gbk((max_npix + 1023) / 1024, ns);
  ip_project_kernel<<<gpt, 256, 0, L->stream>>>(in, tab, winner);
  ip_range_kernel<<<gpx, 256, 0, L->stream>>>(in, tab, winner, range, parent, size, rows);
  ip_union_kernel<<<gpx, 256, 0, L->stream>>>(tab, range, parent);
  ip_stats_kernel<<<gpx, 256, 0, L->stream>>>(tab, parent, size, rows);
  ip_kind_kernel<<<gbk, 1024, 0, L->stream>>>(tab, winner, parent, size, rows, kind, blk_cnt);
  ip_extract_kernel<<<gbk, 1024, 0, L->stream>>>(in, tab, winner, kind, blk_cnt, out, L->pp_cnt, dst);
  L->launches += 6;
  QB_CUDA_TRY(L, cudaGetLastError());
  return QB200_OK;
}

// The caller's arrays of a whole call.  Host arrays are filled from the scratch after the counts are back, device arrays by the kernels.
struct PpOut {
  float4* arr[4];   // ground, non-ground, valid, outlier (nullptr: not asked for)
  long long cap;
  int device;
};

// One wave on lane L: scans [0, ns) whose pointers and sizes are in L->h_cloud_ptr / h_cloud_n (`kind` memory) through ground
// removal (pp) and then sub-cluster removal of its non-ground output (sp), or through sub-cluster removal alone (pp == nullptr).
// Scan s of the wave uses pp[s] / sp[s] when `each` is set, else pp[0] / sp[0]; it is scan first + s of `out`; its counts go to
// counts[s * 4 ...] (ground, non-ground, valid, outlier), its patchwork status to status[s].  The wave's parameter table goes to the
// device in one copy ahead of its scans, and its counts come back in one copy.
static int preprocess_wave(Lane* L, int ns, qb200_mem_kind kind, const qb200_patchwork_params* pp, const qb200_segment_params* sp, bool each,
                           const PpOut& out, long long first, int32_t* counts, int32_t* status) {
  int rc, max_n = 0, max_np = 0, max_npix = 0;
  long long pix = 0, blk = 0;
  for (int s = 0; s < ns; ++s) {
    max_n = L->h_cloud_n[s] > max_n ? L->h_cloud_n[s] : max_n;
    if (!sp) continue;
    const int npix = sp[each ? s : 0].n_scan * sp[each ? s : 0].horizon_scan;
    pix += npix;
    blk += (npix + 1023) / 1024;
  }
  if ((rc = ensure_pp_scratch(L, ns, pp != nullptr, sp ? ip_bytes(pix, blk) : 0))) return rc;
  pix = blk = 0;
  for (int s = 0; s < ns; ++s) {   // the previous wave ended in a sync: the pinned table is free
    PpScan& e = L->h_pp[s];
    e = PpScan{};
    if (pp) {
      e.pw = pw_entry(pp[each ? s : 0]);
      max_np = e.pw.n_patches > max_np ? e.pw.n_patches : max_np;
    }
    if (sp) {
      e.ip = ip_entry(sp[each ? s : 0]);
      e.npix = e.ip.p.n_scan * e.ip.p.horizon_scan;
      e.pix0 = pix;
      e.blk0 = (int)blk;
      pix += e.npix;
      blk += (e.npix + 1023) / 1024;
      max_npix = e.npix > max_npix ? e.npix : max_npix;
    }
  }
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->d_pp, L->h_pp, (size_t)ns * sizeof(PpScan), cudaMemcpyHostToDevice, L->stream));
  if ((rc = stage_raw(L, ns, kind, L->stream))) return rc;
  QB_CUDA_TRY(L, cudaMemsetAsync(L->pp_cnt, 0, (size_t)ns * kPpCnt * sizeof(int), L->stream));
  PpDev dst = {{nullptr, nullptr, nullptr, nullptr}, out.cap};
  if (out.device)
    for (int k = 0; k < 4; ++k) dst.arr[k] = out.arr[k] ? out.arr[k] + first * out.cap : nullptr;
  if (pp && (rc = launch_patchwork_wave(L, ns, max_n, max_np, dst))) return rc;
  if (sp) {
    IpIn in = {L->d_cloud_ptr, L->d_cloud_n, pp ? L->pw_out.get() : nullptr, L->pp_cnt, L->R};
    if ((rc = launch_segment_wave(L, ns, max_n, in, pix, blk, max_npix, dst))) return rc;
  }
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->pp_hcnt, L->pp_cnt, (size_t)ns * kPpCnt * sizeof(int), cudaMemcpyDeviceToHost, L->stream));
  QB_CUDA_TRY(L, cudaStreamSynchronize(L->stream));
  bool copied = false;
  for (int s = 0; s < ns; ++s) {
    const int* hc = L->pp_hcnt + (size_t)s * kPpCnt;
    const int c4[4] = {hc[0], hc[1], hc[3], hc[4]};
    for (int k = 0; k < 4; ++k) counts[4 * s + k] = c4[k];
    status[s] = hc[2];
    if (out.device) continue;
    for (int k = 0; k < 4; ++k) {
      const long long m = c4[k] < out.cap ? c4[k] : out.cap;
      if (!out.arr[k] || m <= 0) continue;
      // scratch of scan s: ground | non-ground at pw_out + s * R, valid | outlier at the range-image outputs + pix0
      const float4* src = k < 2 ? L->pw_out + (size_t)s * L->R + (k == 1 ? hc[0] : 0)
                                : reinterpret_cast<const float4*>(L->ip_buf.get()) + (size_t)L->h_pp[s].pix0 + (k == 3 ? hc[3] : 0);
      QB_CUDA_TRY(L, cudaMemcpyAsync(out.arr[k] + (first + s) * out.cap, src, (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost, L->stream));
      copied = true;
    }
  }
  if (copied) QB_CUDA_TRY(L, cudaStreamSynchronize(L->stream));
  return QB200_OK;
}

// true when an entry of the per-scan tables pp[0..n) / sp[0..n) (sp may be nullptr) fails the checks of a broadcast call; msg names
// the first such entry
static bool bad_entry(const qb200_patchwork_params* pp, const qb200_segment_params* sp, int n, char* msg, size_t len) {
  for (int i = 0; i < n; ++i) {
    const char* what = !pw_params_valid(pp[i]) ? "patchwork" : (sp && !ip_params_valid(sp[i])) ? "segment" : nullptr;
    if (what) {
      snprintf(msg, len, "invalid %s parameters of scan %d", what, i);
      return true;
    }
  }
  return false;
}

// qb200_preprocess_batch (each == false: pp[0] / sp[0] serve every scan) and qb200_preprocess_batch_each (one entry per scan): every
// check before any work, then waves of 2S scans on lane 0.
static int preprocess_call(qb200_handle* h, const float* const* scans4, const int32_t* n_points, int32_t n_scans, qb200_mem_kind kind,
                           const qb200_patchwork_params* pp, const qb200_segment_params* sp, bool each, const qb200_preprocess_out* out) {
  if (int rc = enter(h)) return rc;
  const char* why = nullptr;
  char msg[96];
  if (n_scans < 0 || (n_scans > 0 && (!scans4 || !n_points))) why = "n_scans < 0, or no scan / size table";
  else if (kind != QB200_MEM_HOST && kind != QB200_MEM_DEVICE) why = "unknown memory kind of the scans";
  else if (!each && (!pp || !pw_params_valid(*pp))) why = "invalid patchwork parameters";
  else if (!each && sp && !ip_params_valid(*sp)) why = "invalid segment parameters";
  else if (each && n_scans > 0 && !pp) why = "no patchwork parameter table";
  else if (each && bad_entry(pp, sp, n_scans, msg, sizeof(msg))) why = msg;
  else if (!out || !out->counts || !out->status) why = "no output descriptor, counts or status";
  else if (out->cap_per_scan < 1) why = "cap_per_scan < 1";
  else if (out->kind != QB200_MEM_HOST && out->kind != QB200_MEM_DEVICE) why = "unknown memory kind of the outputs";
  else if (out->kind == QB200_MEM_DEVICE && !(device_array_of(h, out->ground4, 16) && device_array_of(h, out->nonground4, 16) &&
                                              device_array_of(h, out->valid4, 16) && device_array_of(h, out->outlier4, 16)))
    why = "device output array is misaligned or not memory of the handle's device";
  Lane* L = h->lane[0].get();
  for (int i = 0; i < n_scans && !why; ++i)
    if (n_points[i] < 0 || n_points[i] > L->R || (n_points[i] > 0 && !scans4[i])) why = "scan is null or exceeds max_raw_points";
  if (why) {
    h->fail(__FILE__, __LINE__, why);
    return QB200_ERR_BAD_ARG;
  }
  const PpOut o = {{reinterpret_cast<float4*>(out->ground4), reinterpret_cast<float4*>(out->nonground4), reinterpret_cast<float4*>(out->valid4),
                    reinterpret_cast<float4*>(out->outlier4)},
                   out->cap_per_scan, out->kind == QB200_MEM_DEVICE ? 1 : 0};
  const int C = 2 * L->S;
  for (int w0 = 0; w0 < n_scans; w0 += C) {
    const int ns = n_scans - w0 < C ? n_scans - w0 : C;
    for (int s = 0; s < ns; ++s) {
      L->h_cloud_ptr[s] = reinterpret_cast<const float4*>(scans4[w0 + s]);
      L->h_cloud_n[s] = n_points[w0 + s];
    }
    const size_t e0 = each ? (size_t)w0 : 0;
    if (int rc = preprocess_wave(L, ns, kind, pp + e0, sp ? sp + e0 : nullptr, each, o, w0, out->counts + 4 * (size_t)w0, out->status + w0))
      return rc;
  }
  return QB200_OK;
}

}  // namespace qb

using namespace qb;

extern "C" {

// ---- pre-processing: ground removal (patchwork.hpp:329-455), a wave of one ----------------------------
int qb200_patchwork(qb200_handle* h, const float* pts4, int32_t n, const qb200_patchwork_params* p, float* ground4, int32_t* n_ground,
                    float* nonground4, int32_t* n_nonground) {
  if (int rc = enter(h)) return rc;
  if (!p || !n_ground || !n_nonground || n < 0 || (n > 0 && !pts4)) return QB200_ERR_BAD_ARG;
  *n_ground = *n_nonground = 0;
  Lane* L = h->lane[0].get();
  if (n > L->R) { h->fail(__FILE__, __LINE__, "n exceeds max_raw_points"); return QB200_ERR_BAD_ARG; }
  if (!pw_params_valid(*p)) return QB200_ERR_BAD_ARG;
  L->h_cloud_ptr[0] = reinterpret_cast<const float4*>(pts4);
  L->h_cloud_n[0] = n;
  const PpOut out = {{reinterpret_cast<float4*>(ground4), reinterpret_cast<float4*>(nonground4), nullptr, nullptr}, n, 0};
  int32_t counts[4], status = QB200_OK;
  if (int rc = preprocess_wave(L, 1, QB200_MEM_HOST, p, nullptr, false, out, 0, counts, &status)) return rc;
  *n_ground = counts[0];
  *n_nonground = counts[1];
  return status;
}

// ---- pre-processing: range-image sub-cluster removal (imageProjection.hpp:273-294), a wave of one ------------
int qb200_segment_cloud(qb200_handle* h, const float* pts4, int32_t n, const qb200_segment_params* p, float* valid4, int32_t* n_valid,
                        float* outlier4, int32_t* n_outlier) {
  if (int rc = enter(h)) return rc;
  if (!p || !n_valid || !n_outlier || n < 0 || (n > 0 && !pts4)) return QB200_ERR_BAD_ARG;
  *n_valid = *n_outlier = 0;
  Lane* L = h->lane[0].get();
  if (n > L->R) { h->fail(__FILE__, __LINE__, "n exceeds max_raw_points"); return QB200_ERR_BAD_ARG; }
  if (!ip_params_valid(*p)) return QB200_ERR_BAD_ARG;
  L->h_cloud_ptr[0] = reinterpret_cast<const float4*>(pts4);
  L->h_cloud_n[0] = n;
  const PpOut out = {{nullptr, nullptr, reinterpret_cast<float4*>(valid4), reinterpret_cast<float4*>(outlier4)}, (long long)p->n_scan * p->horizon_scan, 0};
  int32_t counts[4], status = QB200_OK;
  if (int rc = preprocess_wave(L, 1, QB200_MEM_HOST, nullptr, p, false, out, 0, counts, &status)) return rc;
  *n_valid = counts[2];
  *n_outlier = counts[3];
  return QB200_OK;
}

// ---- pre-processing of many scans: ground removal, then sub-cluster removal, in waves of 2S scans ----------
int qb200_preprocess_batch(qb200_handle* h, const float* const* scans4, const int32_t* n_points, int32_t n_scans, qb200_mem_kind kind,
                           const qb200_patchwork_params* pp, const qb200_segment_params* sp, const qb200_preprocess_out* out) {
  return preprocess_call(h, scans4, n_points, n_scans, kind, pp, sp, false, out);
}

// ---- the same with one parameter entry per scan ----------
int qb200_preprocess_batch_each(qb200_handle* h, const float* const* scans4, const int32_t* n_points, int32_t n_scans, qb200_mem_kind kind,
                                const qb200_patchwork_params* pp, const qb200_segment_params* sp, const qb200_preprocess_out* out) {
  return preprocess_call(h, scans4, n_points, n_scans, kind, pp, sp, true, out);
}

}  // extern "C"

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
