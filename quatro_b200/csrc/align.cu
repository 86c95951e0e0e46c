// align.cu -- the example's step after computeTransformation (examples/run_global_registration.cpp:253-288) for every pair of an
// align wave (qb200_align_batch_*): the source scan and the matched source keypoints transformed by the pose, and the good matches.
//
//  - align_good_kernel, one CTA per set: checks every correspondence index first (a set with one out of range is refused before any
//    point is read through it), then gathers each correspondence's keypoints, transforms the source one (matched4), applies the
//    good-match test and compacts the good ids in correspondence order with a block-wide ballot scan, so the order never depends on
//    the block size.
//  - align_points_kernel, a grid over (set, chunk of kAlignPts points) of the whole wave in one launch: streams the clouds of the sets
//    align_good_kernel did not refuse, 16 bytes in and 16 bytes out per point, with the set's pose in registers.
//
// Both evaluate pcl::transformPointCloud with a Matrix4d exactly: every product and sum in double, rounded one at a time, left to
// right, then the cast to float (align_point).
#include "handle.cuh"

namespace qb {
namespace {

constexpr int kAlignThreads = 256;
constexpr int kAlignWarps = kAlignThreads / 32;
constexpr int kAlignPerThread = kAlignPts / kAlignThreads;
static_assert(kAlignPts % kAlignThreads == 0, "align_points_kernel: whole points per thread");

// (float)(T(r,0)*x + T(r,1)*y + T(r,2)*z + T(r,3)) for r = 0..2 in double, no contraction; w copied.  A point with a non-finite x, y
// or z is copied through unchanged (PCL's !is_dense branch).
__device__ __forceinline__ float4 align_point(const double (&T)[12], const float4 p) {
  if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return p;
  const double x = p.x, y = p.y, z = p.z;
  float r[3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
    r[i] = __double2float_rn(
        __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4 * i], x), __dmul_rn(T[4 * i + 1], y)), __dmul_rn(T[4 * i + 2], z)), T[4 * i + 3]));
  return make_float4(r[0], r[1], r[2], p.w);
}

__device__ __forceinline__ void load_pose(const AlignSrc& e, double (&T)[12]) {
#pragma unroll
  for (int i = 0; i < 12; ++i) T[i] = e.T[i];
}

__global__ void __launch_bounds__(kAlignThreads) align_good_kernel(const AlignSrc* __restrict__ sets, int* __restrict__ status,
                                                                   int* __restrict__ n_good) {
  const int set = blockIdx.x, tid = threadIdx.x;
  const AlignSrc& e = sets[set];
  const int n = e.n_corr, cap = e.cap_corr;
  const unsigned ns = (unsigned)e.n_src, nt = (unsigned)e.n_tgt;
  const int2* __restrict__ corr = e.corr;
  int bad = 0;
  for (int k = tid; k < n; k += kAlignThreads) {
    const int2 c = corr[k];
    bad |= (unsigned)c.x >= ns || (unsigned)c.y >= nt;  // -1 and INT32_MAX alike
  }
  if (__syncthreads_or(bad)) {
    if (tid == 0) status[set] = QB200_ERR_BAD_ARG;
    return;
  }
  double T[12];
  load_pose(e, T);
  const double thr = e.thr;
  const float4* __restrict__ src = e.src_kp;
  const float4* __restrict__ tgt = e.tgt_kp;
  float4* __restrict__ matched = e.matched;
  float4* __restrict__ good = e.good;
  int* __restrict__ ids = e.good_ids;
  __shared__ int warp_total[kAlignWarps];
  const int lane = tid & 31, warp = tid >> 5;
  int base = 0;  // good correspondences before this round
  for (int k0 = 0; k0 < n; k0 += kAlignThreads) {
    const int k = k0 + tid;
    bool pass = false;
    float4 m = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k < n) {
      const int2 c = corr[k];
      m = align_point(T, src[c.x]);
      const float4 t = tgt[c.y];
      if (matched && k < cap) matched[k] = m;
      const double dx = __dsub_rn((double)m.x, (double)t.x), dy = __dsub_rn((double)m.y, (double)t.y),
                   dz = __dsub_rn((double)m.z, (double)t.z);
      pass = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz))) < thr;
    }
    const unsigned ball = __ballot_sync(0xffffffffu, pass);
    if (lane == 0) warp_total[warp] = __popc(ball);
    __syncthreads();
    int before = __popc(ball & ((1u << lane) - 1u)), total = 0;
#pragma unroll
    for (int w = 0; w < kAlignWarps; ++w) {
      const int t = warp_total[w];
      before += w < warp ? t : 0;
      total += t;
    }
    const int pos = base + before;
    if (pass && pos < cap) {
      if (ids) ids[pos] = k;
      if (good) good[pos] = m;
    }
    base += total;
    __syncthreads();  // warp_total is rewritten by the next round
  }
  if (tid == 0) {
    status[set] = QB200_OK;
    n_good[set] = base;
  }
}

// Block b belongs to the last set whose first block is <= b (sets without blocks share their successor's blk0).  The cloud and the
// output may be the same staging region (host-kind clouds aligned into host-kind output): each thread reads its points before it
// writes them, so they carry no __restrict__.
__global__ void __launch_bounds__(kAlignThreads) align_points_kernel(const AlignSrc* __restrict__ sets, int n_sets,
                                                                     const int* __restrict__ status) {
  const int b = blockIdx.x;
  int lo = 0, hi = n_sets - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (sets[mid].blk0 <= b) lo = mid;
    else hi = mid - 1;
  }
  if (status[lo] != QB200_OK) return;
  const AlignSrc& e = sets[lo];
  double T[12];
  load_pose(e, T);
  const int m = min(e.n_points, e.cap_points);
  const float4* in = e.cloud;
  float4* out = e.aligned;
  const int first = (b - e.blk0) * kAlignPts + threadIdx.x;
  float4 v[kAlignPerThread];
#pragma unroll
  for (int r = 0; r < kAlignPerThread; ++r) {
    const int i = first + r * kAlignThreads;
    if (i < m) v[r] = in[i];
  }
#pragma unroll
  for (int r = 0; r < kAlignPerThread; ++r) {
    const int i = first + r * kAlignThreads;
    if (i < m) out[i] = align_point(T, v[r]);
  }
}

}  // namespace

int launch_align_good(Lane* h, int n_sets) {
  if (n_sets <= 0) return QB200_OK;
  align_good_kernel<<<n_sets, kAlignThreads, 0, h->stream>>>(h->d_aln, h->ctr.cloud_status, h->ctr.n_final);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

int launch_align_points(Lane* h, int n_blocks, int n_sets) {
  if (n_blocks <= 0 || n_sets <= 0) return QB200_OK;
  align_points_kernel<<<n_blocks, kAlignThreads, 0, h->stream>>>(h->d_aln, n_sets, h->ctr.cloud_status);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

}  // namespace qb
