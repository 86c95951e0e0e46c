// pose.cu -- K10 (GNC-TLS yaw) + K11 (component-wise translation estimate, COTE).   sm_90a
//
// Replaces the tail of Quatro::computeTransformation (include/quatro.hpp:806-936):
// chain TIMs over the sorted clique (:817-844), solveForRotation2D (:430-572, with
// teaser::utils::svdRot2d, include/teaser/utils.h:151-166), rotation-inlier bookkeeping (:857-874),
// solveForTranslation / estimate (:585-747) and the final inlier list (:914-930).
// One CTA per registration pair, everything in fp64, the whole GNC loop inside the kernel.
//
//  * svdRot2d: for a 2x2 correlation H = sum w x y^T the rotation V U^T (with the det fix) is the
//    maximiser of trace(R H), i.e. yaw = atan2(H01 - H10, H00 + H11): no SVD is needed.
//  * COTE: the 2c interval end points are sorted with a bitonic network on the key (value, insertion index) -- the total
//    order a stable sort by value produces -- in shared memory, or for cliques of more than kPoseSmemClique members in a
//    global-memory workspace of the pair (same code, L2-resident) -- and the running
//    sums of the sweep are then accumulated sequentially by one thread in exactly the reference's
//    order, so the argmin and the "median" candidate set follow the CPU path.
//
// A pose wave (qb200_solve_pose_batch_*) runs the same kernel on cliques the caller supplies: inlier_import_kernel brings each set's
// ids into its clique slot and refuses a set with an id outside [0, L) before pose_kernel runs; pose_records_kernel writes the
// refused sets' records after it.
#include "handle.cuh"

namespace qb {

constexpr int kPoseThreads = 256;

__device__ __forceinline__ double block_sum(double v, double* scratch) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if (lane_id() == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += scratch[w];
  return t;
}
__device__ __forceinline__ double block_max(double v, double* scratch) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane_id() == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = scratch[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) t = fmax(t, scratch[w]);
  return t;
}

static int next_pow2(int n) {
  int p = 32;
  while (p < n) p <<= 1;
  return p;
}
__host__ __device__ inline size_t pose_smem_bytes(int Lp) {
  return (size_t)4 * Lp * sizeof(double) + (size_t)4 * Lp * sizeof(unsigned short) + (size_t)2 * Lp;
}

// ascending bitonic sort of n2 (power of two) keys (val, tag); every thread of the block calls it
__device__ void bitonic_sort(double* val, unsigned short* tag, int n2) {
  for (int k = 2; k <= n2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < n2; t += blockDim.x) {
        const int x = t ^ j;
        if (x > t) {
          const double a = val[t], b = val[x];
          const unsigned short ta = tag[t], tb = tag[x];
          const bool gt = (a > b) || (a == b && ta > tb);
          const bool up = (t & k) == 0;
          if (up ? gt : !gt) {
            val[t] = b; val[x] = a;
            tag[t] = tb; tag[x] = ta;
          }
        }
      }
      __syncthreads();
    }
  }
}

template <bool kWs>
__global__ void __launch_bounds__(kPoseThreads) pose_kernel(const float4* __restrict__ ma, const float4* __restrict__ mb, const int* __restrict__ n_corr,
                                                            int Lc, int Lp, int Lg, unsigned char* __restrict__ ws, const int* __restrict__ clique_all,
                                                            const int* __restrict__ n_clique, const PairSolve* __restrict__ solve,
                                                            qb200_result* __restrict__ results, unsigned char* __restrict__ rot_mask_out,
                                                            unsigned char* __restrict__ trans_mask_out, int* __restrict__ final_inl,
                                                            int* __restrict__ n_final) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ double scratch[kPoseThreads / 32];
  __shared__ double s_bcast[4];
  __shared__ int s_ibcast[4];
  __shared__ int s_scan[33];

  const int pair = blockIdx.x, tid = threadIdx.x;
  const int L = n_corr[pair];
  const int c = n_clique[pair];
  if ((c > Lp) != kWs) return;  // the other instance solves this pair
  const PoseParams& pp = solve[pair].pp;
  // workspace of Lq = power-of-two capacity (so the bitonic networks fit): shared memory (Lp) for cliques of up to Lp members, else
  // the pair's slot of ws (Lg = next_pow2(Lc)).  At Lq = 32768 the 65536 COTE events fill the u16 tags 0..65535 without padding.
  //   ev[2Lq] f64 | wX[Lq] f64 | aux[Lq] f64 | tag[2Lq] u16 | ctag[Lq] u16 | list[Lq] u16 | rm[Lq] u8 | tm[Lq] u8
  constexpr bool in_smem = !kWs;
  const int Lq = in_smem ? Lp : Lg;
  double* ev = reinterpret_cast<double*>(in_smem ? smem_raw : ws + (size_t)pair * pose_smem_bytes(Lg));
  double* wX = ev + 2 * Lq;
  double* aux = wX + Lq;
  unsigned short* tag = reinterpret_cast<unsigned short*>(aux + Lq);
  unsigned short* ctag = tag + 2 * Lq;
  unsigned short* list = ctag + Lq;
  unsigned char* rm = reinterpret_cast<unsigned char*>(list + Lq);
  unsigned char* tm = rm + Lq;
  const float4* __restrict__ A = ma + (size_t)pair * Lc;
  const float4* __restrict__ B = mb + (size_t)pair * Lc;
  const int* __restrict__ cl = clique_all + (size_t)pair * Lc;
  qb200_result* __restrict__ res = results + pair;

  if (c <= 1) {  // quatro.hpp:809-813 (output stays identity here instead of "untouched")
    if (tid == 0) {
      res->valid = 0;
      res->status = (L < 2) ? QB200_DEGENERATE_INPUT : QB200_DEGENERATE_CLIQUE;
      res->clique_size = c; res->gnc_iters = 0; res->n_rot_inliers = 0; res->n_final_inliers = 0; res->cost = 0.0;
      for (int i = 0; i < 16; ++i) res->T[i] = (i % 5 == 0) ? 1.0 : 0.0;
      n_final[pair] = 0;
    }
    return;
  }

  // ---- GNC-TLS on the XY rows of the chain TIMs ----
  for (int j = tid; j < c; j += kPoseThreads) wX[j] = 1.0;
  double noise_bound_sq = pp.rot_noise_bound * pp.rot_noise_bound;
  if (noise_bound_sq < 1e-16) noise_bound_sq = 1e-2;
  double mu = 1.0, prev_cost = INFINITY, cost = INFINITY;
  double r00 = 1.0, r01 = 0.0, r10 = 0.0, r11 = 1.0;
  int iters = 0;
  __syncthreads();
  for (int it = 0; it < pp.max_iterations; ++it) {
    iters = it + 1;
    double h00 = 0.0, h01 = 0.0, h10 = 0.0, h11 = 0.0;
    for (int j = tid; j < c; j += kPoseThreads) {
      const int root = cl[j], leaf = (j != c - 1) ? cl[j + 1] : cl[0];
      const float4 ar = A[root], al = A[leaf], br = B[root], bl = B[leaf];
      const double x0 = (double)al.x - (double)ar.x, x1 = (double)al.y - (double)ar.y;
      const double y0 = (double)bl.x - (double)br.x, y1 = (double)bl.y - (double)br.y;
      const double w = wX[j];
      h00 += x0 * w * y0; h01 += x0 * w * y1; h10 += x1 * w * y0; h11 += x1 * w * y1;
    }
    h00 = block_sum(h00, scratch); h01 = block_sum(h01, scratch); h10 = block_sum(h10, scratch); h11 = block_sum(h11, scratch);
    const double cc = h00 + h11, ss = h01 - h10;
    const double nn = sqrt(cc * cc + ss * ss);
    double cs = 1.0, sn = 0.0;
    if (nn > 0.0) { cs = cc / nn; sn = ss / nn; }
    r00 = cs; r01 = -sn; r10 = sn; r11 = cs;
    double mymax = -INFINITY;
    for (int j = tid; j < c; j += kPoseThreads) {
      const int root = cl[j], leaf = (j != c - 1) ? cl[j + 1] : cl[0];
      const float4 ar = A[root], al = A[leaf], br = B[root], bl = B[leaf];
      const double x0 = (double)al.x - (double)ar.x, x1 = (double)al.y - (double)ar.y;
      const double y0 = (double)bl.x - (double)br.x, y1 = (double)bl.y - (double)br.y;
      const double dx = y0 - (r00 * x0 + r01 * x1), dy = y1 - (r10 * x0 + r11 * x1);
      const double r2 = dx * dx + dy * dy;
      aux[j] = r2;
      mymax = fmax(mymax, r2);
    }
    if (it == 0) {
      const double max_residual = block_max(mymax, scratch);
      mu = 1 / (2 * max_residual / noise_bound_sq - 1);
      if (mu <= 0) break;
    }
    const double th1 = (mu + 1) / mu * noise_bound_sq;
    const double th2 = mu / (mu + 1) * noise_bound_sq;
    double pc = 0.0;
    for (int j = tid; j < c; j += kPoseThreads) {
      const double r2 = aux[j];
      pc += wX[j] * r2;
      double w;
      if (r2 >= th1) w = 0;
      else if (r2 <= th2) w = 1;
      else w = sqrt(noise_bound_sq * mu * (mu + 1) / r2) - mu;
      wX[j] = w;
    }
    cost = block_sum(pc, scratch);
    const double cost_diff = fabs(cost - prev_cost);
    mu = mu * pp.gnc_factor;
    prev_cost = cost;
    if (cost_diff < pp.cost_threshold) break;
  }
  __syncthreads();
  for (int j = tid; j < c; j += kPoseThreads) rm[j] = wX[j] >= 0.4 ? 1 : 0;
  __syncthreads();

  // ---- rotation inliers (quatro.hpp:857-874): ordered list of j with mask[j-1] && mask[j] (cyclic) ----
  int n_rot = 0;
  {
    int carry = 0;
    for (int base = 0; base < c; base += kPoseThreads) {
      const int j = base + tid;
      const int keep = (j < c && rm[j] && rm[j == 0 ? c - 1 : j - 1]) ? 1 : 0;
      int tot;
      const int ex = block_excl_scan(keep, s_scan, &tot);
      if (keep) list[carry + ex] = (unsigned short)j;
      carry += tot;
    }
    n_rot = carry;
  }
  __syncthreads();
  const bool use_rot = pp.use_rot_inliers && n_rot > 0;
  const int N = use_rot ? n_rot : c;

  // full rotation: Rz(yaw) (* RyRx when given, quatro.hpp:419-426)
  double R[9] = {r00, r01, 0.0, r10, r11, 0.0, 0.0, 0.0, 1.0};
  double Q[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (pp.use_RyRx) {
    double Rn[9];
    for (int i = 0; i < 9; ++i) Q[i] = pp.RyRx[i];
    for (int r = 0; r < 3; ++r)
      for (int k = 0; k < 3; ++k) Rn[3 * r + k] = R[3 * r] * Q[k] + R[3 * r + 1] * Q[3 + k] + R[3 * r + 2] * Q[6 + k];
    for (int i = 0; i < 9; ++i) R[i] = Rn[i];
  }

  // ---- COTE per axis ----
  const double range = pp.cote_range;
  double tvec[3] = {0.0, 0.0, 0.0};
  for (int i = tid; i < N; i += kPoseThreads) tm[i] = 1;
  int n2 = 2;
  while (n2 < 2 * N) n2 <<= 1;
  for (int ax = 0; ax < 3; ++ax) {
    __syncthreads();
    for (int i = tid; i < N; i += kPoseThreads) {
      const int v = use_rot ? cl[list[i]] : cl[i];
      const float4 a = A[v], b = B[v];
      double sx = (double)a.x, sy = (double)a.y, sz = (double)a.z;
      if (!use_rot) {
        const double tx = Q[0] * sx + Q[1] * sy + Q[2] * sz, ty = Q[3] * sx + Q[4] * sy + Q[5] * sz, tz = Q[6] * sx + Q[7] * sy + Q[8] * sz;
        sx = tx; sy = ty; sz = tz;
      }
      const double rr = 1.0 * R[3 * ax] * sx + 1.0 * R[3 * ax + 1] * sy + 1.0 * R[3 * ax + 2] * sz;
      const double bb = ax == 0 ? (double)b.x : (ax == 1 ? (double)b.y : (double)b.z);
      const double X = bb - rr;
      wX[i] = X;
      ev[2 * i] = X - range; tag[2 * i] = (unsigned short)(2 * i);
      ev[2 * i + 1] = X + range; tag[2 * i + 1] = (unsigned short)(2 * i + 1);
    }
    for (int t = 2 * N + tid; t < n2; t += kPoseThreads) { ev[t] = INFINITY; tag[t] = 0xFFFF; }
    __syncthreads();
    bitonic_sort(ev, tag, n2);
    if (tid == 0) {
      const double weight = 1.0 / (range * range);
      double ranges_inverse_sum = 0.0;
      for (int i = 0; i < N; ++i) ranges_inverse_sum += range;
      double dot_X_weights = 0, dot_weights_consensus = 0, sum_xi = 0, sum_xi_square = 0;
      int card = 0, min_idx = 0, min_card = 0;
      double min_cost = 0.0, min_xhat = 0.0;
      for (int i = 0; i < 2 * N; ++i) {
        const int idx = tag[i] >> 1;
        const int epsilon = (tag[i] & 1) ? -1 : 1;
        const double Xi = wX[idx];
        card += epsilon;
        dot_weights_consensus += epsilon * weight;
        dot_X_weights += epsilon * weight * Xi;
        ranges_inverse_sum -= epsilon * range;
        sum_xi += epsilon * Xi;
        sum_xi_square += epsilon * Xi * Xi;
        const double x_hat = dot_X_weights / dot_weights_consensus;
        const double residual = card * x_hat * x_hat + sum_xi_square - 2 * sum_xi * x_hat;
        const double x_cost = residual + ranges_inverse_sum;
        if (i == 0 || x_cost < min_cost) { min_cost = x_cost; min_idx = i; min_card = card; min_xhat = x_hat; }
      }
      s_bcast[0] = min_xhat;
      s_ibcast[0] = min_idx;
      s_ibcast[1] = min_card;
    }
    __syncthreads();
    double est = s_bcast[0];
    if (pp.cote_median) {
      const int min_idx = s_ibcast[0], n_card = s_ibcast[1];
      if (n_card > 0) {
        int m2 = 1;
        while (m2 < n_card) m2 <<= 1;
        for (int j = tid; j < m2; j += kPoseThreads) {
          aux[j] = j < n_card ? wX[tag[min_idx - j] >> 1] : INFINITY;
        }
        __syncthreads();
        // tags are irrelevant for plain values: a scratch tag array keeps the sorted events intact
        for (int j = tid; j < m2; j += kPoseThreads) ctag[j] = 0;
        __syncthreads();
        if (m2 > 1) bitonic_sort(aux, ctag, m2);
        if (n_card == 1) est = aux[0];
        else est = (aux[n_card / 2 - 1] + aux[n_card / 2]) / 2.0;
      }
    }
    tvec[ax] = est;
    __syncthreads();
    for (int i = tid; i < N; i += kPoseThreads) tm[i] = (tm[i] && (fabs(wX[i] - est) <= range)) ? 1 : 0;
  }
  __syncthreads();

  // ---- final inliers (quatro.hpp:914-930) ----
  int n_fin = 0;
  {
    int carry = 0;
    for (int base = 0; base < N; base += kPoseThreads) {
      const int i = base + tid;
      const int keep = (i < N && tm[i]) ? 1 : 0;
      int tot;
      const int ex = block_excl_scan(keep, s_scan, &tot);
      if (keep) final_inl[(size_t)pair * Lc + carry + ex] = use_rot ? cl[list[i]] : cl[i];
      carry += tot;
    }
    n_fin = carry;
  }
  for (int j = tid; j < c; j += kPoseThreads) rot_mask_out[(size_t)pair * Lc + j] = rm[j];
  // members past the N COTE inputs (rotation-inlier COTE) get 0, so the mask never shows what an earlier pair left in the slot
  for (int i = tid; i < c; i += kPoseThreads) trans_mask_out[(size_t)pair * Lc + i] = i < N ? tm[i] : 0;
  if (tid == 0) {
    res->valid = 1;
    res->status = QB200_OK;
    res->clique_size = c; res->gnc_iters = iters; res->n_rot_inliers = n_rot; res->n_final_inliers = n_fin; res->cost = cost;
    double* T = res->T;  // column-major
    T[0] = R[0]; T[1] = R[3]; T[2] = R[6]; T[3] = 0.0;
    T[4] = R[1]; T[5] = R[4]; T[6] = R[7]; T[7] = 0.0;
    T[8] = R[2]; T[9] = R[5]; T[10] = R[8]; T[11] = 0.0;
    T[12] = tvec[0]; T[13] = tvec[1]; T[14] = tvec[2]; T[15] = 1.0;
    n_final[pair] = n_fin;
  }
}

// per-pair bookkeeping counters -> result record (runs before pose_kernel fills the solver fields)
__global__ void fill_counters_kernel(qb200_result* __restrict__ results, int n_pairs, WaveCounters c, int have_frontend) {
  const int pair = blockIdx.x * blockDim.x + threadIdx.x;
  if (pair >= n_pairs) return;
  qb200_result* r = results + pair;
  r->n_src_vox = have_frontend ? c.n_vox[2 * pair] : 0;
  r->n_tgt_vox = have_frontend ? c.n_vox[2 * pair + 1] : 0;
  r->n_mutual = have_frontend ? c.n_mutual[pair] : 0;
  r->n_corr = c.n_corr[pair];
  r->max_core = c.max_core[pair];
  r->n_edges = c.n_edges[pair] / 2;
  r->flags = c.flags[pair];
}

// status fix-up after the solve: front-end failures (capacity / voxel overflow) invalidate the pair
__global__ void finalize_status_kernel(qb200_result* __restrict__ results, int n_pairs, WaveCounters c) {
  const int pair = blockIdx.x * blockDim.x + threadIdx.x;
  if (pair >= n_pairs) return;
  const int s0 = c.cloud_status[2 * pair], s1 = c.cloud_status[2 * pair + 1];
  const int bad = s0 != 0 ? s0 : s1;
  if (bad != 0) {
    qb200_result* r = results + pair;
    r->valid = 0;
    r->status = bad;
    for (int i = 0; i < 16; ++i) r->T[i] = (i % 5 == 0) ? 1.0 : 0.0;
  }
}

// One CTA per set of a pose wave: the caller's ids (device memory in place, host ids from the staging) into the set's clique slot, in
// the caller's order, duplicates kept.  A set with an id outside [0, L) gets n_clique = 0 and QB200_ERR_BAD_ARG in bad[set]; it is
// decided before pose_kernel runs, so no point is read through such an id.
__global__ void __launch_bounds__(kPoseThreads) inlier_import_kernel(const InlierSrc* __restrict__ src, const int* __restrict__ n_corr, int Lc,
                                                                     int* __restrict__ clique, int* __restrict__ n_clique, int* __restrict__ bad) {
  const int set = blockIdx.x;
  const InlierSrc e = src[set];
  const unsigned L = (unsigned)n_corr[set];
  int* __restrict__ cl = clique + (size_t)set * Lc;
  int out = 0;
  for (int i = threadIdx.x; i < e.n; i += kPoseThreads) {
    const int v = e.ids[i];
    out |= (unsigned)v >= L;  // -1 and INT32_MAX alike
    cl[i] = v;
  }
  out = __syncthreads_or(out);
  if (threadIdx.x == 0) {
    n_clique[set] = out ? 0 : e.n;
    bad[set] = out ? QB200_ERR_BAD_ARG : QB200_OK;
  }
}

// after pose_kernel: a refused set's record (pose_kernel solved it as an empty clique) becomes QB200_ERR_BAD_ARG with n_corr = L
__global__ void pose_records_kernel(qb200_result* __restrict__ results, int n_sets, const int* __restrict__ bad, const int* __restrict__ n_corr) {
  const int set = blockIdx.x * blockDim.x + threadIdx.x;
  if (set >= n_sets || bad[set] == QB200_OK) return;
  qb200_result r = {};
  r.status = bad[set];
  r.n_corr = n_corr[set];
  for (int i = 0; i < 16; ++i) r.T[i] = (i % 5 == 0) ? 1.0 : 0.0;
  results[set] = r;
}

__global__ void iota_clique_kernel(const int* __restrict__ n_corr, const PairSolve* __restrict__ solve, int Lc, int* __restrict__ clique,
                                   int* __restrict__ n_clique, int* __restrict__ max_core) {
  const int pair = blockIdx.y;
  if (solve[pair].mode != QB200_INLIER_NONE) return;
  const int L = n_corr[pair];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < L) clique[(size_t)pair * Lc + i] = i;
  if (i == 0) { n_clique[pair] = L; max_core[pair] = 0; }
}

size_t pose_ws_bytes(int Lc) { return pose_smem_bytes(next_pow2(Lc)); }

PoseParams pose_params(const qb200_params& p) {
  PoseParams pp;
  pp.rot_noise_bound = p.rot_noise_bound;  // resolved by the entry point (api.cu: resolve_params, the handle's latch)
  pp.cote_range = p.cote_noise_bound * sqrt(p.cbar2);
  pp.gnc_factor = p.rotation_gnc_factor;
  pp.cost_threshold = p.rotation_cost_threshold;
  pp.max_iterations = p.rotation_max_iterations;
  pp.cote_median = p.cote_mode == QB200_COTE_MEDIAN;
  pp.use_rot_inliers = p.using_rot_inliers_when_estimating_cote;
  pp.use_RyRx = p.use_pre_estimated_RyRx;
  for (int i = 0; i < 9; ++i) pp.RyRx[i] = p.RyRx[i];
  return pp;
}

int launch_pose(Lane* h, int n_pairs) {
  if (n_pairs <= 0) return QB200_OK;
  const int Lp = next_pow2(h->Lc < kPoseSmemClique ? h->Lc : kPoseSmemClique);
  const size_t smem = pose_smem_bytes(Lp);
  QB_CUDA_TRY(h, ensure_dyn_smem(h->device, (const void*)pose_kernel<false>, smem));
  pose_kernel<false><<<n_pairs, kPoseThreads, smem, h->stream>>>(h->ma, h->mb, h->ctr.n_corr, h->Lc, Lp, next_pow2(h->Lc), h->pose_ws, h->clique,
                                                                 h->ctr.n_clique, h->d_solve, h->d_results, h->rot_mask, h->trans_mask, h->final_inl,
                                                                 h->ctr.n_final);
  h->launches++;
  if (h->Lc > kPoseSmemClique) {  // cliques above Lp members: the same code on the pair's slot of pose_ws
    pose_kernel<true><<<n_pairs, kPoseThreads, 0, h->stream>>>(h->ma, h->mb, h->ctr.n_corr, h->Lc, Lp, next_pow2(h->Lc), h->pose_ws, h->clique,
                                                               h->ctr.n_clique, h->d_solve, h->d_results, h->rot_mask, h->trans_mask, h->final_inl,
                                                               h->ctr.n_final);
    h->launches++;
  }
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

int launch_fill_counters(Lane* h, int n_pairs, int have_frontend) {
  fill_counters_kernel<<<(n_pairs + 127) / 128, 128, 0, h->stream>>>(h->d_results, n_pairs, h->ctr, have_frontend);
  h->launches++;
  return QB200_OK;
}
int launch_finalize_status(Lane* h, int n_pairs) {
  finalize_status_kernel<<<(n_pairs + 127) / 128, 128, 0, h->stream>>>(h->d_results, n_pairs, h->ctr);
  h->launches++;
  return QB200_OK;
}
int launch_inlier_import(Lane* h, int n_sets) {
  if (n_sets <= 0) return QB200_OK;
  inlier_import_kernel<<<n_sets, kPoseThreads, 0, h->stream>>>(h->d_inl, h->ctr.n_corr, h->Lc, h->clique, h->ctr.n_clique, h->ctr.cloud_status);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}
int launch_pose_records(Lane* h, int n_sets) {
  if (n_sets <= 0) return QB200_OK;
  pose_records_kernel<<<(n_sets + 127) / 128, 128, 0, h->stream>>>(h->d_results, n_sets, h->ctr.cloud_status, h->ctr.n_corr);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}
int launch_iota_clique(Lane* h, int n_pairs) {
  const dim3 g((h->Lc + 255) / 256, n_pairs);
  iota_clique_kernel<<<g, 256, 0, h->stream>>>(h->ctr.n_corr, h->d_solve, h->Lc, h->clique, h->ctr.n_clique, h->ctr.max_core);
  h->launches++;
  return QB200_OK;
}

}  // namespace qb
