// api.cu -- the C-ABI of include/quatro_b200.h: handle lifetime, lanes, waves, pair lists, the scan cache and the batch entry
// points.  The single-pair stage entry points, the qb200_get_last_* getters and the debug hooks are in stages.cu.
#include <cmath>
#include <new>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <map>
#include <mutex>
#include <utility>
#include <vector>

#include "handle.cuh"

using namespace qb;

namespace {

__global__ void wave_init_kernel(int* ctr_block, int n_ints, int* bbox, int n_clouds) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_ints) ctr_block[i] = 0;
  if (i < n_clouds * 6) bbox[i] = (i % 6) < 3 ? INT_MAX : INT_MIN;
}

// ---- scan cache (qb200_cache_*): copies between the wave buffers of a lane and the per-scan cache slots ----
// blockIdx.z = cloud of the wave, blockIdx.y = 0..39 descriptor row | 40 voxel points | 41 normals | 42 counters
__global__ void cache_copy_kernel(int to_cache, const int* __restrict__ slot_of_cloud, int V, float4* __restrict__ w_vox, float4* __restrict__ w_nrm,
                                  float* __restrict__ w_desc, int* __restrict__ w_n, int* __restrict__ w_status, float4* __restrict__ c_vox,
                                  float4* __restrict__ c_nrm, float* __restrict__ c_desc, int* __restrict__ c_n, int* __restrict__ c_status) {
  const int cloud = blockIdx.z, slot = slot_of_cloud[cloud], row = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot < 0) return;
  const int n = to_cache ? w_n[cloud] : c_n[slot];
  if (row == 42) {
    if (q == 0) {
      if (to_cache) { c_n[slot] = w_n[cloud]; c_status[slot] = w_status[cloud]; }
      else { w_n[cloud] = c_n[slot]; w_status[cloud] = c_status[slot]; }
    }
    return;
  }
  if (q >= n || q >= V) return;
  if (row < kDescK) {
    float* w = w_desc + ((size_t)cloud * kDescK + row) * V + q;
    float* c = c_desc + ((size_t)slot * kDescK + row) * V + q;
    if (to_cache) *c = *w; else *w = *c;
  } else if (row == 40) {
    if (to_cache) c_vox[(size_t)slot * V + q] = w_vox[(size_t)cloud * V + q]; else w_vox[(size_t)cloud * V + q] = c_vox[(size_t)slot * V + q];
  } else {
    if (to_cache) c_nrm[(size_t)slot * V + q] = w_nrm[(size_t)cloud * V + q]; else w_nrm[(size_t)cloud * V + q] = c_nrm[(size_t)slot * V + q];
  }
}

// Carve the counter block at `base` into *c and return its size in ints; base == nullptr only counts.  One int block, so a wave
// reset is a single launch.  n_edges (long long) comes first, at an 8-byte offset; two spare ints close the block.
size_t carve_counters(int* base, size_t S, WaveCounters* c) {
  const size_t C = 2 * S;
  size_t n = 0;
  auto take = [&](size_t k) {
    int* p = base ? base + n : nullptr;
    n += k;
    return p;
  };
  c->n_edges = reinterpret_cast<long long*>(take(2 * S));
  c->n_valid = take(C);
  c->n_vox = take(C);
  c->n_fpfh = take(C);
  c->n_lat = take(C);
  c->n_cells = take(C);
  c->cloud_status = take(C);
  c->bbox = take(C * 6);
  c->vox_digits = take(C);
  c->n_mutual = take(S);
  c->n_corr = take(S);
  c->swapped = take(S);
  c->n_clique = take(S);
  c->max_core = take(S);
  c->n_final = take(S);
  c->flags = take(S);
  return n + 2;
}

// A new lane in *out with the settings of `like` (dims, device, n_sm, matcher switches, error sink), its own stream and every
// buffer of DESIGN §4.  On failure *out is left as it was.
int lane_alloc(const Lane& like, std::unique_ptr<Lane>* out) {
  std::unique_ptr<Lane> L(new (std::nothrow) Lane());
  if (!L) return QB200_ERR_CUDA;
  L->S = like.S; L->R = like.R; L->V = like.V; L->Lc = like.Lc; L->W = like.W; L->NS = like.NS;
  L->device = like.device; L->n_sm = like.n_sm; L->force_exact_match = like.force_exact_match; L->err = like.err;
  L->tc_verify = like.tc_verify; L->tc_prof = like.tc_prof;
  QB_CUDA_TRY(L, L->own_stream.create(cudaStreamNonBlocking));
  L->stream = L->own_stream;
  const size_t S = L->S, R = L->R, V = L->V, Lc = L->Lc, W = L->W, C = 2 * S;
  QB_CUDA_TRY(L, L->d_cloud_ptr.alloc(C));
  QB_CUDA_TRY(L, L->d_cloud_n.alloc(C));
  QB_CUDA_TRY(L, L->d_raw_off.alloc(C + 1));
  QB_CUDA_TRY(L, L->h_cloud_ptr.alloc(C));
  QB_CUDA_TRY(L, L->h_cloud_n.alloc(C));
  QB_CUDA_TRY(L, L->h_raw_off.alloc(C + 1));
  QB_CUDA_TRY(L, L->raw_stage.alloc(C * R));
  QB_CUDA_TRY(L, L->d_slot_of_cloud.alloc(C));
  QB_CUDA_TRY(L, L->h_slot_of_cloud.alloc(C));
  QB_CUDA_TRY(L, L->d_feat.alloc(C));
  QB_CUDA_TRY(L, L->h_feat.alloc(C));
  QB_CUDA_TRY(L, L->d_graph.alloc(S));
  QB_CUDA_TRY(L, L->h_graph.alloc(S));
  QB_CUDA_TRY(L, L->d_inl.alloc(S));
  QB_CUDA_TRY(L, L->h_inl.alloc(S));
  QB_CUDA_TRY(L, L->d_aln.alloc(S));
  QB_CUDA_TRY(L, L->h_aln.alloc(S));
  // the sort workspace serves the voxel sort (C*R items, digit histograms in val_a, chunk counts C*kVsChunks <= n_sort in val_b),
  // the lattice / norm sorts (C*V items) and, afterwards, the duplicate-class tables of K6 (2S*V + 2S words in key_a): size it for
  // the largest user
  const size_t n_sort = C * (R > V ? R : V) + 64;
  const size_t n_hist = C * 256 * ((R + kVsTile - 1) / kVsTile);
  QB_CUDA_TRY(L, L->key_a.alloc(n_sort));
  QB_CUDA_TRY(L, L->key_b.alloc(n_sort));
  QB_CUDA_TRY(L, L->val_a.alloc(n_sort > n_hist ? n_sort : n_hist));
  QB_CUDA_TRY(L, L->val_b.alloc(n_sort));
  QB_CUDA_TRY(L, L->aos_scratch.alloc(2 * V * kDescDim));
  // the library radix sort only sorts lattice / norm keys of clouds too large for cloud_sort_kernel: at most C*V items
  L->cub_bytes = sort_temp_bytes((int)(C * V));
  QB_CUDA_TRY(L, L->cub_temp.alloc_bytes(L->cub_bytes));
  QB_CUDA_TRY(L, L->vox_start.alloc(C * (V + 1)));
  QB_CUDA_TRY(L, L->vox_pts.alloc(C * V));
  QB_CUDA_TRY(L, L->cell_key.alloc(C * V));
  QB_CUDA_TRY(L, L->cell_start.alloc(C * (V + 1)));
  QB_CUDA_TRY(L, L->normals.alloc(C * V));
  QB_CUDA_TRY(L, L->spfh.alloc(C * V * kDescPad));
  QB_CUDA_TRY(L, L->nbr_list.alloc(C * kNbrGlobalCap * V));
  QB_CUDA_TRY(L, L->nbr_cnt.alloc(C * V));
  QB_CUDA_TRY(L, L->desc_t.alloc(C * kDescK * V));
  QB_CUDA_TRY(L, cudaMemset(L->desc_t, 0, C * kDescK * V * sizeof(float)));
  QB_CUDA_TRY(L, L->desc_tiles.alloc(C * kDescK * V * 3));
  QB_CUDA_TRY(L, cudaMemset(L->desc_tiles, 0, C * kDescK * V * 3 * sizeof(float)));
  QB_CUDA_TRY(L, L->desc_norm.alloc(C * V));
  QB_CUDA_TRY(L, L->tc_fallback.alloc(S));
  QB_CUDA_TRY(L, L->tc_stats.alloc(32));
  QB_CUDA_TRY(L, cudaMemset(L->tc_stats, 0, 32 * sizeof(unsigned long long)));
  QB_CUDA_TRY(L, L->rowbest.alloc(S * V));
  QB_CUDA_TRY(L, L->colpart.alloc(L->colpart_count()));
  QB_CUDA_TRY(L, L->colbest.alloc(S * V));
  QB_CUDA_TRY(L, L->mut_i.alloc(S * V));
  QB_CUDA_TRY(L, L->mut_j.alloc(S * V));
  QB_CUDA_TRY(L, L->mark.alloc(S * V));
  QB_CUDA_TRY(L, L->partner.alloc(S * V));
  QB_CUDA_TRY(L, L->mean.alloc(C * 4));
  QB_CUDA_TRY(L, L->corr_src.alloc(S * Lc));
  QB_CUDA_TRY(L, L->corr_tgt.alloc(S * Lc));
  QB_CUDA_TRY(L, L->ma.alloc(S * Lc));
  QB_CUDA_TRY(L, L->mb.alloc(S * Lc));
  QB_CUDA_TRY(L, L->adj.alloc(S * Lc * W));
  QB_CUDA_TRY(L, L->adjp.alloc(S * Lc * W));
  QB_CUDA_TRY(L, L->deg.alloc(S * Lc));
  QB_CUDA_TRY(L, L->kcore.alloc(S * (Lc + 2)));
  QB_CUDA_TRY(L, L->korder.alloc(S * (Lc + 2)));
  QB_CUDA_TRY(L, L->rank_of.alloc(S * (Lc + 2)));
  QB_CUDA_TRY(L, L->by_rank.alloc(S * (Lc + 2)));
  QB_CUDA_TRY(L, L->kbin.alloc(S * (Lc + 2)));
  QB_CUDA_TRY(L, L->clique.alloc(S * Lc));
  QB_CUDA_TRY(L, L->final_inl.alloc(S * Lc));
  QB_CUDA_TRY(L, L->rot_mask.alloc(S * Lc));
  QB_CUDA_TRY(L, L->trans_mask.alloc(S * Lc));
  QB_CUDA_TRY(L, L->d_solve.alloc(S));
  QB_CUDA_TRY(L, L->h_solve.alloc(S));
  QB_CUDA_TRY(L, L->d_front.alloc(C));
  QB_CUDA_TRY(L, L->h_front.alloc(C));
  // workspaces of the pairs whose graph or clique outgrows the shared-memory layouts (clique.cu, pose.cu); only wide handles have them
  if (Lc > (size_t)kKcoreSmemVerts) {
    QB_CUDA_TRY(L, L->kcore_ws.alloc(S * kcore_ws_bytes((int)Lc)));
    QB_CUDA_TRY(L, L->chain_ws.alloc(S * kCliqueWarps * Lc));
  }
  if (Lc > (size_t)kPoseSmemClique) QB_CUDA_TRY(L, L->pose_ws.alloc(S * pose_ws_bytes((int)Lc)));
  QB_CUDA_TRY(L, L->d_results.alloc(S));
  QB_CUDA_TRY(L, cudaMemset(L->d_results, 0, S * sizeof(qb200_result)));
  QB_CUDA_TRY(L, L->h_results.alloc(S));
  L->ctr_ints = carve_counters(nullptr, S, &L->ctr);
  QB_CUDA_TRY(L, L->ctr_block.alloc(L->ctr_ints));
  QB_CUDA_TRY(L, L->hctr_block.alloc(L->ctr_ints));
  carve_counters(L->ctr_block, S, &L->ctr);
  carve_counters(L->hctr_block, S, &L->hctr);
  for (Event& e : L->ev) QB_CUDA_TRY(L, e.create());
  for (Event& e : L->kev) QB_CUDA_TRY(L, e.create());
  QB_CUDA_TRY(L, L->ev_cache_in.create(cudaEventDisableTiming));
  QB_CUDA_TRY(L, L->ev_cache_out.create(cudaEventDisableTiming));
  QB_CUDA_TRY(L, cudaStreamSynchronize(L->stream));
  *out = std::move(L);
  return QB200_OK;
}

// stage and kernel times of a batch call start from zero
void reset_timers(qb200_handle* h) {
  memset(h->stage_ms, 0, sizeof(h->stage_ms));
  memset(h->kernel_ms, 0, sizeof(h->kernel_ms));
  memset(h->kernel_calls, 0, sizeof(h->kernel_calls));
}

}  // namespace

namespace qb {
cudaError_t ensure_dyn_smem(int device, const void* kernel, size_t bytes) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, size_t> current;
  std::lock_guard<std::mutex> lock(mu);
  size_t& cur = current[std::make_pair(kernel, device)];
  if (bytes > cur) {
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return e;
    cur = bytes;
  }
  return cudaSuccess;
}

int wave_reset(Lane* L, int n_clouds) {
  const int n = (int)L->ctr_ints;
  wave_init_kernel<<<(n + 255) / 256, 256, 0, L->stream>>>(L->ctr_block, n, L->ctr.bbox, n_clouds);
  L->launches++;
  L->waves++;
  QB_CUDA_TRY(L, cudaGetLastError());
  return QB200_OK;
}

bool params_ok(const qb200_params* p, bool solver) {
  if (!p) return false;
  if (!(p->voxel_size > 0) || !(p->normal_radius > 0) || !(p->fpfh_radius > 0)) return false;
  if (p->normal_radius > p->fpfh_radius) return false;  // FPFHManager::setFeaturePair throws here, fpfh_manager.hpp:99-102
  if (p->tuple_trials_per_corr < 0) return false;
  if (!solver) return true;
  if (!(p->noise_bound > 0) || !(p->cbar2 > 0) || !(p->cote_noise_bound > 0)) return false;
  if (p->cote_mode != QB200_COTE_MEDIAN && p->cote_mode != QB200_COTE_WEIGHTED_MEAN) return false;  // quatro.hpp:911
  if (p->inlier_selection_mode < 0 || p->inlier_selection_mode > 3 || p->max_clique_node_limit < 0) return false;
  if (p->rotation_max_iterations < 0) return false;
  return true;
}

// default cell = (1 + 2^-9) fpfh_radius: with the cell a hair larger than the radius, |x' - x| < r keeps the cell index of a
// neighbour within +-1 even after the float rounding of x / cell, so the walk covers 27 cells instead of 125
float lattice_cell(const qb200_params& p) { return p.grid_cell > 0 ? p.grid_cell : p.fpfh_radius * 1.001953125f; }

// The lattice fields of an entry of qb200_describe_points_each, the only ones it reads: finite positive radii, normal_radius <=
// fpfh_radius (fpfh_manager.hpp:99-102), a finite grid_cell and a finite resolved cell
bool lattice_ok(const qb200_params& p) {
  return std::isfinite(p.normal_radius) && std::isfinite(p.fpfh_radius) && p.normal_radius > 0 && p.fpfh_radius > 0 &&
         p.normal_radius <= p.fpfh_radius && std::isfinite(p.grid_cell) && std::isfinite(lattice_cell(p));
}

CloudFront front_entry(const qb200_params& p, bool lattice_only) {
  CloudFront e;
  memset(&e, 0, sizeof(e));
  if (!lattice_only) front_voxel(&e, p.voxel_size, p.skip_flagged);
  front_lattice(&e, p.normal_radius, p.fpfh_radius, lattice_cell(p));
  return e;
}

// p with its rotation noise bound resolved.  The reference latches 2*noise_bound of the FIRST registration into a function-local
// static (quatro.hpp:469-470 after :851); here the latch is a per-handle field, overridable via params.  Every lane gets the
// resolved value, so a pair's GNC bound never depends on the wave / lane it lands on.
qb200_params resolve_params(qb200_handle* h, const qb200_params& p) {
  qb200_params r = p;
  if (!(r.rot_noise_bound > 0)) {
    if (h->rot_noise_bound_latched <= 0) h->rot_noise_bound_latched = 2.0 * p.noise_bound;
    r.rot_noise_bound = h->rot_noise_bound_latched;
  }
  return r;
}

// what qb200_get_last_* read back after a single-pair registration or solve
void set_last(qb200_handle* h, const qb200_result& r) {
  h->last_n_corr = r.n_corr;
  h->last_n_clique = r.clique_size;
  h->last_n_final = r.n_final_inliers;
}

void stamp_last(qb200_handle* h, std::initializer_list<LastList> lists) {
  for (const LastList l : lists) h->last_wave[l] = h->lane[0]->waves;
}

bool last_is_live(qb200_handle* h, LastList list) {
  if (h->lane[0]->waves == h->last_wave[list]) return true;
  h->fail(__FILE__, __LINE__, "a later call reused the buffers of the most recent single-pair call: fetch its lists right after it");
  return false;
}

// a match wave's entry: the matcher fields of p (K7's tuple test), nothing of the solver
PairSolve match_entry(const qb200_params& p) {
  PairSolve e;
  memset(&e, 0, sizeof(e));
  match_fields(&e, p);
  return e;
}

// a graph wave's entry: the clique fields of p as qb200_max_clique_ex takes them, nothing of the graph or pose stages
PairSolve clique_entry(const qb200_params& p) {
  PairSolve e;
  memset(&e, 0, sizeof(e));
  e.kcore_thr = p.kcore_heuristic_threshold;
  e.node_limit = p.max_clique_node_limit > 0 ? p.max_clique_node_limit : (long long)QB200_DEFAULT_CLIQUE_NODE_LIMIT;
  e.mode = p.inlier_selection_mode;
  return e;
}

// a pose wave's entry: the pose fields of p (rotation noise bound resolved) as qb200_solve_pose reads them; nothing of the matcher,
// graph or clique stages
PairSolve pose_entry(const qb200_params& p) {
  PairSolve e;
  memset(&e, 0, sizeof(e));
  e.pp = pose_params(p);
  return e;
}

// a TIM graph wave's entry: K8's beta from noise_bound and cbar2, and a mode that builds the graph (K8 and degree_kernel skip
// QB200_INLIER_NONE), as qb200_build_graph sets them; nothing of the matcher, clique or pose stages
PairSolve graph_entry(const qb200_params& p) {
  PairSolve e;
  memset(&e, 0, sizeof(e));
  e.gc = graph_const(p.noise_bound, p.cbar2);
  e.mode = QB200_PMC_HEU;
  return e;
}

PairSolve solve_entry(const qb200_params& p) {
  PairSolve e;
  memset(&e, 0, sizeof(e));
  e.gc = graph_const(p.noise_bound, p.cbar2);
  e.pp = pose_params(p);
  e.kcore_thr = p.kcore_heuristic_threshold;
  e.node_limit = p.max_clique_node_limit > 0 ? p.max_clique_node_limit : (long long)QB200_DEFAULT_CLIQUE_NODE_LIMIT;
  e.mode = p.inlier_selection_mode;
  match_fields(&e, p);
  return e;
}

int upload_solve(Lane* L, int n) {
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->d_solve, L->h_solve, (size_t)n * sizeof(PairSolve), cudaMemcpyHostToDevice, L->stream));
  return QB200_OK;
}

// graph -> clique -> pose for pairs [0, n) whose matched points / n_corr are already on the device and whose solver entries are in
// L->h_solve and (upload_solve) L->d_solve.  The host reads the wave's modes from the table and launches only what they need: no K8 / K9
// when every pair is in QB200_INLIER_NONE, no exact search without a PMC_EXACT pair, no iota clique without a QB200_INLIER_NONE pair.
int run_solver(Lane* L, int n_pairs, int have_frontend) {
  bool graph = false, none = false, exact = false;
  for (int s = 0; s < n_pairs; ++s) {
    const int m = L->h_solve[s].mode;
    graph |= m != QB200_INLIER_NONE;
    none |= m == QB200_INLIER_NONE;
    exact |= m == QB200_PMC_EXACT;
  }
  int rc;
  if (graph) {
    if ((rc = launch_graph(L, n_pairs))) return rc;
    if (L->ev[5]) cudaEventRecord(L->ev[5], L->stream);
    if ((rc = launch_clique(L, n_pairs, exact))) return rc;
  }
  // the reference leaves max_clique_ empty in INLIER_NONE (quatro.hpp:782); TEASER++ semantics: all measurements
  if (none && (rc = launch_iota_clique(L, n_pairs))) return rc;
  if (L->ev[6]) cudaEventRecord(L->ev[6], L->stream);
  if ((rc = launch_fill_counters(L, n_pairs, have_frontend))) return rc;
  if ((rc = launch_pose(L, n_pairs))) return rc;
  if ((rc = launch_finalize_status(L, n_pairs))) return rc;
  return QB200_OK;
}

// Stage the raw clouds [0, ncl) of a wave whose caller pointers and point counts are in L->h_cloud_ptr / h_cloud_n, then copy the
// cloud tables; every copy goes on stream cs.  Device clouds are read in place.  Host clouds go to raw_stage; clouds that lie back
// to back in the caller's memory (one big pinned buffer is the usual case) cross PCIe as one copy: far fewer DMA descriptors than
// one per cloud.
int stage_raw(Lane* L, int ncl, qb200_mem_kind kind, cudaStream_t cs) {
  int total = 0, run_dst = 0, run_n = 0, rc;
  const float4* run_src = nullptr;
  auto flush_run = [&]() -> int {
    if (run_n > 0)
      QB_CUDA_TRY(L, cudaMemcpyAsync(L->raw_stage + run_dst, run_src, (size_t)run_n * sizeof(float4), cudaMemcpyHostToDevice, cs));
    run_n = 0;
    return QB200_OK;
  };
  for (int c = 0; c < ncl; ++c) {
    const float4* src = L->h_cloud_ptr[c];
    const int n = L->h_cloud_n[c];
    L->h_raw_off[c] = total;
    if (kind == QB200_MEM_HOST) {
      L->h_cloud_ptr[c] = L->raw_stage + total;
      if (n > 0) {
        if (run_n > 0 && src == run_src + run_n && run_n < (1 << 26)) {
          run_n += n;
        } else {
          if ((rc = flush_run())) return rc;
          run_src = src; run_dst = total; run_n = n;
        }
      }
    }
    total += n;
  }
  if ((rc = flush_run())) return rc;
  L->h_raw_off[ncl] = total;
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->d_cloud_ptr, L->h_cloud_ptr, (size_t)ncl * sizeof(float4*), cudaMemcpyHostToDevice, cs));
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->d_cloud_n, L->h_cloud_n, (size_t)ncl * sizeof(int), cudaMemcpyHostToDevice, cs));
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->d_raw_off, L->h_raw_off, (size_t)(ncl + 1) * sizeof(int), cudaMemcpyHostToDevice, cs));
  return QB200_OK;
}

// A descriptor wave's clouds of other lengths than 33 (h_feat[0, ncl) entries whose dim is not kDescDim) in the lane's dd_buf: each
// cloud's dimension-major rows at FeatureSrc::out, ld = n rounded up to 4 points (every row starts 16-byte aligned for nn_dim_kernel's
// cp.async), then, with host rows, those rows packed behind them from *stage on.  The buffer is allocated on the first wave that has
// such a cloud and grows to the largest wave so far; the lane's previous wave has been collected, so the old buffer is idle.
int layout_other_dims(Lane* L, int ncl, bool host, float** stage) {
  size_t major = 0, rows = 0;
  for (int c = 0; c < ncl; ++c) {
    FeatureSrc& f = L->h_feat[c];
    if (!f.desc || f.dim == kDescDim) continue;
    f.ld = (f.n + 3) & ~3;
    major += (size_t)f.dim * f.ld;
    rows += (size_t)f.dim * f.n;
  }
  const size_t need = major + (host ? rows : 0);
  if (need > L->dd_cap) {
    L->dd_cap = 0;
    QB_CUDA_TRY(L, L->dd_buf.alloc(need));
    L->dd_cap = need;
  }
  size_t off = 0;
  for (int c = 0; c < ncl; ++c) {
    FeatureSrc& f = L->h_feat[c];
    if (!f.desc || f.dim == kDescDim) continue;
    f.out = L->dd_buf + off;
    off += (size_t)f.dim * f.ld;
  }
  *stage = need > 0 ? L->dd_buf + major : nullptr;
  return QB200_OK;
}

int stage_features(Lane* L, int ncl, qb200_mem_kind kind, cudaStream_t cs) {
  float* other = nullptr;
  if (int rc = layout_other_dims(L, ncl, kind == QB200_MEM_HOST, &other)) return rc;
  if (kind == QB200_MEM_HOST) {
    // Host clouds are packed into areas a feature wave leaves idle: keypoints into normals, FPFH-33 rows into spfh (33 floats each),
    // rows of other lengths behind the dimension-major rows of dd_buf (dim floats each).  A run of clouds that lie back to back in
    // the caller's memory crosses PCIe as one copy per array, as raw scans do (stage_raw); rows with a stride past their descriptor
    // cross by one 2-D copy per cloud that leaves the rest of each row behind.
    const char* run_src[2] = {nullptr, nullptr};
    char* run_dst[2] = {nullptr, nullptr};
    size_t run_bytes[2] = {0, 0};
    auto flush_run = [&](int k) -> int {
      if (run_bytes[k] > 0) QB_CUDA_TRY(L, cudaMemcpyAsync(run_dst[k], run_src[k], run_bytes[k], cudaMemcpyHostToDevice, cs));
      run_bytes[k] = 0;
      return QB200_OK;
    };
    auto add = [&](int k, const void* src, void* dst, size_t bytes) -> int {
      const char* s = static_cast<const char*>(src);
      char* d = static_cast<char*>(dst);
      if (bytes == 0) return QB200_OK;
      if (run_bytes[k] > 0 && s == run_src[k] + run_bytes[k] && d == run_dst[k] + run_bytes[k]) {
        run_bytes[k] += bytes;
        return QB200_OK;
      }
      if (int rc = flush_run(k)) return rc;
      run_src[k] = s; run_dst[k] = d; run_bytes[k] = bytes;
      return QB200_OK;
    };
    size_t off = 0;
    for (int c = 0; c < ncl; ++c) {
      FeatureSrc& f = L->h_feat[c];
      float4* pts = L->normals.get() + off;
      float* desc = f.dim == kDescDim ? L->spfh + off * kDescDim : other;
      if (f.pts) {
        if (int rc = add(0, f.pts, pts, (size_t)f.n * sizeof(float4))) return rc;
        f.pts = pts;
      }
      if (f.desc) {  // (a describe-points wave stages keypoints only)
        const size_t row = (size_t)f.dim * sizeof(float);
        if (f.stride == f.dim) {
          if (int rc = add(1, f.desc, desc, f.n * row)) return rc;
        } else if (f.n > 0) {
          QB_CUDA_TRY(L, cudaMemcpy2DAsync(desc, row, f.desc, (size_t)f.stride * sizeof(float), row, f.n, cudaMemcpyHostToDevice, cs));
        }
        f.desc = desc;
        f.stride = f.dim;
        if (f.dim != kDescDim) other += (size_t)f.dim * f.n;
      }
      off += f.n;
    }
    for (int k = 0; k < 2; ++k)
      if (int rc = flush_run(k)) return rc;
  }
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->d_feat, L->h_feat, (size_t)ncl * sizeof(FeatureSrc), cudaMemcpyHostToDevice, cs));
  return QB200_OK;
}

}  // namespace qb

namespace {

// ---- scan cache ---------------------------------------------------------------------------------------------------------
// FPFHManager keeps the last target's descriptors and reuses them as the next source (odometry mode, fpfh_manager.hpp:74-77,
// 111-118); a loop-closure sweep matches one scan against many.  The cache keeps voxel points, normals and FPFH-33 of a scan
// resident on the device so that the front end (voxel + normals + FPFH, ~45 % of a wave) runs once per SCAN, not once per pair.

// clouds [0, n_clouds) of lane L's wave to (to_cache = 1) or from their cache slots L->h_slot_of_cloud[]
int cache_copy(qb200_handle* h, Lane* L, int to_cache, int n_clouds) {
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->d_slot_of_cloud, L->h_slot_of_cloud, (size_t)n_clouds * sizeof(int), cudaMemcpyHostToDevice, L->stream));
  const dim3 g((L->V + 255) / 256, 43, n_clouds);
  cache_copy_kernel<<<g, 256, 0, L->stream>>>(to_cache, L->d_slot_of_cloud, L->V, L->vox_pts, L->normals, L->desc_t, L->ctr.n_vox, L->ctr.cloud_status,
                                              h->c_vox, h->c_nrm, h->c_desc, h->c_n, h->c_status);
  L->launches++;
  QB_CUDA_TRY(L, cudaGetLastError());
  return QB200_OK;
}

bool share_a_slot(const std::vector<int>& a, const std::vector<int>& b) {
  for (size_t i = 0, j = 0; i < a.size() && j < b.size();) {
    if (a[i] == b[j]) return true;
    if (a[i] < b[j]) ++i; else ++j;
  }
  return false;
}

// The slots of the wave about to copy clouds [0, ncl) of lane L to (write) or from its slot table L->h_slot_of_cloud go to
// L->pend_slots, and L's stream waits for the conflicting cache copies of the waves in flight on the other lanes: a write for their
// copy-ins and copy-outs of its slots (WAR, WAW), a read for their copy-outs (RAW).  Every wave that was enqueued earlier has been
// collected or is the one wave in flight on its lane, and a lane's waves run in order, so these device-side waits put every access to
// a slot in enqueue order.  A write names a slot more than once only when scans of one call do: the last one wins, as it would in a
// later wave, and the others are not copied.
int cache_waits(qb200_handle* h, Lane* L, int ncl, bool write) {
  std::vector<std::pair<int, int>> by_slot(ncl);
  for (int c = 0; c < ncl; ++c) by_slot[c] = std::make_pair(L->h_slot_of_cloud[c], c);
  std::sort(by_slot.begin(), by_slot.end());
  L->pend_slots.clear();
  L->pend_writes = write;
  for (int i = 0; i < ncl; ++i) {
    if (i + 1 == ncl || by_slot[i + 1].first != by_slot[i].first) L->pend_slots.push_back(by_slot[i].first);
    else if (write) L->h_slot_of_cloud[by_slot[i].second] = -1;
  }
  for (const std::unique_ptr<Lane>& Y : h->lane) {
    if (!Y || Y.get() == L || Y->pend_np == 0 || !(write || Y->pend_writes) || !share_a_slot(L->pend_slots, Y->pend_slots)) continue;
    QB_CUDA_TRY(L, cudaStreamWaitEvent(L->stream, Y->pend_writes ? Y->ev_cache_out : Y->ev_cache_in, 0));
  }
  return QB200_OK;
}

// ---- batch calls ----------------------------------------------------------------------------------------------------------
// The params entries of a call: one for the whole batch, one per input whose front-end fields (voxel_size .. seed) are bit-identical
// in every entry, or one per input that may differ in any field (the _mixed forms and the calls that read no shared front end)
enum class Entries { One, Each, Mixed };

// One batch call as its entry point received it (handle.cuh lists the valid source and sink pairs): n inputs of its source, of
// which only the array of that source is read, in `kind` memory (cached pairs: host), and the outputs of its sink.
struct BatchCall {
  Source src = Source::RawPairs;
  Sink sink = Sink::Solve;
  int n = 0;
  qb200_mem_kind kind = QB200_MEM_HOST;
  const qb200_params* caller = nullptr;
  Entries entries = Entries::One;
  // the inputs, one array per source
  const qb200_pair* pairs = nullptr;           // RawPairs
  const qb200_slot_pair* slots = nullptr;      // CachedPairs
  const qb200_feature_pair* feats = nullptr;   // FeaturePairs: keypoints and FPFH-33 rows, front-end fields of the entries ignored
  const qb200_descriptor_pair* descs = nullptr;  // DescriptorPairs: keypoints and descriptor rows of any length, the same
  const qb200_corr_set* sets = nullptr;        // CorrSets
  const qb200_graph* graphs = nullptr;         // Graphs
  const qb200_inlier_set* inlier_sets = nullptr;  // InlierSets
  const qb200_align_set* align_sets = nullptr;    // AlignSets
  const float* const* scans = nullptr;         // RawScans, KeypointClouds (described with the lattice fields of their entries alone):
  const int32_t* n_points = nullptr;           // scan i has n_points[i] points
  // the outputs, one set per sink
  qb200_result* results = nullptr;             // Solve, Match, Clique, Graph, Pose: one record per input
  const qb200_pair_lists* lists = nullptr;     // ... and the per-pair lists, nullptr = records only
  const int32_t* slot_ids = nullptr;           // CacheSlots: scan i goes to slot slot_ids[i]
  const qb200_feature_out* out = nullptr;      // Export: the caller's feature arrays
  const qb200_graph_out* graph_out = nullptr;  // Graph: the caller's adjacency, degree and edge arrays
  const qb200_align_out* align_out = nullptr;  // AlignOut: the caller's aligned clouds, matched points, good matches, counts and status
  // set by enqueue_call.  The params the pairs are solved with, rotation noise bounds resolved (Solve, Pose), laid out like `caller`.
  const qb200_params* params = nullptr;
  // host inputs of a multi-wave batch crossing PCIe: the batch's copy stream, or nullptr = copy on the lane's own stream.  Copies
  // queued on several streams share the PCIe link, so every wave's scans would arrive late; on one stream they arrive wave after
  // wave and the first waves compute while the later ones are still crossing.
  cudaStream_t copy_stream = nullptr;
  bool each() const { return entries != Entries::One; }
};

// The facts of each source that the checks and the waves read, written down once

// clouds one input takes in the wave's 2S cloud buffers: two per pair, one per scan, none per set (its matched points go to ma / mb,
// an inlier set's ids to clique), graph (its adjacency goes to adj) or align set (read through its own table entry)
int clouds_per_input(Source s) {
  switch (s) {
    case Source::RawPairs: case Source::CachedPairs: case Source::FeaturePairs: case Source::DescriptorPairs: return 2;
    case Source::RawScans: case Source::KeypointClouds: return 1;
    case Source::CorrSets: case Source::Graphs: case Source::InlierSets: case Source::AlignSets: return 0;
  }
  return 0;
}

// the wave matches pairs of clouds (K6..K7) before its records: the solver's counters come from a front end (have_frontend)
bool is_pairs(Source s) { return clouds_per_input(s) == 2; }

// Host-kind inputs of the source cross PCIe in a staged front (stage_raw, stage_features, front_align): a multi-wave batch sends them
// on the shared copy stream and opens with a quarter wave.  Cached pairs, correspondence sets, graphs and inlier sets do neither.
bool crosses_pcie(Source s) {
  switch (s) {
    case Source::RawPairs: case Source::FeaturePairs: case Source::DescriptorPairs: case Source::RawScans: case Source::KeypointClouds:
    case Source::AlignSets:
      return true;
    case Source::CachedPairs: case Source::CorrSets: case Source::Graphs: case Source::InlierSets: return false;
  }
  return false;
}

// The wave uploads the front-end table d_front: K1..K5 (K2..K5 for keypoint clouds) read each cloud's entry.  The solver table
// d_solve is uploaded by the waves with records (Solve, Match, Clique, Graph, Pose), i.e. of pairs, sets and graphs.
bool runs_front_end(Source s) {
  switch (s) {
    case Source::RawPairs: case Source::RawScans: case Source::KeypointClouds: return true;
    case Source::CachedPairs: case Source::FeaturePairs: case Source::DescriptorPairs: case Source::CorrSets: case Source::Graphs:
    case Source::InlierSets: case Source::AlignSets:
      return false;
  }
  return false;
}

bool has_records(Sink k) { return k == Sink::Solve || k == Sink::Match || k == Sink::Clique || k == Sink::Graph || k == Sink::Pose; }

// The stage-time slots of qb200_get_stage_ms a wave reports (bit i = slot i, the time between events i and i + 1 of Lane::ev).
// A wave reports the stages its source runs: cached pairs their copy-in in the fpfh slot, caller features their copy and import in
// h2d.  Cached pairs and sets report no d2h slot; waves without records report none (they register nothing).  A match wave reports
// the slots up to match as its source has them, and d2h.  A graph wave reports h2d, its import in the graph slot, clique and d2h; a
// TIM graph wave h2d, graph (K8 and its outputs) and d2h; a pose wave h2d (with the id import), pose and d2h.
unsigned stage_slots(Source s, Sink k) {
  enum : unsigned { kH2d = 1, kVoxel = 2, kFpfh = 4, kMatch = 8, kGraph = 16, kClique = 32, kPose = 64, kD2h = 128 };
  constexpr unsigned kSolver = kGraph | kClique | kPose;
  if (!has_records(k)) return 0u;
  if (k == Sink::Clique) return kH2d | kGraph | kClique | kD2h;
  if (k == Sink::Graph) return kH2d | kGraph | kD2h;
  if (k == Sink::Pose) return kH2d | kPose | kD2h;
  unsigned m = 0;
  switch (s) {
    case Source::RawPairs: m = kH2d | kVoxel | kFpfh | kMatch | kSolver | kD2h; break;
    case Source::FeaturePairs: case Source::DescriptorPairs: m = kH2d | kMatch | kSolver | kD2h; break;
    case Source::CachedPairs: m = kFpfh | kMatch | kSolver; break;
    case Source::CorrSets: m = kSolver; break;
    case Source::RawScans: case Source::KeypointClouds: case Source::Graphs: case Source::InlierSets: case Source::AlignSets: break;
  }
  return k == Sink::Match ? (m & (kH2d | kVoxel | kFpfh | kMatch)) | kD2h : m;
}

// Host-kind lists: the lane's pinned staging block holds cap entries of every list for each slot.  It only grows, and a failed
// allocation leaves the lane as it was.  The lane's previous wave has been collected, so the old block is not in use.
int ensure_list_stage(Lane* L, const qb200_pair_lists& l) {
  if (L->lst_cap >= l.cap_per_pair) return QB200_OK;
  ListDst d;
  PinnedMem<unsigned char> m;
  QB_CUDA_TRY(L, m.alloc(ListDst::carve(nullptr, L->S, l.cap_per_pair, l, &d)));
  L->lst_stage = std::move(m);
  L->lst_cap = l.cap_per_pair;
  return QB200_OK;
}

// Enqueue the list pack of the wave on lane L (pairs [w0, w0 + np)): straight into the caller's device arrays, or into the lane's
// staging block that wave_collect hands on to the caller's host arrays.  It marks clipped records, so it precedes their D2H.
int submit_lists(Lane* L, const qb200_pair_lists& l, int w0, int np) {
  int rc;
  ListDst d = ListDst::caller(l, w0);
  if (l.kind == QB200_MEM_HOST) {
    if ((rc = ensure_list_stage(L, l))) return rc;
    ListDst::carve(L->lst_stage, L->S, L->lst_cap, l, &d);
  }
  return launch_pack_lists(L, np, d);
}

// the live prefix of every pair's lists from the lane's staging block to the caller's host arrays (h_results holds the records)
void deliver_lists(Lane* L, const qb200_pair_lists& l, int w0, int np) {
  ListDst st, to = ListDst::caller(l, w0);
  ListDst::carve(L->lst_stage, L->S, L->lst_cap, l, &st);
  auto put = [](auto* dst, const auto* src, size_t d0, size_t s0, int m) {
    if (dst && m > 0) memcpy(dst + d0, src + s0, (size_t)m * sizeof(*dst));
  };
  for (int s = 0; s < np; ++s) {
    const qb200_result& r = L->h_results[s];
    if (r.status == QB200_CAPACITY_EXCEEDED) continue;
    const int mc = list_entries(r.n_corr, L->Lc, to.cap), mq = list_entries(r.clique_size, L->Lc, to.cap);
    const size_t d0 = (size_t)s * to.stride, s0 = (size_t)s * st.stride;
    put(to.corr, st.corr, d0, s0, mc);
    put(to.sm, st.sm, d0, s0, mc);
    put(to.tm, st.tm, d0, s0, mc);
    put(to.clique, st.clique, d0, s0, mq);
    put(to.rm, st.rm, d0, s0, mq);
    put(to.tmask, st.tmask, d0, s0, mq);
    put(to.fin, st.fin, d0, s0, list_entries(r.n_final_inliers, L->Lc, to.cap));
  }
}

// The lane's staging block as a describe wave's destination (base == nullptr: only its size): counts and status of the 2S clouds, and
// in host kind min(cap_per_scan, V) entries per cloud of every array the caller asked for
size_t export_stage(const Lane* L, const qb200_feature_out& o, unsigned char* base, ExportDst* d) {
  qb200_feature_out staged = o;
  if (o.kind == QB200_MEM_DEVICE) staged.vox4 = staged.normals4 = staged.desc33 = nullptr;  // counts and status only
  return ExportDst::carve(base, 2 * L->S, o.cap_per_scan < L->V ? o.cap_per_scan : L->V, staged, d);
}

// Enqueue the export of a describe wave (scans [w0, w0 + ncl) of lane L): its counts and status into the lane's staging block, its
// entries straight into the caller's device arrays or into that block, from where wave_collect hands them on (deliver_export).  The
// lane's previous wave has been collected, so a block that must grow is not in use.  voxels: a voxelize wave, whose export reports
// every cloud as qb200_voxelize does (ExportSrc::n_kept) and whose pass-through clouds get their kept points from passthrough_kernel:
// straight into the caller's device vox4, or into their raw_stage regions, which no copy overwrites before wave_collect (the lane's next
// wave stages its scans only after it).
int submit_export(Lane* L, const qb200_feature_out& o, int w0, int ncl, bool voxels) {
  ExportDst d;
  const size_t bytes = export_stage(L, o, nullptr, &d);
  if (L->exp_bytes < bytes) {
    PinnedMem<unsigned char> m;
    QB_CUDA_TRY(L, m.alloc(bytes));
    L->exp_stage = std::move(m);
    L->exp_bytes = bytes;
  }
  export_stage(L, o, L->exp_stage, &d);
  const ExportDst to = ExportDst::caller(o, w0);
  if (o.kind == QB200_MEM_DEVICE) {
    d.vox = to.vox; d.nrm = to.nrm; d.desc = to.desc; d.stride = to.stride; d.cap = to.cap;
  }
  const ExportSrc s{L->vox_pts, L->normals, L->desc_t, L->ctr.n_vox, L->ctr.cloud_status, voxels ? L->ctr.n_valid : nullptr};
  if (int rc = launch_feature_export(L, ncl, s, d, L->V)) return rc;
  if (!voxels || !o.vox4) return QB200_OK;
  return o.kind == QB200_MEM_DEVICE ? launch_passthrough(L, ncl, to.vox, to.stride, to.cap) : launch_passthrough(L, ncl, nullptr, 0, 0);
}

// a collected describe wave's counts and status, and in host kind its entries, from the lane's staging block to the caller; a
// voxelize wave's pass-through clouds (voxels) from their raw_stage regions
int deliver_export(Lane* L, const qb200_feature_out& o, int w0, int ncl, bool voxels) {
  ExportDst st;
  export_stage(L, o, L->exp_stage, &st);
  memcpy(o.counts + w0, st.counts, (size_t)ncl * sizeof(int));
  memcpy(o.status + w0, st.status, (size_t)ncl * sizeof(int));
  if (o.kind == QB200_MEM_DEVICE) return QB200_OK;
  const ExportDst to = ExportDst::caller(o, w0);
  bool copied = false;
  for (int c = 0; c < ncl; ++c) {
    const size_t d0 = (size_t)c * to.stride, s0 = (size_t)c * st.stride;
    if (voxels && st.status[c] == QB200_ERR_VOXEL_OVERFLOW) {
      const int m = st.counts[c] < to.cap ? st.counts[c] : to.cap;
      if (to.vox && m > 0) {
        QB_CUDA_TRY(L, cudaMemcpyAsync(to.vox + d0, L->raw_stage + L->h_raw_off[c], (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost, L->stream));
        copied = true;
      }
      continue;
    }
    const int m = st.counts[c] < st.cap ? st.counts[c] : st.cap;
    if (m <= 0) continue;
    if (to.vox) memcpy(to.vox + d0, st.vox + s0, (size_t)m * sizeof(float4));
    if (to.nrm) memcpy(to.nrm + d0, st.nrm + s0, (size_t)m * sizeof(float4));
    if (to.desc) memcpy(to.desc + d0 * kDescDim, st.desc + s0 * kDescDim, (size_t)m * kDescDim * sizeof(float));
  }
  if (copied) QB_CUDA_TRY(L, cudaStreamSynchronize(L->stream));
  return QB200_OK;
}

// An output descriptor of a describe call: capacity and kinds in range, counts and status present, device arrays on the handle's
// device and aligned for the export's stores; points: no vox4 (the keypoints are the caller's own)
int check_out(qb200_handle* h, const qb200_feature_out* o, bool points) {
  const char* why = nullptr;
  if (!o) why = "the output descriptor is null";
  else if (points && o->vox4) why = "vox4 must be null: the keypoints are the caller's own";
  else if (o->cap_per_scan < 1) why = "cap_per_scan < 1";
  else if (!o->counts || !o->status) why = "the counts or status array is null";
  else if (o->kind != QB200_MEM_HOST && o->kind != QB200_MEM_DEVICE) why = "unknown memory kind of the outputs";
  else if (o->kind == QB200_MEM_DEVICE && !device_array_of(h, o->vox4, 16)) why = "device vox4 is misaligned or not memory of the handle's device";
  else if (o->kind == QB200_MEM_DEVICE && !device_array_of(h, o->normals4, 16))
    why = "device normals4 is misaligned or not memory of the handle's device";
  else if (o->kind == QB200_MEM_DEVICE && !device_array_of(h, o->desc33, 4)) why = "device desc33 is misaligned or not memory of the handle's device";
  if (!why) return QB200_OK;
  h->fail(__FILE__, __LINE__, why);
  return QB200_ERR_BAD_ARG;
}

// The output descriptor of a TIM graph call: a known kind, row and word counts that hold the rows asked for, a capacity for the edges
// asked for, and device arrays on the handle's device and aligned for the kernels' stores.  Each set's L is checked against
// rows_per_set with the set.
int check_graph_out(qb200_handle* h, const qb200_graph_out* o) {
  const char* why = nullptr;
  const bool device = o && o->kind == QB200_MEM_DEVICE;
  if (!o) why = "the output descriptor is null";
  else if (o->kind != QB200_MEM_HOST && o->kind != QB200_MEM_DEVICE) why = "unknown memory kind of the outputs";
  else if ((o->adj || o->degree) && o->rows_per_set < 0) why = "rows_per_set < 0";
  else if (o->adj && o->words_per_row < (o->rows_per_set + 31LL) / 32) why = "words_per_row < ceil(rows_per_set / 32)";
  else if (o->edges && o->cap_edges < 1) why = "cap_edges < 1";
  else if (device && !device_array_of(h, o->adj, 4)) why = "device adj is misaligned or not memory of the handle's device";
  else if (device && !device_array_of(h, o->degree, 4)) why = "device degree is misaligned or not memory of the handle's device";
  else if (device && !device_array_of(h, o->edges, 8)) why = "device edges is misaligned or not memory of the handle's device";
  if (!why) return QB200_OK;
  h->fail(__FILE__, __LINE__, why);
  return QB200_ERR_BAD_ARG;
}

// The output descriptor of an align call: a known kind, caps that are not negative and at least 1 for the arrays given, and device
// arrays on the handle's device and aligned for the kernels' stores
int check_align_out(qb200_handle* h, const qb200_align_out* o) {
  const char* why = nullptr;
  const bool device = o && o->kind == QB200_MEM_DEVICE;
  if (!o) why = "the output descriptor is null";
  else if (o->kind != QB200_MEM_HOST && o->kind != QB200_MEM_DEVICE) why = "unknown memory kind of the outputs";
  else if (o->cap_points < 0 || o->cap_corr < 0) why = "cap_points or cap_corr < 0";
  else if (o->aligned4 && o->cap_points < 1) why = "cap_points < 1 with aligned4";
  else if ((o->matched4 || o->good_ids || o->good4) && o->cap_corr < 1) why = "cap_corr < 1 with matched4, good_ids or good4";
  else if (device && !(device_array_of(h, o->aligned4, 16) && device_array_of(h, o->matched4, 16) && device_array_of(h, o->good4, 16)))
    why = "device aligned4, matched4 or good4 is misaligned (16 bytes) or not memory of the handle's device";
  else if (device && !device_array_of(h, o->good_ids, 4)) why = "device good_ids is misaligned (4 bytes) or not memory of the handle's device";
  if (!why) return QB200_OK;
  h->fail(__FILE__, __LINE__, why);
  return QB200_ERR_BAD_ARG;
}

// A list descriptor from the caller: capacity and kind in range, device arrays on the handle's device and aligned for the pack's
// vector stores; for_sets: the caller supplied the correspondences, so there are none to hand back; for_match: nothing is solved, so
// there are no clique, final inliers or masks to hand back; for_graphs: a graph has a clique and nothing else.
int check_lists(qb200_handle* h, const qb200_pair_lists* l, bool for_sets, bool for_match, bool for_graphs) {
  if (!l) return QB200_OK;
  const char* why = nullptr;
  if (l->cap_per_pair < 1 || l->cap_per_pair > h->cfg.max_corr) why = "cap_per_pair outside 1 .. max_corr";
  else if (l->kind != QB200_MEM_HOST && l->kind != QB200_MEM_DEVICE) why = "unknown memory kind of the lists";
  else if (for_graphs && (l->corr || l->src_matched4 || l->tgt_matched4 || l->final_inliers || l->rot_inlier_mask || l->trans_inlier_mask))
    why = "a graph batch has only a clique to return";
  else if (for_sets && (l->corr || l->src_matched4 || l->tgt_matched4)) why = "a correspondence-set batch has no corr / matched points to return";
  else if (for_match && (l->clique || l->final_inliers || l->rot_inlier_mask || l->trans_inlier_mask))
    why = "a match call solves nothing: it has no clique, final inliers or inlier masks to return";
  else if (l->kind == QB200_MEM_DEVICE &&
           !(device_array_of(h, l->corr, 8) && device_array_of(h, l->src_matched4, 16) && device_array_of(h, l->tgt_matched4, 16) &&
             device_array_of(h, l->clique, 1) && device_array_of(h, l->final_inliers, 1) && device_array_of(h, l->rot_inlier_mask, 1) &&
             device_array_of(h, l->trans_inlier_mask, 1)))
    why = "device list array is misaligned or not memory of the handle's device";
  if (!why) return QB200_OK;
  h->fail(__FILE__, __LINE__, why);
  return QB200_ERR_BAD_ARG;
}

// The wave's tables (the lane's previous wave has been collected: their pinned mirrors are free), copied before anything else of the
// wave: on a stream of host batches the copy engine carries the scans, and a copy queued ahead of this wave's scans only waits for
// the earlier waves' scans, which the lane waits for anyway.  An input's entries (a pair's and both of its clouds') come from its own
// params.
int fill_tables(Lane* L, const BatchCall& in, int w0, int np) {
  const bool one_cloud = clouds_per_input(in.src) == 1;
  for (int s = 0; s < np; ++s) {
    const bool own = in.each() || s == 0;
    const qb200_params& p = in.params[in.each() ? w0 + s : 0];
    if (one_cloud && in.sink == Sink::Voxels) {  // the voxel fields alone: a voxelize call reads nothing else of its entries
      memset(&L->h_front[s], 0, sizeof(CloudFront));
      front_voxel(&L->h_front[s], p.voxel_size, p.skip_flagged);
      continue;
    }
    if (one_cloud) {
      L->h_front[s] = own ? front_entry(p, in.src == Source::KeypointClouds) : L->h_front[0];
      continue;
    }
    L->h_solve[s] = !own                      ? L->h_solve[0]
                    : in.sink == Sink::Match  ? match_entry(p)
                    : in.sink == Sink::Clique ? clique_entry(p)
                    : in.sink == Sink::Graph  ? graph_entry(p)
                    : in.sink == Sink::Pose   ? pose_entry(p)
                                              : solve_entry(p);
    if (in.src == Source::RawPairs) L->h_front[2 * s] = L->h_front[2 * s + 1] = own ? front_entry(p) : L->h_front[0];
  }
  int rc;
  if (has_records(in.sink) && (rc = upload_solve(L, np))) return rc;
  if (runs_front_end(in.src) && (rc = upload_front(L, np * clouds_per_input(in.src)))) return rc;
  return QB200_OK;
}

// The H2D of the staged fronts: the wave's inputs (raw scans, or caller keypoints and rows) on the batch's copy stream or the lane's
// own, then the reset of the wave's counters, and the lane's stream waits for the copies
int stage_inputs(qb200_handle* h, Lane* L, const BatchCall& in, int ncl) {
  const cudaStream_t cs = in.copy_stream ? in.copy_stream : L->stream;
  const bool raw = in.src == Source::RawPairs || in.src == Source::RawScans;
  int rc = raw ? stage_raw(L, ncl, in.kind, cs) : stage_features(L, ncl, in.kind, cs);
  if (rc || (rc = wave_reset(L, ncl))) return rc;
  if (in.copy_stream) {
    QB_CUDA_TRY(L, cudaEventRecord(h->ev_copied, in.copy_stream));
    QB_CUDA_TRY(L, cudaStreamWaitEvent(L->stream, h->ev_copied, 0));
  }
  return QB200_OK;
}

// Raw pairs and raw scans: the H2D of host scans, K1 (voxel) and K2..K5 (normals, FPFH); a voxelize wave stops after K1
int front_raw(qb200_handle* h, Lane* L, const BatchCall& in, int w0, int np, int ncl) {
  int rc;
  cudaEventRecord(L->ev[0], L->stream);
  for (int s = 0; s < np; ++s) {
    if (in.src == Source::RawScans) {
      L->h_cloud_ptr[s] = reinterpret_cast<const float4*>(in.scans[w0 + s]);
      L->h_cloud_n[s] = in.n_points[w0 + s];
      if (in.sink == Sink::CacheSlots) L->h_slot_of_cloud[s] = in.slot_ids[w0 + s];
      continue;
    }
    const qb200_pair& pr = in.pairs[w0 + s];
    L->h_cloud_ptr[2 * s] = reinterpret_cast<const float4*>(pr.src);
    L->h_cloud_ptr[2 * s + 1] = reinterpret_cast<const float4*>(pr.tgt);
    L->h_cloud_n[2 * s] = pr.n_src;
    L->h_cloud_n[2 * s + 1] = pr.n_tgt;
  }
  if ((rc = stage_inputs(h, L, in, ncl))) return rc;
  cudaEventRecord(L->ev[1], L->stream);
  if ((rc = launch_voxel(L, ncl))) return rc;
  cudaEventRecord(L->ev[2], L->stream);
  if (in.sink != Sink::Voxels && (rc = launch_fpfh(L, ncl))) return rc;
  cudaEventRecord(L->ev[3], L->stream);
  return QB200_OK;
}

// Feature pairs, descriptor pairs and keypoint clouds: the caller's keypoints (and a pair's descriptor rows) imported as they are;
// keypoint clouds, which come without descriptors, are then described by K2..K5.  A descriptor pair of 33 floats is imported into
// desc_t like a feature pair (whatever its stride); one of another length into dd_buf (stage_features places it).
int front_features(qb200_handle* h, Lane* L, const BatchCall& in, int w0, int np, int ncl) {
  int rc;
  cudaEventRecord(L->ev[0], L->stream);
  for (int s = 0; s < np; ++s) {
    if (in.src == Source::KeypointClouds) {
      L->h_feat[s] = fpfh_src(L, s, in.scans[w0 + s], nullptr, in.n_points[w0 + s]);
      continue;
    }
    if (in.src == Source::DescriptorPairs) {
      const qb200_descriptor_pair& d = in.descs[w0 + s];
      for (int side = 0; side < 2; ++side) {
        const int c = 2 * s + side;
        FeatureSrc& f = L->h_feat[c];
        f = fpfh_src(L, c, side ? d.tgt : d.src, side ? d.tgt_desc : d.src_desc, side ? d.n_tgt : d.n_src);
        f.stride = d.stride;
        if (d.dim != kDescDim) {  // dd_buf's: stage_features places it
          f.out = nullptr;
          f.dim = d.dim;
          f.ld = 0;
        }
      }
      continue;
    }
    const qb200_feature_pair& f = in.feats[w0 + s];
    L->h_feat[2 * s] = fpfh_src(L, 2 * s, f.src, f.src_desc, f.n_src);
    L->h_feat[2 * s + 1] = fpfh_src(L, 2 * s + 1, f.tgt, f.tgt_desc, f.n_tgt);
  }
  if ((rc = stage_inputs(h, L, in, ncl))) return rc;
  if ((rc = launch_feature_import(L, ncl))) return rc;
  for (int i = 1; i <= 2; ++i) cudaEventRecord(L->ev[i], L->stream);  // no voxel stage: slot 1 is not reported
  if (in.src == Source::KeypointClouds && (rc = launch_fpfh(L, ncl))) return rc;
  cudaEventRecord(L->ev[3], L->stream);  // no FPFH stage in a feature wave: slot 2 is not reported either
  return QB200_OK;
}

// Cached pairs: both clouds of every pair copied out of their cache slots
int front_cached(qb200_handle* h, Lane* L, const BatchCall& in, int w0, int np, int ncl) {
  int rc;
  for (int s = 0; s < np; ++s) {
    L->h_slot_of_cloud[2 * s] = in.slots[w0 + s].src_slot;
    L->h_slot_of_cloud[2 * s + 1] = in.slots[w0 + s].tgt_slot;
  }
  if ((rc = wave_reset(L, ncl))) return rc;
  if ((rc = cache_waits(h, L, ncl, false))) return rc;
  cudaEventRecord(L->ev[2], L->stream);
  if ((rc = cache_copy(h, L, 0, ncl))) return rc;
  QB_CUDA_TRY(L, cudaEventRecord(L->ev_cache_in, L->stream));
  cudaEventRecord(L->ev[3], L->stream);
  return QB200_OK;
}

// set s's n matched points a / b (caller memory of the call's kind) into its slots of ma / mb, and n into h_cloud_n[s]
int copy_set_points(Lane* L, const BatchCall& in, int s, const float* a, const float* b, int n) {
  const cudaMemcpyKind ck = in.kind == QB200_MEM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
  L->h_cloud_n[s] = n;
  if (n > 0) {
    QB_CUDA_TRY(L, cudaMemcpyAsync(L->ma + (size_t)s * L->Lc, a, (size_t)n * sizeof(float4), ck, L->stream));
    QB_CUDA_TRY(L, cudaMemcpyAsync(L->mb + (size_t)s * L->Lc, b, (size_t)n * sizeof(float4), ck, L->stream));
  }
  return QB200_OK;
}

// Correspondence sets: the matched points of every set into ma / mb and its size into n_corr
int front_sets(Lane* L, const BatchCall& in, int w0, int np) {
  cudaEventRecord(L->ev[0], L->stream);
  if (int rc = wave_reset(L, 0)) return rc;
  for (int s = 0; s < np; ++s) {
    const qb200_corr_set& cs = in.sets[w0 + s];
    if (int rc = copy_set_points(L, in, s, cs.a, cs.b, cs.L)) return rc;
  }
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->ctr.n_corr, L->h_cloud_n, (size_t)np * sizeof(int), cudaMemcpyHostToDevice, L->stream));
  for (int i = 1; i <= 4; ++i) cudaEventRecord(L->ev[i], L->stream);  // no voxel, fpfh or match stage: slots 1 .. 3 are not reported
  return QB200_OK;
}

// Inlier sets: the matched points as front_sets copies them, then every set's ids into its slot of clique (inlier_import_kernel).
// Device ids are read in place through the table d_inl; host ids cross PCIe into the set's slot of corr_src, which a pose wave leaves
// idle (it has no correspondences to pack), and are imported from there.  The import is part of the h2d stage.
int front_inlier_sets(Lane* L, const BatchCall& in, int w0, int np) {
  cudaEventRecord(L->ev[0], L->stream);
  if (int rc = wave_reset(L, 0)) return rc;
  const bool host = in.kind == QB200_MEM_HOST;
  for (int s = 0; s < np; ++s) {
    const qb200_inlier_set& is = in.inlier_sets[w0 + s];
    if (int rc = copy_set_points(L, in, s, is.a, is.b, is.L)) return rc;
    int* stage = L->corr_src + (size_t)s * L->Lc;
    if (host && is.n_inliers > 0)
      QB_CUDA_TRY(L, cudaMemcpyAsync(stage, is.inliers, (size_t)is.n_inliers * sizeof(int), cudaMemcpyHostToDevice, L->stream));
    L->h_inl[s] = InlierSrc{host ? stage : is.inliers, is.n_inliers, 0};
  }
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->d_inl, L->h_inl, (size_t)np * sizeof(InlierSrc), cudaMemcpyHostToDevice, L->stream));
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->ctr.n_corr, L->h_cloud_n, (size_t)np * sizeof(int), cudaMemcpyHostToDevice, L->stream));
  if (int rc = launch_inlier_import(L, np)) return rc;
  for (int i = 1; i <= 4; ++i) cudaEventRecord(L->ev[i], L->stream);  // no voxel, fpfh or match stage: slots 1 .. 3 are not reported
  return QB200_OK;
}

// Host edge lists cross PCIe through the larger of two lane buffers that a graph wave leaves idle: raw_stage (it reads no scans) and
// adjp (K9 writes it only after the import).  Returns the capacity in edges.
long long edge_stage(Lane* L, int2** out) {
  const long long raw = 2LL * L->S * L->R * (long long)(sizeof(float4) / sizeof(int2));
  const long long perm = (long long)L->S * L->Lc * L->W * (long long)sizeof(uint32_t) / (long long)sizeof(int2);
  *out = raw >= perm ? reinterpret_cast<int2*>(L->raw_stage.get()) : reinterpret_cast<int2*>(L->adjp.get());
  return raw >= perm ? raw : perm;
}

// Graphs: every graph's adjacency into its slot of adj.  Host rows arrive by one 2-D copy each; host edge lists are packed into the
// edge staging as long as they fit, and a list that does not fit crosses in chunks after the wave's launch, each chunk imported before
// the next one overwrites the staging (the stream orders them).  Device edges and rows are read in place.
int front_graphs(Lane* L, const BatchCall& in, int w0, int np) {
  cudaEventRecord(L->ev[0], L->stream);
  if (int rc = wave_reset(L, 0)) return rc;
  const bool host = in.kind == QB200_MEM_HOST;
  int2* stage = nullptr;
  const long long cap = edge_stage(L, &stage);
  long long used = 0, max_edges = 0;
  int max_L = 0;
  std::vector<int> streamed;  // host edge lists that did not fit beside the others
  for (int s = 0; s < np; ++s) {
    const qb200_graph& g = in.graphs[w0 + s];
    GraphSrc& e = L->h_graph[s];
    e = GraphSrc{nullptr, nullptr, g.edges ? g.n_edges : 0, g.L, 0};
    L->h_cloud_n[s] = g.L;
    max_L = std::max(max_L, g.L);
    if (g.adj && g.L > 0) {
      uint32_t* slot = L->adj + (size_t)s * L->Lc * L->W;
      const size_t nb = (size_t)(g.L + 31) / 32;
      if (host)
        QB_CUDA_TRY(L, cudaMemcpy2DAsync(slot, (size_t)L->W * 4, g.adj, (size_t)g.words_per_row * 4, nb * 4, g.L, cudaMemcpyHostToDevice,
                                         L->stream));
      e.rows = host ? slot : g.adj;
      e.stride = host ? L->W : g.words_per_row;
    }
    if (!g.edges || g.n_edges <= 0) continue;
    const int2* src = reinterpret_cast<const int2*>(g.edges);
    if (!host) {
      e.edges = src;
    } else if (g.n_edges <= cap - used) {
      QB_CUDA_TRY(L, cudaMemcpyAsync(stage + used, src, (size_t)g.n_edges * sizeof(int2), cudaMemcpyHostToDevice, L->stream));
      e.edges = stage + used;
      used += g.n_edges;
    } else {
      streamed.push_back(s);
      continue;
    }
    max_edges = std::max(max_edges, (long long)g.n_edges);
  }
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->d_graph, L->h_graph, (size_t)np * sizeof(GraphSrc), cudaMemcpyHostToDevice, L->stream));
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->ctr.n_corr, L->h_cloud_n, (size_t)np * sizeof(int), cudaMemcpyHostToDevice, L->stream));
  for (int i = 1; i <= 4; ++i) cudaEventRecord(L->ev[i], L->stream);  // no voxel, fpfh or match stage: slots 1 .. 3 are not reported
  int rc;
  if ((rc = launch_row_import(L, np, max_L)) || (rc = launch_edge_import(L, np, max_edges, -1, nullptr))) return rc;
  for (const int s : streamed) {
    const qb200_graph& g = in.graphs[w0 + s];
    const int2* src = reinterpret_cast<const int2*>(g.edges);
    for (long long off = 0; off < g.n_edges; off += cap) {
      const long long m = std::min(cap, (long long)g.n_edges - off);
      QB_CUDA_TRY(L, cudaMemcpyAsync(stage, src + off, (size_t)m * sizeof(int2), cudaMemcpyHostToDevice, L->stream));
      if ((rc = launch_edge_import(L, 1, m, s, stage))) return rc;
    }
  }
  return launch_symmetry_check(L, np, max_L);
}

// TIM graphs: K8 and the degrees, then the device-kind outputs written straight into the caller's arrays, the edge offsets of every
// set when edges are asked for (host-kind edges are emitted from them at collect time) and the records
int submit_graph(Lane* L, const qb200_graph_out& o, int w0, int np) {
  int rc;
  if ((rc = launch_graph(L, np))) return rc;
  const bool device = o.kind == QB200_MEM_DEVICE;
  const size_t rows0 = (size_t)w0 * o.rows_per_set;
  if (device) {
    const GraphDst d{o.adj ? o.adj + rows0 * o.words_per_row : nullptr, o.degree ? o.degree + rows0 : nullptr, o.rows_per_set,
                     o.words_per_row};
    if ((rc = launch_graph_export(L, np, d))) return rc;
  }
  if (o.edges && (rc = launch_edge_offsets(L, np))) return rc;
  if (o.edges && device) {
    int2* e = reinterpret_cast<int2*>(o.edges) + (size_t)w0 * o.cap_edges;
    if ((rc = launch_edge_emit(L, np, -1, 0, o.cap_edges, e, o.cap_edges))) return rc;
  }
  return launch_graph_records(L, np, o.edges ? o.cap_edges : 0);
}

// A collected TIM graph wave's host-kind outputs (h_results holds its records), before the lane is reused: each set's rows by one
// 2-D copy with the words past ceil(L / 32) zeroed here, its degrees by one copy, and its edge list emitted in windows through the
// edge staging (K9 does not run in a graph wave, so it is idle), each window copied out before the next one overwrites it.
int deliver_graph(Lane* L, const qb200_graph_out& o, int w0, int np) {
  int2* stage = nullptr;
  const long long cap = edge_stage(L, &stage);
  int rc;
  for (int s = 0; s < np; ++s) {
    const qb200_result& r = L->h_results[s];
    const int n = r.n_corr, nb = (n + 31) / 32;
    const size_t row0 = (size_t)(w0 + s) * o.rows_per_set;
    if (o.adj && n > 0)
      QB_CUDA_TRY(L, cudaMemcpy2DAsync(o.adj + row0 * o.words_per_row, (size_t)o.words_per_row * 4, L->adj + (size_t)s * L->Lc * L->W,
                                       (size_t)L->W * 4, (size_t)nb * 4, n, cudaMemcpyDeviceToHost, L->stream));
    if (o.degree && n > 0)
      QB_CUDA_TRY(L, cudaMemcpyAsync(o.degree + row0, L->deg + (size_t)s * L->Lc, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, L->stream));
    if (!o.edges) continue;
    int2* dst = reinterpret_cast<int2*>(o.edges) + (size_t)(w0 + s) * o.cap_edges;
    const long long m = std::min((long long)r.n_edges, (long long)o.cap_edges);
    for (long long e0 = 0; e0 < m; e0 += cap) {
      const long long e1 = std::min(m, e0 + cap);
      if ((rc = launch_edge_emit(L, 1, s, e0, e1, stage, 0))) return rc;
      QB_CUDA_TRY(L, cudaMemcpyAsync(dst + e0, stage, (size_t)(e1 - e0) * sizeof(int2), cudaMemcpyDeviceToHost, L->stream));
    }
  }
  QB_CUDA_TRY(L, cudaStreamSynchronize(L->stream));
  for (int s = 0; o.adj && s < np; ++s) {
    const int n = L->h_results[s].n_corr, nb = (n + 31) / 32;
    if (o.words_per_row == nb) continue;
    uint32_t* rows = o.adj + (size_t)(w0 + s) * o.rows_per_set * o.words_per_row;
    for (int i = 0; i < n; ++i) memset(rows + (size_t)i * o.words_per_row + nb, 0, (size_t)(o.words_per_row - nb) * sizeof(uint32_t));
  }
  return QB200_OK;
}

// Align sets: every set's table entry (its pose rows, threshold, counts, caps and where it is read and written), host-kind inputs
// staged: clouds back to back in raw_stage (at h_raw_off), source and target keypoints in the set's two slots of vox_pts, correspondences
// in aln_stage.  Host-kind outputs go to staging that wave_collect copies out: aligned clouds to the set's raw_stage region (in place
// for a host cloud), the correspondence outputs to aln_stage.  Device arrays are read and written in place.  Host inputs of a
// multi-wave batch cross on the batch's copy stream, and the lane waits for them.
int front_align(qb200_handle* h, Lane* L, const BatchCall& in, int w0, int np, int* n_blocks) {
  const qb200_align_out& o = *in.align_out;
  const bool host = in.kind == QB200_MEM_HOST, host_out = o.kind == QB200_MEM_HOST;
  const cudaStream_t cs = in.copy_stream ? in.copy_stream : L->stream;
  if ((host || host_out) && !L->aln_stage) QB_CUDA_TRY(L, L->aln_stage.alloc(AlignStage::bytes(L->S, L->Lc)));
  const AlignStage st = L->aln_stage ? AlignStage::carve(L->aln_stage, L->S, L->Lc) : AlignStage{};
  if (int rc = wave_reset(L, 0)) return rc;
  auto h2d = [&](void* dst, const void* src, size_t bytes) -> int {
    if (bytes) QB_CUDA_TRY(L, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, cs));
    return QB200_OK;
  };
  int raw = 0, blocks = 0;
  for (int s = 0; s < np; ++s) {
    const qb200_align_set& a = in.align_sets[w0 + s];
    const long long i = w0 + s;
    AlignSrc& e = L->h_aln[s];
    memset(&e, 0, sizeof(e));
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 4; ++c) e.T[4 * r + c] = a.T[4 * c + r];  // column-major in, T(r, c) out
    e.thr = 3.0 * (double)in.caller[i].voxel_size;
    e.n_points = a.n_points; e.n_src = a.n_src; e.n_tgt = a.n_tgt; e.n_corr = a.n_corr;
    e.cap_points = o.cap_points; e.cap_corr = o.cap_corr;
    e.cloud = reinterpret_cast<const float4*>(a.cloud);
    e.src_kp = reinterpret_cast<const float4*>(a.src_kp);
    e.tgt_kp = reinterpret_cast<const float4*>(a.tgt_kp);
    e.corr = reinterpret_cast<const int2*>(a.corr);
    float4* region = L->raw_stage + raw;
    L->h_raw_off[s] = raw;
    raw += a.n_points;
    if (host) {
      float4* sk = L->vox_pts + (size_t)s * L->V;
      float4* tk = L->vox_pts + (size_t)(L->S + s) * L->V;
      int2* cr = st.corr + (size_t)s * L->Lc;
      int rc;
      if ((o.aligned4 && (rc = h2d(region, a.cloud, (size_t)a.n_points * sizeof(float4)))) ||
          (rc = h2d(sk, a.src_kp, (size_t)a.n_src * sizeof(float4))) || (rc = h2d(tk, a.tgt_kp, (size_t)a.n_tgt * sizeof(float4))) ||
          (rc = h2d(cr, a.corr, (size_t)a.n_corr * sizeof(int2))))
        return rc;
      e.cloud = region; e.src_kp = sk; e.tgt_kp = tk; e.corr = cr;
    }
    if (host_out) {
      if (o.aligned4) e.aligned = region;
      if (o.matched4) e.matched = st.matched + (size_t)s * L->Lc;
      if (o.good4) e.good = st.good + (size_t)s * L->Lc;
      if (o.good_ids) e.good_ids = st.ids + (size_t)s * L->Lc;
    } else {
      if (o.aligned4) e.aligned = reinterpret_cast<float4*>(o.aligned4) + i * o.cap_points;
      if (o.matched4) e.matched = reinterpret_cast<float4*>(o.matched4) + i * o.cap_corr;
      if (o.good4) e.good = reinterpret_cast<float4*>(o.good4) + i * o.cap_corr;
      if (o.good_ids) e.good_ids = o.good_ids + i * o.cap_corr;
    }
    e.blk0 = blocks;
    if (o.aligned4) blocks += (std::min(a.n_points, o.cap_points) + kAlignPts - 1) / kAlignPts;
  }
  *n_blocks = blocks;
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->d_aln, L->h_aln, (size_t)np * sizeof(AlignSrc), cudaMemcpyHostToDevice, L->stream));
  if (in.copy_stream) {
    QB_CUDA_TRY(L, cudaEventRecord(h->ev_copied, in.copy_stream));
    QB_CUDA_TRY(L, cudaStreamWaitEvent(L->stream, h->ev_copied, 0));
  }
  return QB200_OK;
}

// Align sets: the good matches (and the refusals) first, then the clouds of the sets that were not refused, then every set's status
// and good count to the pinned mirror of the counter block
int submit_align(Lane* L, int np, int n_blocks) {
  int rc;
  if ((rc = launch_align_good(L, np)) || (rc = launch_align_points(L, n_blocks, np))) return rc;
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->hctr.cloud_status, L->ctr.cloud_status, (size_t)np * sizeof(int), cudaMemcpyDeviceToHost, L->stream));
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->hctr.n_final, L->ctr.n_final, (size_t)np * sizeof(int), cudaMemcpyDeviceToHost, L->stream));
  return QB200_OK;
}

// A collected align wave: status and counts of every set to the caller's host arrays (a refused set: its status alone), and in host
// kind the entries of every set that was not refused, from the staging its table entry names
int deliver_align(Lane* L, const qb200_align_out& o, int w0, int np) {
  bool copied = false;
  auto d2h = [&](void* dst, const void* src, int m, size_t size) -> int {
    if (dst && m > 0) {
      QB_CUDA_TRY(L, cudaMemcpyAsync(dst, src, (size_t)m * size, cudaMemcpyDeviceToHost, L->stream));
      copied = true;
    }
    return QB200_OK;
  };
  for (int s = 0; s < np; ++s) {
    const AlignSrc& e = L->h_aln[s];
    const int status = L->hctr.cloud_status[s], n_good = L->hctr.n_final[s];
    const long long i = w0 + s;
    if (o.status) o.status[i] = status;
    if (status != QB200_OK) continue;
    if (o.counts) {
      o.counts[3 * i] = e.n_points;
      o.counts[3 * i + 1] = e.n_corr;
      o.counts[3 * i + 2] = n_good;
    }
    if (o.kind != QB200_MEM_HOST) continue;
    const int mp = std::min(e.n_points, o.cap_points), mc = std::min(e.n_corr, o.cap_corr), mg = std::min(n_good, o.cap_corr);
    int rc;
    if ((rc = d2h(o.aligned4 ? o.aligned4 + 4 * i * o.cap_points : nullptr, e.aligned, mp, sizeof(float4))) ||
        (rc = d2h(o.matched4 ? o.matched4 + 4 * i * o.cap_corr : nullptr, e.matched, mc, sizeof(float4))) ||
        (rc = d2h(o.good_ids ? o.good_ids + i * o.cap_corr : nullptr, e.good_ids, mg, sizeof(int))) ||
        (rc = d2h(o.good4 ? o.good4 + 4 * i * o.cap_corr : nullptr, e.good, mg, sizeof(float4))))
      return rc;
  }
  if (copied) QB_CUDA_TRY(L, cudaStreamSynchronize(L->stream));
  return QB200_OK;
}

// The end of every wave with records: the list pack, the D2H of the records
int send_records(Lane* L, const BatchCall& in, int w0, int np) {
  if (in.lists)
    if (int rc = submit_lists(L, *in.lists, w0, np)) return rc;
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->h_results, L->d_results, (size_t)np * sizeof(qb200_result), cudaMemcpyDeviceToHost, L->stream));
  cudaEventRecord(L->ev[8], L->stream);
  return QB200_OK;
}

// Enqueue one wave (inputs [w0, w0 + np) of the call: np <= S pairs or sets, or np <= 2S scans) on lane L: its tables, the front of
// its source, then the tail of its sink: Solve K6..K7 (pairs) and K8..K11, Match K6..K7 and match_records_kernel, both then the lists
// and the D2H of the records; CacheSlots the copy into the cache slots; Export and Voxels the export to the caller's arrays.  No sync:
// wave_collect hands the outputs on.  The lane's previous wave must have been collected.
int wave_submit(qb200_handle* h, Lane* L, const BatchCall& in, int w0, int np) {
  const int ncl = np * clouds_per_input(in.src);
  int rc, n_blocks = 0;
  L->kev_armed[0] = L->kev_armed[1] = 0;
  L->pend_slots.clear();
  L->pend_writes = 0;
  if ((rc = fill_tables(L, in, w0, np))) return rc;
  switch (in.src) {
    case Source::RawPairs: case Source::RawScans: rc = front_raw(h, L, in, w0, np, ncl); break;
    case Source::FeaturePairs: case Source::DescriptorPairs: case Source::KeypointClouds: rc = front_features(h, L, in, w0, np, ncl); break;
    case Source::CachedPairs: rc = front_cached(h, L, in, w0, np, ncl); break;
    case Source::CorrSets: rc = front_sets(L, in, w0, np); break;
    case Source::Graphs: rc = front_graphs(L, in, w0, np); break;
    case Source::InlierSets: rc = front_inlier_sets(L, in, w0, np); break;
    case Source::AlignSets: rc = front_align(h, L, in, w0, np, &n_blocks); break;
  }
  if (rc) return rc;
  const bool match_pairs = is_pairs(in.src);
  const bool caller_kp = in.src == Source::FeaturePairs || in.src == Source::DescriptorPairs;
  int dims = 0;  // a descriptor wave: which K6 its pairs need
  for (int s = 0; in.src == Source::DescriptorPairs && s < np; ++s) dims |= in.descs[w0 + s].dim == kDescDim ? kDimsFpfh : kDimsOther;
  switch (in.sink) {
    case Sink::Solve:
      if (match_pairs && (rc = launch_match(L, np, caller_kp, dims))) return rc;
      cudaEventRecord(L->ev[4], L->stream);
      cudaEventRecord(L->ev[5], L->stream);  // re-recorded inside run_solver when the graph stage runs
      if ((rc = run_solver(L, np, match_pairs ? 1 : 0))) return rc;
      cudaEventRecord(L->ev[7], L->stream);
      rc = send_records(L, in, w0, np);
      break;
    case Sink::Match:  // no solver tail: the records come from the matcher's counters, and graph, clique and pose take no time
      if ((rc = launch_match(L, np, caller_kp, dims))) return rc;
      if ((rc = launch_match_records(L, np))) return rc;
      for (int i = 4; i <= 7; ++i) cudaEventRecord(L->ev[i], L->stream);
      rc = send_records(L, in, w0, np);
      break;
    case Sink::CacheSlots:
      if ((rc = cache_waits(h, L, ncl, true))) return rc;
      if ((rc = cache_copy(h, L, 1, ncl))) return rc;
      QB_CUDA_TRY(L, cudaEventRecord(L->ev_cache_out, L->stream));
      break;
    case Sink::Export: case Sink::Voxels: rc = submit_export(L, *in.out, w0, ncl, in.sink == Sink::Voxels); break;
    case Sink::Graph:  // no clique or pose stage: the graph slot holds K8 and the outputs
      if ((rc = submit_graph(L, *in.graph_out, w0, np))) return rc;
      for (int i = 5; i <= 7; ++i) cudaEventRecord(L->ev[i], L->stream);
      rc = send_records(L, in, w0, np);
      break;
    case Sink::Clique: {  // K9 on the imported graphs (a refused graph is in QB200_INLIER_NONE now, and every K9 kernel skips it)
      bool exact = false;
      for (int s = 0; s < np; ++s) exact |= L->h_solve[s].mode == QB200_PMC_EXACT;
      cudaEventRecord(L->ev[5], L->stream);
      if ((rc = launch_degree(L, np)) || (rc = launch_clique(L, np, exact))) return rc;
      cudaEventRecord(L->ev[6], L->stream);
      if ((rc = launch_clique_records(L, np))) return rc;
      cudaEventRecord(L->ev[7], L->stream);
      rc = send_records(L, in, w0, np);
      break;
    }
    case Sink::Pose:  // K10 / K11 on the imported ids, with the counters qb200_solve_pose gives (no front end), then the refusals
      for (int i = 5; i <= 6; ++i) cudaEventRecord(L->ev[i], L->stream);
      if ((rc = launch_fill_counters(L, np, 0)) || (rc = launch_pose(L, np)) || (rc = launch_pose_records(L, np))) return rc;
      cudaEventRecord(L->ev[7], L->stream);
      rc = send_records(L, in, w0, np);
      break;
    case Sink::AlignOut: rc = submit_align(L, np, n_blocks); break;
  }
  if (rc) return rc;
  L->pend_w0 = w0;
  L->pend_np = np;
  L->pend_stages = stage_slots(in.src, in.sink);
  L->pend_sink = in.sink;
  L->pend_dst = in.results;
  L->pend_host_lists = in.lists && in.lists->kind == QB200_MEM_HOST;
  if (in.lists) L->pend_lists = *in.lists;
  if (in.sink == Sink::Export || in.sink == Sink::Voxels) L->pend_out = *in.out;
  if (in.sink == Sink::Graph) L->pend_graph = *in.graph_out;
  if (in.sink == Sink::AlignOut) L->pend_align = *in.align_out;
  return QB200_OK;
}

// wait for the wave in flight on lane L, hand out what its sink produced and add its stage / kernel times to the handle
int wave_collect(qb200_handle* h, Lane* L) {
  if (L->pend_np == 0) return QB200_OK;
  const int np = L->pend_np;
  L->pend_np = 0;
  if (cudaStreamSynchronize(L->stream) != cudaSuccess) {
    h->fail(__FILE__, __LINE__, cudaGetErrorString(cudaGetLastError()));
    return QB200_ERR_CUDA;
  }
  int rc = QB200_OK;
  switch (L->pend_sink) {
    case Sink::Solve: case Sink::Match: case Sink::Clique: case Sink::Pose:
      memcpy(L->pend_dst + L->pend_w0, L->h_results, (size_t)np * sizeof(qb200_result));
      if (L->pend_host_lists) deliver_lists(L, L->pend_lists, L->pend_w0, np);
      break;
    case Sink::Graph:
      memcpy(L->pend_dst + L->pend_w0, L->h_results, (size_t)np * sizeof(qb200_result));
      if (L->pend_graph.kind == QB200_MEM_HOST) rc = deliver_graph(L, L->pend_graph, L->pend_w0, np);
      break;
    case Sink::CacheSlots: break;
    case Sink::Export: case Sink::Voxels: rc = deliver_export(L, L->pend_out, L->pend_w0, np, L->pend_sink == Sink::Voxels); break;
    case Sink::AlignOut: rc = deliver_align(L, L->pend_align, L->pend_w0, np); break;
  }
  if (h->timeline && (L->pend_stages & 1u)) {  // stage boundaries of a raw-scan or feature wave relative to the start of the batch (ms): start, h2d, voxel, fpfh, match, graph, clique, pose, d2h
    fprintf(stderr, "[qb200 timeline] wave w0=%d np=%d:", L->pend_w0, np);
    for (int i = 0; i < 9; ++i) {
      float ms = -1.f;
      cudaEventElapsedTime(&ms, h->ev_fork, L->ev[i]);
      fprintf(stderr, " %.2f", ms);
    }
    fprintf(stderr, "\n");
  }
  for (int i = 0; i < 8; ++i) {
    if (!(L->pend_stages >> i & 1u)) continue;
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, L->ev[i], L->ev[i + 1]) == cudaSuccess) h->stage_ms[i] += ms;
  }
  for (int k = 0; k < 2; ++k) {
    float ms = 0.f;
    if (L->kev_armed[k] && cudaEventElapsedTime(&ms, L->kev[2 * k], L->kev[2 * k + 1]) == cudaSuccess) {
      h->kernel_ms[k] += ms;
      h->kernel_calls[k] += 1;
    }
    L->kev_armed[k] = 0;
  }
  return rc;
}

// wait for the waves in flight (oldest first) whose records go to dst, or for all of them (dst == nullptr), and hand out their records
int collect_waves(qb200_handle* h, const qb200_result* dst) {
  int rc = QB200_OK;
  const int n = h->lanes_active > 0 ? h->lanes_active : 1;
  for (int i = 0; i < n; ++i) {
    Lane* L = h->lane[(h->lane_cursor + i) % n].get();
    if (!L || (dst && L->pend_dst != dst)) continue;
    const int rc2 = wave_collect(h, L);
    if (rc == QB200_OK) rc = rc2;
  }
  return rc;
}

int batch_flush(qb200_handle* h) {
  const int rc = collect_waves(h, nullptr);
  h->lanes_active = 0;
  h->lane_cursor = 0;
  return rc;
}

// The params of a call: one entry for the whole batch, or (each) one per pair (n entries; NULL is fine when n == 0).  Every entry passes
// params_ok (solver: its solver fields too); same_frontend: the call runs a front end or matches cached scans with one front-end
// configuration (the _each forms), so every entry carries the first entry's front-end fields (voxel_size .. seed, bit for bit).  A
// rejection names the entry.
int check_params(qb200_handle* h, const qb200_params* p, int n, bool each, bool same_frontend, bool solver) {
  const int m = each ? n : 1;
  char why[128];
  for (int i = 0; i < m; ++i) {
    if (!params_ok(p ? p + i : nullptr, solver)) {
      if (each) snprintf(why, sizeof(why), "params entry %d is null or out of range", i);
      h->fail(__FILE__, __LINE__, each ? why : "params are null or out of range");
      return QB200_ERR_BAD_ARG;
    }
    if (same_frontend && i > 0 && memcmp(p + i, p, offsetof(qb200_params, noise_bound)) != 0) {
      snprintf(why, sizeof(why), "params entry %d differs from entry 0 in its front-end fields (voxel_size .. seed)", i);
      h->fail(__FILE__, __LINE__, why);
      return QB200_ERR_BAD_ARG;
    }
  }
  return QB200_OK;
}

// The entries of a checked call of n > 0 pairs with their rotation noise bounds resolved (resolve_params): the one entry, or every
// pair's in pair order, as a sequence of single-pair calls in that order would latch them.  Empty on an allocation failure.
std::unique_ptr<qb200_params[]> resolve_call(qb200_handle* h, const qb200_params* p, int n, bool each) {
  const int m = each ? n : 1;
  std::unique_ptr<qb200_params[]> r(new (std::nothrow) qb200_params[m]);
  if (!r) {
    h->fail(__FILE__, __LINE__, "out of host memory for the params");
    return r;
  }
  for (int i = 0; i < m; ++i) r[i] = resolve_params(h, p[i]);
  return r;
}

// the call's input array: the one of its source
const void* input_of(const BatchCall& c) {
  switch (c.src) {
    case Source::RawPairs: return c.pairs;
    case Source::CachedPairs: return c.slots;
    case Source::FeaturePairs: return c.feats;
    case Source::DescriptorPairs: return c.descs;
    case Source::CorrSets: return c.sets;
    case Source::RawScans: case Source::KeypointClouds: return c.scans;
    case Source::Graphs: return c.graphs;
    case Source::InlierSets: return c.inlier_sets;
    case Source::AlignSets: return c.align_sets;
  }
  return nullptr;
}

// Every argument check of a batch call, in one order whatever its source, so that a call with several faults returns the same code:
// counts and arrays, the params entries, the cross-check, the lists, the outputs, then every input.  A rejection names its fault in
// qb200_last_error.
int check_call(qb200_handle* h, const BatchCall& c) {
  auto reject = [h](const char* why) {
    h->fail(__FILE__, __LINE__, why);
    return QB200_ERR_BAD_ARG;
  };
  const bool scans = clouds_per_input(c.src) == 1;
  if (c.n < 0) return reject("n < 0");
  if (c.n > 0 && !input_of(c)) return reject("the input array is null");
  if (c.n > 0 && scans && (!c.n_points || (c.sink == Sink::CacheSlots && !c.slot_ids))) return reject("the n_points or slot_ids array is null");
  if (c.n > 0 && has_records(c.sink) && !c.results) return reject("the results array is null");
  if (c.kind != QB200_MEM_HOST && c.kind != QB200_MEM_DEVICE) return reject("unknown memory kind of the inputs");
  const qb200_params* p = c.caller;
  char why[192];
  if (c.sink == Sink::Voxels) {  // only voxel_size and skip_flagged are read; the leaf is checked as qb200_voxelize checks it
    for (int i = 0; i < c.n; ++i) {
      if (!p || !(p[i].voxel_size > 0)) {
        snprintf(why, sizeof(why), "params entry %d is null or its voxel_size is not > 0", i);
        return reject(why);
      }
    }
  } else if (c.src == Source::KeypointClouds) {  // only the lattice fields are read
    for (int i = 0; i < c.n; ++i) {
      if (!p || !lattice_ok(p[i])) {
        snprintf(why, sizeof(why), "params entry %d is null or its radii or lattice cell are out of range", i);
        return reject(why);
      }
    }
  } else if (c.src == Source::Graphs) {  // only the clique fields are read
    for (int i = 0; i < c.n; ++i) {
      if (!p || (p[i].inlier_selection_mode != QB200_PMC_EXACT && p[i].inlier_selection_mode != QB200_PMC_HEU &&
                 p[i].inlier_selection_mode != QB200_KCORE_HEU) || p[i].max_clique_node_limit < 0) {
        snprintf(why, sizeof(why), "params entry %d is null, its inlier_selection_mode is not PMC_EXACT, PMC_HEU or KCORE_HEU, or its "
                 "max_clique_node_limit is negative", i);
        return reject(why);
      }
    }
  } else if (c.sink == Sink::AlignOut) {  // only voxel_size is read: the good-match threshold
    for (int i = 0; i < c.n; ++i) {
      if (!p || !(p[i].voxel_size > 0)) {
        snprintf(why, sizeof(why), "params entry %d is null or its voxel_size is not > 0", i);
        return reject(why);
      }
    }
  } else if (c.sink == Sink::Graph) {  // only noise_bound and cbar2 are read, checked as qb200_build_graph checks them
    for (int i = 0; i < c.n; ++i) {
      if (!p || !(p[i].noise_bound > 0) || !(p[i].cbar2 > 0)) {
        snprintf(why, sizeof(why), "params entry %d is null, or its noise_bound or cbar2 is not > 0", i);
        return reject(why);
      }
    }
  } else if (int rc = check_params(h, p, c.n, c.each(), c.src != Source::CorrSets && c.entries == Entries::Each, c.sink != Sink::Match)) {
    return rc;
  }
  for (int i = 0; is_pairs(c.src) && i < (c.each() ? c.n : 1); ++i) {
    if (!p[i].use_crosscheck) {
      if (c.each()) {
        snprintf(why, sizeof(why), "params entry %d: use_crosscheck = 0 is not supported", i);
        h->fail(__FILE__, __LINE__, why);
      }
      return QB200_ERR_UNSUPPORTED;
    }
  }
  const bool sets = c.src == Source::CorrSets || c.src == Source::InlierSets;
  if (int rc = check_lists(h, c.lists, sets, c.sink == Sink::Match, c.src == Source::Graphs)) return rc;
  if (c.sink == Sink::Export || c.sink == Sink::Voxels)
    if (int rc = check_out(h, c.out, c.src == Source::KeypointClouds)) return rc;
  if (c.sink == Sink::Voxels && (c.out->normals4 || c.out->desc33))
    return reject("normals4 and desc33 must be null: a voxelize call returns voxel centroids alone");
  if (c.sink == Sink::Graph)
    if (int rc = check_graph_out(h, c.graph_out)) return rc;
  if (c.sink == Sink::AlignOut)
    if (int rc = check_align_out(h, c.align_out)) return rc;
  const int R = h->cfg.max_raw_points;
  for (int i = 0; i < c.n; ++i) {
    const char* bad = nullptr;
    switch (c.src) {
      case Source::RawPairs: {
        const qb200_pair& q = c.pairs[i];
        if (q.n_src < 0 || q.n_tgt < 0 || q.n_src > R || q.n_tgt > R || (q.n_src > 0 && !q.src) || (q.n_tgt > 0 && !q.tgt))
          return reject("pair has a null cloud or exceeds max_raw_points");
        break;
      }
      case Source::CachedPairs: {
        const qb200_params& pe = p[c.each() ? i : 0];  // the pair's own entry
        for (const int sl : {c.slots[i].src_slot, c.slots[i].tgt_slot}) {
          if (sl < 0 || sl >= h->c_slots) return reject("slot outside qb200_cache_reserve()");
          const float* sig = h->c_sig.get() + 4 * (size_t)sl;
          if (sig[0] != pe.voxel_size || sig[1] != pe.normal_radius || sig[2] != pe.fpfh_radius || sig[3] != lattice_cell(pe)) {
            snprintf(why, sizeof(why), "pair %d: cached scan in slot %d was computed with other front-end parameters (or the slot is empty)",
                     i, sl);
            return reject(why);
          }
        }
        break;
      }
      case Source::FeaturePairs: {
        const qb200_feature_pair& f = c.feats[i];
        for (int side = 0; side < 2; ++side) {
          const int n = side ? f.n_tgt : f.n_src;
          const float* pts = side ? f.tgt : f.src;
          const float* desc = side ? f.tgt_desc : f.src_desc;
          if (n < 0 || n > h->cfg.max_voxel_points) bad = "count outside 0 .. max_voxel_points";
          else if (n > 0 && (!pts || !desc)) bad = "null keypoints or descriptors";
          else if (n > 0 && c.kind == QB200_MEM_DEVICE && !(device_array_of(h, pts, 16) && device_array_of(h, desc, 4)))
            bad = "keypoints (16-byte) or descriptors (4-byte) misaligned or not memory of the handle's device";
          if (bad) {
            snprintf(why, sizeof(why), "feature pair %d, %s: %s", i, side ? "target" : "source", bad);
            return reject(why);
          }
        }
        break;
      }
      case Source::DescriptorPairs: {
        const qb200_descriptor_pair& d = c.descs[i];
        if (d.dim < 1 || d.dim > QB200_MAX_DESC_DIM) bad = "dim outside 1 .. QB200_MAX_DESC_DIM";
        else if (d.stride < d.dim) bad = "stride < dim";
        if (bad) {
          snprintf(why, sizeof(why), "descriptor pair %d: %s", i, bad);
          return reject(why);
        }
        for (int side = 0; side < 2; ++side) {
          const int n = side ? d.n_tgt : d.n_src;
          const float* pts = side ? d.tgt : d.src;
          const float* desc = side ? d.tgt_desc : d.src_desc;
          if (n < 0 || n > h->cfg.max_voxel_points) bad = "count outside 0 .. max_voxel_points";
          else if (n > 0 && (!pts || !desc)) bad = "null keypoints or descriptors";
          else if (n > 0 && c.kind == QB200_MEM_DEVICE && !(device_array_of(h, pts, 16) && device_array_of(h, desc, 4)))
            bad = "keypoints (16-byte) or descriptors (4-byte) misaligned or not memory of the handle's device";
          if (bad) {
            snprintf(why, sizeof(why), "descriptor pair %d, %s: %s", i, side ? "target" : "source", bad);
            return reject(why);
          }
        }
        break;
      }
      case Source::CorrSets: {
        const qb200_corr_set& s = c.sets[i];
        const bool rows = c.sink == Sink::Graph && (c.graph_out->adj || c.graph_out->degree);
        if (s.L < 0 || s.L > h->cfg.max_corr || (s.L > 0 && (!s.a || !s.b))) bad = "it is null or its L is outside 0 .. max_corr";
        else if (rows && s.L > c.graph_out->rows_per_set) bad = "its L exceeds rows_per_set";
        if (bad && c.sink != Sink::Graph) return reject("correspondence set is null or exceeds max_corr");
        if (bad) {
          snprintf(why, sizeof(why), "set %d: %s", i, bad);
          return reject(why);
        }
        break;
      }
      case Source::InlierSets: {
        const qb200_inlier_set& s = c.inlier_sets[i];
        const bool device = c.kind == QB200_MEM_DEVICE;
        if (s.L < 0 || s.L > h->cfg.max_corr) bad = "its L is outside 0 .. max_corr";
        else if (s.n_inliers < 0 || s.n_inliers > s.L) bad = "its n_inliers is outside 0 .. L";
        else if (s.L > 0 && (!s.a || !s.b)) bad = "its points are null";
        else if (s.n_inliers > 0 && !s.inliers) bad = "its inlier list is null";
        else if (device && s.L > 0 && !(device_array_of(h, s.a, 16) && device_array_of(h, s.b, 16)))
          bad = "its points are misaligned (16 bytes) or not memory of the handle's device";
        else if (device && s.n_inliers > 0 && !device_array_of(h, s.inliers, 4))
          bad = "its inlier list is misaligned (4 bytes) or not memory of the handle's device";
        if (bad) {
          snprintf(why, sizeof(why), "set %d: %s", i, bad);
          return reject(why);
        }
        break;
      }
      case Source::AlignSets: {
        const qb200_align_set& s = c.align_sets[i];
        const bool device = c.kind == QB200_MEM_DEVICE;
        bool finite = true;
        for (const double t : s.T) finite &= std::isfinite(t);
        if (s.n_points < 0 || s.n_points > R) bad = "its n_points is outside 0 .. max_raw_points";
        else if (s.n_src < 0 || s.n_src > h->cfg.max_voxel_points || s.n_tgt < 0 || s.n_tgt > h->cfg.max_voxel_points)
          bad = "its n_src or n_tgt is outside 0 .. max_voxel_points";
        else if (s.n_corr < 0 || s.n_corr > h->cfg.max_corr) bad = "its n_corr is outside 0 .. max_corr";
        else if ((s.n_points > 0 && !s.cloud) || (s.n_src > 0 && !s.src_kp) || (s.n_tgt > 0 && !s.tgt_kp) || (s.n_corr > 0 && !s.corr))
          bad = "an array with a count > 0 is null";
        else if (!finite) bad = "its T has an entry that is not finite";
        else if (device && !(device_array_of(h, s.cloud, 16) && device_array_of(h, s.src_kp, 16) && device_array_of(h, s.tgt_kp, 16) &&
                             device_array_of(h, s.corr, 8)))
          bad = "points (16-byte) or corr (8-byte) misaligned or not memory of the handle's device";
        if (bad) {
          snprintf(why, sizeof(why), "set %d: %s", i, bad);
          return reject(why);
        }
        break;
      }
      case Source::KeypointClouds: {
        const int np = c.n_points[i];
        if (np < 0 || np > h->cfg.max_voxel_points) bad = "its point count is outside 0 .. max_voxel_points";
        else if (np > 0 && !c.scans[i]) bad = "it is null";
        else if (np > 0 && c.kind == QB200_MEM_DEVICE && !device_array_of(h, c.scans[i], 16))
          bad = "it is misaligned (16 bytes) or not memory of the handle's device";
        if (bad) {
          snprintf(why, sizeof(why), "cloud %d: %s", i, bad);
          return reject(why);
        }
        break;
      }
      case Source::Graphs: {
        const qb200_graph& g = c.graphs[i];
        if (g.L < 0 || g.L > h->cfg.max_corr) bad = "L is outside 0 .. max_corr";
        else if (g.edges && g.adj) bad = "edges and adj are both given";
        else if (g.edges && g.n_edges < 0) bad = "n_edges < 0";
        else if (!g.edges && !g.adj && g.L > 0 && g.n_edges > 0) bad = "it has edges but neither an edge list nor an adjacency matrix";
        else if (g.adj && g.words_per_row < (g.L + 31) / 32) bad = "words_per_row < ceil(L / 32)";
        else if (c.kind == QB200_MEM_DEVICE && !(device_array_of(h, g.edges, 8) && device_array_of(h, g.adj, 4)))
          bad = "edges (8-byte) or adj (4-byte) misaligned or not memory of the handle's device";
        if (bad) {
          snprintf(why, sizeof(why), "graph %d: %s", i, bad);
          return reject(why);
        }
        break;
      }
      case Source::RawScans: {
        const int np = c.n_points[i];
        if (c.sink == Sink::CacheSlots) {
          const int sl = c.slot_ids[i];
          if (sl < 0 || sl >= h->c_slots || np < 0 || np > R || (np > 0 && !c.scans[i])) {
            snprintf(why, sizeof(why), "scan %d is null, exceeds max_raw_points or names a slot outside qb200_cache_reserve()", i);
            return reject(why);
          }
          break;
        }
        if (np < 0 || np > R) bad = "its point count is outside 0 .. max_raw_points";
        else if (np > 0 && !c.scans[i]) bad = "it is null";
        else if (c.sink == Sink::Voxels && np > 0 && c.kind == QB200_MEM_DEVICE && !device_array_of(h, c.scans[i], 16))
          bad = "it is misaligned (16 bytes) or not memory of the handle's device";
        if (bad) {
          snprintf(why, sizeof(why), "scan %d: %s", i, bad);
          return reject(why);
        }
        break;
      }
    }
  }
  return QB200_OK;
}

// Check a batch call and queue it: its waves rotate over up to h->max_lanes lanes whatever its input, and a lane is collected (its
// records copied out) only when it is needed again, so the tail of one batch runs under the copies and front-end kernels of the
// next.  Each lane has its own slot table; cache writes and cached pairs order their copies to and from the scan cache by
// cache_waits, and qb200_cache_reserve / _copy / _read flush first (enter).  The caller's input arrays (host kind), `results` and
// lists must stay valid until batch_flush (in qb200_register_batch_flush or the next call that is not an enqueue) has returned them.
int enqueue_call(qb200_handle* h, BatchCall c) {
  if (!h) return QB200_ERR_BAD_ARG;
  int rc;
  if ((rc = check_call(h, c))) return rc;
  cudaSetDevice(h->cfg.device);
  const bool pipelined = h->lanes_active > 0;  // waves of an earlier enqueue are still in flight
  if (!pipelined) reset_timers(h);
  // An empty call resolves no params: the reference latches the rotation noise bound inside computeTransformation, which an empty
  // batch never calls.
  if (c.n == 0) return QB200_OK;
  // only the solver and the pose read the rotation noise bound: the other sinks resolve nothing
  std::unique_ptr<qb200_params[]> pr;
  const bool solves = c.sink == Sink::Solve || c.sink == Sink::Pose;
  if (solves && !(pr = resolve_call(h, c.caller, c.n, c.each()))) return QB200_ERR_CUDA;
  c.params = solves ? pr.get() : c.caller;
  // S: inputs per wave, pairs, sets or scans; the clouds of a wave fill the lane's 2 * max_batch_slots cloud buffers
  const int S = h->cfg.max_batch_slots * (clouds_per_input(c.src) == 1 ? 2 : 1), lanes = h->max_lanes;
  // host inputs crossing PCIe: the copy stream and the quarter-wave opening below are theirs alone
  const bool host_scans = crosses_pcie(c.src) && c.kind == QB200_MEM_HOST;
  // More than one wave: rotate over the lanes so that one wave's PCIe copies and single-warp solver tail run under the
  // other waves' dense kernels.  Results do not depend on the lane (no state is shared between waves).
  // Wave plan.  Host scans: nothing can run before the first wave's scans crossed PCIe, so the batch opens with a quarter
  // wave (its copy is the only one that is not hidden) followed by the remaining three quarters; all other waves are full.
  // (Closing with small waves as well does not pay: every wave carries the same single-warp solver tail.)
  int wave_n[64], n_waves = 0;
  {
    int left = c.n;
    if (host_scans && c.n > S && S >= 8 && lanes > 1) {
      wave_n[n_waves++] = S / 4;
      wave_n[n_waves++] = S - S / 4;
      left -= S;
    }
    while (left > 0 && n_waves < 63) {
      wave_n[n_waves] = left < S ? left : S;
      left -= wave_n[n_waves++];
    }
    if (left > 0) n_waves = 0;  // more than ~60 waves: no special opening, walk uniformly below
  }
  const bool planned = n_waves > 0;
  if (!planned) n_waves = (c.n + S - 1) / S;
  const int n_lanes = n_waves < lanes ? n_waves : lanes;
  if (pipelined && h->lanes_active != n_lanes) {  // a different lane count: start a fresh rotation
    if ((rc = batch_flush(h))) return rc;
  }
  const bool fresh = h->lanes_active == 0;
  for (int l = 1; l < n_lanes; ++l) {
    if (!h->lane[l]) {
      if ((rc = lane_alloc(*h->lane[0], &h->lane[l]))) {
        h->fail(__FILE__, __LINE__, "cannot allocate another lane");
        return rc;
      }
    }
    // the lanes start after whatever the caller queued on lane 0's stream (first batch of a pipelined sequence only: later
    // on lane 0's stream carries a wave of its own)
    if (fresh) {
      if (l == 1) QB_CUDA_TRY(h, cudaEventRecord(h->ev_fork, h->lane[0]->stream));
      QB_CUDA_TRY(h, cudaStreamWaitEvent(h->lane[l]->stream, h->ev_fork, 0));
    }
  }
  // host scans of a multi-wave batch: one copy stream, ordered after whatever the caller queued on lane 0's stream
  if (host_scans && n_lanes > 1) {
    c.copy_stream = h->copy_stream;
    if (fresh) QB_CUDA_TRY(h, cudaStreamWaitEvent(c.copy_stream, h->ev_fork, 0));
  }
  h->lanes_active = n_lanes;
  // a cache write's signatures, in scan order (a slot named twice ends with its last scan's): the checks of the calls queued after it
  // see them
  for (int i = 0; c.sink == Sink::CacheSlots && i < c.n; ++i) {
    const qb200_params& pc = c.params[c.each() ? i : 0];
    float* sig = h->c_sig.get() + 4 * (size_t)c.slot_ids[i];
    sig[0] = pc.voxel_size; sig[1] = pc.normal_radius; sig[2] = pc.fpfh_radius; sig[3] = lattice_cell(pc);
  }
  for (int w0 = 0, wave = 0; w0 < c.n && rc == QB200_OK; ++wave) {
    Lane* L = h->lane[h->lane_cursor].get();
    int np = planned ? wave_n[wave] : S;
    if (np > c.n - w0) np = c.n - w0;
    if ((rc = wave_collect(h, L))) break;  // the lane's previous wave (its pinned tables are reused)
    rc = wave_submit(h, L, c, w0, np);
    h->lane_cursor = (h->lane_cursor + 1) % n_lanes;  // always the lane that has been busy longest
    w0 += np;
  }
  return rc;
}

// A blocking batch call: enqueue_call + batch_flush, which waits for everything in flight also after an error (the copies read caller
// memory).  With one pair it also sets what qb200_get_last_* read.
int run_call(qb200_handle* h, const BatchCall& c) {
  int rc = enqueue_call(h, c);
  const int rc2 = h ? batch_flush(h) : QB200_OK;
  if (rc == QB200_OK) rc = rc2;
  if (rc == QB200_OK && c.n == 1 && (c.sink == Sink::Solve || c.sink == Sink::Match)) {
    // what the wave left in slot 0: the clique and final inliers (none in a match), the packed correspondences of a pair (a set's
    // are the caller's points, with no index pairs), the features of a raw pair
    set_last(h, c.results[0]);
    stamp_last(h, {kLastClique, kLastFinal});
    if (is_pairs(c.src)) stamp_last(h, {kLastCorr});
    if (c.src == Source::RawPairs) stamp_last(h, {kLastFeatures});
    if (c.src == Source::DescriptorPairs && c.sink == Sink::Match) {  // what match_mutual_kernel read, as after qb200_match
      const qb200_descriptor_pair& d = c.descs[0];
      const bool both = d.n_src > 0 && d.n_tgt > 0;
      h->last_match_n[0] = both ? d.n_src : 0;
      h->last_match_n[1] = both ? d.n_tgt : 0;
      stamp_last(h, {kLastNn});
    }
  }
  return rc;
}

// One constructor per source: the call's inputs, its params entries and the outputs of its sink
BatchCall raw_pairs(Sink k, Entries e, const qb200_pair* pairs, int32_t n, const qb200_params* p, qb200_mem_kind kind, qb200_result* results,
                    const qb200_pair_lists* lists) {
  BatchCall c{Source::RawPairs, k, n, kind, p, e};
  c.pairs = pairs; c.results = results; c.lists = lists;
  return c;
}

// cached scans are on the device, and their slot pairs in host memory
BatchCall cached_pairs(Sink k, Entries e, const qb200_slot_pair* slots, int32_t n, const qb200_params* p, qb200_result* results,
                       const qb200_pair_lists* lists) {
  BatchCall c{Source::CachedPairs, k, n, QB200_MEM_HOST, p, e};
  c.slots = slots; c.results = results; c.lists = lists;
  return c;
}

// the entries' front-end fields are ignored, so they may differ
BatchCall feature_pairs(Sink k, const qb200_feature_pair* feats, int32_t n, const qb200_params* p, qb200_mem_kind kind, qb200_result* results,
                        const qb200_pair_lists* lists) {
  BatchCall c{Source::FeaturePairs, k, n, kind, p, Entries::Mixed};
  c.feats = feats; c.results = results; c.lists = lists;
  return c;
}

// the entries' front-end fields are ignored, so they may differ
BatchCall descriptor_pairs(Sink k, const qb200_descriptor_pair* descs, int32_t n, const qb200_params* p, qb200_mem_kind kind,
                           qb200_result* results, const qb200_pair_lists* lists) {
  BatchCall c{Source::DescriptorPairs, k, n, kind, p, Entries::Mixed};
  c.descs = descs; c.results = results; c.lists = lists;
  return c;
}

BatchCall corr_sets(Sink k, Entries e, const qb200_corr_set* sets, int32_t n, const qb200_params* p, qb200_mem_kind kind, qb200_result* results,
                    const qb200_pair_lists* lists) {
  BatchCall c{Source::CorrSets, k, n, kind, p, e};
  c.sets = sets; c.results = results; c.lists = lists;
  return c;
}

// TIM graphs of the sets into the caller's arrays: each set is built with its own entry
BatchCall corr_sets(const qb200_corr_set* sets, int32_t n, const qb200_params* p, qb200_mem_kind kind, qb200_result* results,
                    const qb200_graph_out* out) {
  BatchCall c{Source::CorrSets, Sink::Graph, n, kind, p, Entries::Mixed};
  c.sets = sets; c.results = results; c.graph_out = out;
  return c;
}

// slot_ids for the CacheSlots sink, out for Export and Voxels; every scan runs its own front end, so the entries may differ
BatchCall raw_scans(Sink k, Entries e, const float* const* scans4, const int32_t* n_points, int32_t n, const qb200_params* p, qb200_mem_kind kind,
                    const int32_t* slot_ids, const qb200_feature_out* out) {
  BatchCall c{Source::RawScans, k, n, kind, p, e};
  c.scans = scans4; c.n_points = n_points; c.slot_ids = slot_ids; c.out = out;
  return c;
}

BatchCall keypoint_clouds(Sink k, const float* const* pts4, const int32_t* n_points, int32_t n, const qb200_params* p, qb200_mem_kind kind,
                          const qb200_feature_out* out) {
  BatchCall c{Source::KeypointClouds, k, n, kind, p, Entries::Mixed};
  c.scans = pts4; c.n_points = n_points; c.out = out;
  return c;
}

// each graph is solved with its own entry
BatchCall caller_graphs(const qb200_graph* graphs, int32_t n, const qb200_params* p, qb200_mem_kind kind, qb200_result* results,
                        const qb200_pair_lists* lists) {
  BatchCall c{Source::Graphs, Sink::Clique, n, kind, p, Entries::Mixed};
  c.graphs = graphs; c.results = results; c.lists = lists;
  return c;
}

// each inlier set is solved with its own entry
BatchCall inlier_sets(const qb200_inlier_set* sets, int32_t n, const qb200_params* p, qb200_mem_kind kind, qb200_result* results,
                      const qb200_pair_lists* lists) {
  BatchCall c{Source::InlierSets, Sink::Pose, n, kind, p, Entries::Mixed};
  c.inlier_sets = sets; c.results = results; c.lists = lists;
  return c;
}

// each set is aligned with its own entry's voxel size
BatchCall align_sets(const qb200_align_set* sets, int32_t n, const qb200_params* p, qb200_mem_kind kind, const qb200_align_out* out) {
  BatchCall c{Source::AlignSets, Sink::AlignOut, n, kind, p, Entries::Mixed};
  c.align_sets = sets; c.align_out = out;
  return c;
}

}  // namespace

extern "C" {

int qb200_version(void) { return QB200_VERSION; }

void qb200_default_params(qb200_params* p) {
  memset(p, 0, sizeof(*p));
  p->voxel_size = 0.3f; p->normal_radius = 0.5f; p->fpfh_radius = 0.75f; p->grid_cell = 0.0f;  // config/params.yaml:22-25
  p->tuple_scale = 0.95f; p->use_crosscheck = 1; p->use_tuple_test = 1; p->tuple_trials_per_corr = 100;  // fpfh_manager.hpp:126-127
  p->skip_flagged = 1; p->seed = 0x5EED;
  p->noise_bound = 0.3; p->cbar2 = 1.0; p->rot_noise_bound = 0.0; p->cote_noise_bound = 0.3;  // params.yaml:31,34; quatro.hpp:115
  p->rotation_gnc_factor = 1.4; p->rotation_cost_threshold = 0.00011; p->kcore_heuristic_threshold = 0.5;  // params.yaml:41,44
  p->rotation_max_iterations = 50; p->inlier_selection_mode = QB200_PMC_HEU; p->cote_mode = QB200_COTE_MEDIAN;  // params.yaml:38
  p->using_rot_inliers_when_estimating_cote = 0; p->use_pre_estimated_RyRx = 0;
  p->RyRx[0] = p->RyRx[4] = p->RyRx[8] = 1.0;
}

void qb200_default_config(qb200_config* c) {
  memset(c, 0, sizeof(*c));
  c->device = 0; c->max_batch_slots = 64; c->max_raw_points = 131072; c->max_voxel_points = 16384; c->max_corr = 4096;
}

int qb200_create(const qb200_config* cfg_in, qb200_handle** out) {
  if (!out) return QB200_ERR_BAD_ARG;
  *out = nullptr;
  qb200_config cfg;
  if (cfg_in) cfg = *cfg_in; else qb200_default_config(&cfg);
  if (cfg.max_batch_slots < 1 || cfg.max_batch_slots > 2048 || cfg.max_raw_points < 1 || cfg.max_voxel_points < kMatchTile ||
      cfg.max_voxel_points % kMatchTile != 0 || cfg.max_voxel_points > QB200_MAX_VOXEL_POINTS || cfg.max_corr < 32 || cfg.max_corr % 32 != 0 ||
      cfg.max_corr > QB200_MAX_CORR || (long long)cfg.max_batch_slots * 2 * cfg.max_raw_points > 2000000000LL ||
      (long long)cfg.max_batch_slots * 2 * cfg.max_voxel_points > 2000000000LL)
    return QB200_ERR_BAD_ARG;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || cfg.device < 0 || cfg.device >= ndev) return QB200_ERR_NO_DEVICE;
  if (cudaSetDevice(cfg.device) != cudaSuccess) return QB200_ERR_NO_DEVICE;
  Lane like{};  // the settings every lane of the handle shares
  like.S = cfg.max_batch_slots; like.R = cfg.max_raw_points; like.V = cfg.max_voxel_points; like.Lc = cfg.max_corr;
  like.W = like.Lc / 32; like.NS = like.V / kMatchTile;
  like.device = cfg.device;
  if (cudaDeviceGetAttribute(&like.n_sm, cudaDevAttrMultiProcessorCount, cfg.device) != cudaSuccess || like.n_sm <= 0) return QB200_ERR_NO_DEVICE;
  // Every QB200_* switch is read here, once per handle.  K6 implementation switch: the tensor-core filter + in-kernel exact
  // evaluation is the default; QB200_MATCH_EXACT=1 forces the exact CUDA-core kernel everywhere (identical results; A/B and triage)
  auto env_on = [](const char* name) { const char* v = getenv(name); return (v && v[0] == '1') ? 1 : 0; };
  like.force_exact_match = env_on("QB200_MATCH_EXACT");
  like.tc_verify = env_on("QB200_TC_VERIFY");
  like.tc_prof = env_on("QB200_TC_PROF");
  qb200_handle* h = new (std::nothrow) qb200_handle();
  if (!h) return QB200_ERR_CUDA;
  h->cfg = cfg;
  const char* ln = getenv("QB200_LANES");
  h->max_lanes = (ln && ln[0] >= '1' && ln[0] <= '8') ? ln[0] - '0' : 4;
  h->timeline = env_on("QB200_TIMELINE");
  like.err = h->err;
  auto alloc = [&]() -> int {
    QB_CUDA_TRY(h, h->ev_fork.create());  // (timing enabled: QB200_TIMELINE measures the waves against it)
    QB_CUDA_TRY(h, h->copy_stream.create(cudaStreamNonBlocking));
    QB_CUDA_TRY(h, h->ev_copied.create(cudaEventDisableTiming));
    return lane_alloc(like, &h->lane[0]);
  };
  const int rc = alloc();
  if (rc != QB200_OK) {
    fprintf(stderr, "qb200_create: %s\n", h->err);
    qb200_destroy(h);
    return rc;
  }
  *out = h;
  return QB200_OK;
}

void qb200_destroy(qb200_handle* h) {
  if (!h) return;
  cudaSetDevice(h->cfg.device);
  cudaDeviceSynchronize();
  comm_release(h);
  delete h;
}

int qb200_set_stream(qb200_handle* h, void* cuda_stream) {
  if (int rc = enter(h)) return rc;
  Lane* L = h->lane[0].get();
  L->stream = cuda_stream ? (cudaStream_t)cuda_stream : L->own_stream;
  return QB200_OK;
}

const char* qb200_last_error(const qb200_handle* h) { return h ? h->err : "null handle"; }
int64_t qb200_launch_count(const qb200_handle* h) {
  if (!h) return 0;
  int64_t n = 0;
  for (const auto& L : h->lane)
    if (L) n += L->launches;
  return n;
}

// ---- batches of precomputed correspondences -> poses ------------------------------------------------------
int qb200_solve_batch(qb200_handle* h, const qb200_corr_set* sets, int32_t n_sets, const qb200_params* p, qb200_mem_kind kind,
                      qb200_result* results) {
  return qb200_solve_batch_ex(h, sets, n_sets, p, kind, results, nullptr);
}

int qb200_solve_batch_ex(qb200_handle* h, const qb200_corr_set* sets, int32_t n_sets, const qb200_params* p, qb200_mem_kind kind,
                         qb200_result* results, const qb200_pair_lists* lists) {
  return run_call(h, corr_sets(Sink::Solve, Entries::One, sets, n_sets, p, kind, results, lists));
}

int qb200_solve_batch_each(qb200_handle* h, const qb200_corr_set* sets, int32_t n_sets, const qb200_params* params, qb200_mem_kind kind,
                           qb200_result* results, const qb200_pair_lists* lists) {
  return run_call(h, corr_sets(Sink::Solve, Entries::Each, sets, n_sets, params, kind, results, lists));
}

int qb200_solve_batch_enqueue_each(qb200_handle* h, const qb200_corr_set* sets, int32_t n_sets, const qb200_params* params,
                                   qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists) {
  return enqueue_call(h, corr_sets(Sink::Solve, Entries::Each, sets, n_sets, params, kind, results, lists));
}

// ---- raw scans -> pose ------------------------------------------------------------------------------
int qb200_register_batch_flush(qb200_handle* h) { return enter(h); }

int qb200_register_batch(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* p, qb200_mem_kind kind,
                         qb200_result* results) {
  return qb200_register_batch_ex(h, pairs, n_pairs, p, kind, results, nullptr);
}

int qb200_register_batch_ex(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* p, qb200_mem_kind kind,
                            qb200_result* results, const qb200_pair_lists* lists) {
  return run_call(h, raw_pairs(Sink::Solve, Entries::One, pairs, n_pairs, p, kind, results, lists));
}

int qb200_register_batch_each(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* params, qb200_mem_kind kind,
                              qb200_result* results, const qb200_pair_lists* lists) {
  return run_call(h, raw_pairs(Sink::Solve, Entries::Each, pairs, n_pairs, params, kind, results, lists));
}

int qb200_register_batch_enqueue(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* p, qb200_mem_kind kind,
                                 qb200_result* results) {
  return enqueue_call(h, raw_pairs(Sink::Solve, Entries::One, pairs, n_pairs, p, kind, results, nullptr));
}

int qb200_register_batch_enqueue_ex(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* p, qb200_mem_kind kind,
                                    qb200_result* results, const qb200_pair_lists* lists) {
  return enqueue_call(h, raw_pairs(Sink::Solve, Entries::One, pairs, n_pairs, p, kind, results, lists));
}

int qb200_register_batch_enqueue_each(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                      qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists) {
  return enqueue_call(h, raw_pairs(Sink::Solve, Entries::Each, pairs, n_pairs, params, kind, results, lists));
}

int qb200_register_batch_mixed(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* params, qb200_mem_kind kind,
                               qb200_result* results, const qb200_pair_lists* lists) {
  return run_call(h, raw_pairs(Sink::Solve, Entries::Mixed, pairs, n_pairs, params, kind, results, lists));
}

int qb200_register_batch_enqueue_mixed(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                       qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists) {
  return enqueue_call(h, raw_pairs(Sink::Solve, Entries::Mixed, pairs, n_pairs, params, kind, results, lists));
}

int qb200_register_pair(qb200_handle* h, const float* src4, int32_t n_src, const float* tgt4, int32_t n_tgt, const qb200_params* p,
                        qb200_result* res) {
  if (!res) return QB200_ERR_BAD_ARG;
  qb200_pair pr;
  pr.src = src4; pr.tgt = tgt4; pr.n_src = n_src; pr.n_tgt = n_tgt;
  const int rc = qb200_register_batch(h, &pr, 1, p, QB200_MEM_HOST, res);
  if (rc != QB200_OK) return rc;
  return res->status;
}

int qb200_get_stage_ms(qb200_handle* h, float* ms, int32_t n) {
  if (!h || !ms || n < 0) return QB200_ERR_BAD_ARG;
  for (int i = 0; i < n && i < 8; ++i) ms[i] = h->stage_ms[i];
  return QB200_OK;
}

// ---- scan cache ---------------------------------------------------------------------------------------------------------
int qb200_cache_reserve(qb200_handle* h, int32_t n_slots) {
  if (int rc = enter(h)) return rc;
  if (n_slots < 0 || n_slots > (1 << 20)) return QB200_ERR_BAD_ARG;
  QB_CUDA_TRY(h, cudaStreamSynchronize(h->lane[0]->stream));
  // the old cache goes first, so the device never holds two
  h->c_slots = 0;
  h->c_vox.reset(); h->c_nrm.reset(); h->c_desc.reset(); h->c_n.reset(); h->c_status.reset(); h->c_sig.reset();
  if (n_slots == 0) return QB200_OK;
  const size_t V = h->cfg.max_voxel_points, N = (size_t)n_slots;
  QB_CUDA_TRY(h, h->c_vox.alloc(N * V));
  QB_CUDA_TRY(h, h->c_nrm.alloc(N * V));
  QB_CUDA_TRY(h, h->c_desc.alloc(N * kDescK * V));
  QB_CUDA_TRY(h, h->c_n.alloc(N));
  QB_CUDA_TRY(h, h->c_status.alloc(N));
  QB_CUDA_TRY(h, cudaMemset(h->c_n, 0, N * sizeof(int)));
  QB_CUDA_TRY(h, cudaMemset(h->c_status, 0, N * sizeof(int)));
  QB_CUDA_TRY(h, cudaMemset(h->c_desc, 0, N * kDescK * V * sizeof(float)));
  h->c_sig.reset(new (std::nothrow) float[4 * N]());
  if (!h->c_sig) return QB200_ERR_CUDA;
  h->c_slots = n_slots;
  return QB200_OK;
}

int qb200_cache_scans(qb200_handle* h, const float* const* scans4, const int32_t* n_points, const int32_t* slot_ids, int32_t n_scans,
                      const qb200_params* p, qb200_mem_kind kind) {
  return run_call(h, raw_scans(Sink::CacheSlots, Entries::One, scans4, n_points, n_scans, p, kind, slot_ids, nullptr));
}

int qb200_cache_scans_each(qb200_handle* h, const float* const* scans4, const int32_t* n_points, const int32_t* slot_ids, int32_t n_scans,
                           const qb200_params* params, qb200_mem_kind kind) {
  return run_call(h, raw_scans(Sink::CacheSlots, Entries::Mixed, scans4, n_points, n_scans, params, kind, slot_ids, nullptr));
}

int qb200_cache_scans_enqueue_each(qb200_handle* h, const float* const* scans4, const int32_t* n_points, const int32_t* slot_ids,
                                   int32_t n_scans, const qb200_params* params, qb200_mem_kind kind) {
  return enqueue_call(h, raw_scans(Sink::CacheSlots, Entries::Mixed, scans4, n_points, n_scans, params, kind, slot_ids, nullptr));
}

int qb200_register_cached(qb200_handle* h, const qb200_slot_pair* pairs, int32_t n_pairs, const qb200_params* p, qb200_result* results) {
  return qb200_register_cached_ex(h, pairs, n_pairs, p, results, nullptr);
}

int qb200_register_cached_ex(qb200_handle* h, const qb200_slot_pair* pairs, int32_t n_pairs, const qb200_params* p, qb200_result* results,
                             const qb200_pair_lists* lists) {
  return run_call(h, cached_pairs(Sink::Solve, Entries::One, pairs, n_pairs, p, results, lists));
}

int qb200_register_cached_each(qb200_handle* h, const qb200_slot_pair* pairs, int32_t n_pairs, const qb200_params* params, qb200_result* results,
                               const qb200_pair_lists* lists) {
  return run_call(h, cached_pairs(Sink::Solve, Entries::Each, pairs, n_pairs, params, results, lists));
}

int qb200_register_cached_mixed(qb200_handle* h, const qb200_slot_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                qb200_result* results, const qb200_pair_lists* lists) {
  return run_call(h, cached_pairs(Sink::Solve, Entries::Mixed, pairs, n_pairs, params, results, lists));
}

int qb200_register_cached_enqueue_mixed(qb200_handle* h, const qb200_slot_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                        qb200_result* results, const qb200_pair_lists* lists) {
  return enqueue_call(h, cached_pairs(Sink::Solve, Entries::Mixed, pairs, n_pairs, params, results, lists));
}

// ---- caller keypoints and descriptors -> pose ------------------------------------------------------------------------------
int qb200_register_features_each(qb200_handle* h, const qb200_feature_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                 qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists) {
  return run_call(h, feature_pairs(Sink::Solve, pairs, n_pairs, params, kind, results, lists));
}

int qb200_register_features_enqueue_each(qb200_handle* h, const qb200_feature_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                         qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists) {
  return enqueue_call(h, feature_pairs(Sink::Solve, pairs, n_pairs, params, kind, results, lists));
}

// ---- caller keypoints and descriptors of any length -> correspondences, or pose --------------------------------------------------
int qb200_match_descriptors_each(qb200_handle* h, const qb200_descriptor_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                 qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists) {
  return run_call(h, descriptor_pairs(Sink::Match, pairs, n_pairs, params, kind, results, lists));
}

int qb200_match_descriptors_enqueue_each(qb200_handle* h, const qb200_descriptor_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                         qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists) {
  return enqueue_call(h, descriptor_pairs(Sink::Match, pairs, n_pairs, params, kind, results, lists));
}

int qb200_register_descriptors_each(qb200_handle* h, const qb200_descriptor_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                    qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists) {
  return run_call(h, descriptor_pairs(Sink::Solve, pairs, n_pairs, params, kind, results, lists));
}

int qb200_register_descriptors_enqueue_each(qb200_handle* h, const qb200_descriptor_pair* pairs, int32_t n_pairs,
                                            const qb200_params* params, qb200_mem_kind kind, qb200_result* results,
                                            const qb200_pair_lists* lists) {
  return enqueue_call(h, descriptor_pairs(Sink::Solve, pairs, n_pairs, params, kind, results, lists));
}

// ---- raw scans -> voxel keypoints, normals and FPFH-33 in caller memory ---------------------------------------------------------
int qb200_describe_batch_each(qb200_handle* h, const float* const* scans4, const int32_t* n_points, int32_t n_scans, const qb200_params* params,
                              qb200_mem_kind kind, const qb200_feature_out* out) {
  return run_call(h, raw_scans(Sink::Export, Entries::Mixed, scans4, n_points, n_scans, params, kind, nullptr, out));
}

int qb200_describe_batch_enqueue_each(qb200_handle* h, const float* const* scans4, const int32_t* n_points, int32_t n_scans,
                                      const qb200_params* params, qb200_mem_kind kind, const qb200_feature_out* out) {
  return enqueue_call(h, raw_scans(Sink::Export, Entries::Mixed, scans4, n_points, n_scans, params, kind, nullptr, out));
}

// ---- raw scans -> voxel centroids in caller memory ------------------------------------------------------------------------------
int qb200_voxelize_batch_each(qb200_handle* h, const float* const* scans4, const int32_t* n_points, int32_t n_scans, const qb200_params* params,
                              qb200_mem_kind kind, const qb200_feature_out* out) {
  return run_call(h, raw_scans(Sink::Voxels, Entries::Mixed, scans4, n_points, n_scans, params, kind, nullptr, out));
}

int qb200_voxelize_batch_enqueue_each(qb200_handle* h, const float* const* scans4, const int32_t* n_points, int32_t n_scans,
                                      const qb200_params* params, qb200_mem_kind kind, const qb200_feature_out* out) {
  return enqueue_call(h, raw_scans(Sink::Voxels, Entries::Mixed, scans4, n_points, n_scans, params, kind, nullptr, out));
}

// ---- caller keypoint clouds -> normals and FPFH-33 in caller memory -------------------------------------------------------------
int qb200_describe_points_each(qb200_handle* h, const float* const* pts4, const int32_t* n_points, int32_t n_clouds, const qb200_params* params,
                               qb200_mem_kind kind, const qb200_feature_out* out) {
  return run_call(h, keypoint_clouds(Sink::Export, pts4, n_points, n_clouds, params, kind, out));
}

int qb200_describe_points_enqueue_each(qb200_handle* h, const float* const* pts4, const int32_t* n_points, int32_t n_clouds,
                                       const qb200_params* params, qb200_mem_kind kind, const qb200_feature_out* out) {
  return enqueue_call(h, keypoint_clouds(Sink::Export, pts4, n_points, n_clouds, params, kind, out));
}

// ---- raw, cached or caller-feature pairs -> correspondences and matched points, not solved --------------------------------------
int qb200_match_batch_mixed(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* params, qb200_mem_kind kind,
                            qb200_result* results, const qb200_pair_lists* lists) {
  return run_call(h, raw_pairs(Sink::Match, Entries::Mixed, pairs, n_pairs, params, kind, results, lists));
}

int qb200_match_batch_enqueue_mixed(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* params, qb200_mem_kind kind,
                                    qb200_result* results, const qb200_pair_lists* lists) {
  return enqueue_call(h, raw_pairs(Sink::Match, Entries::Mixed, pairs, n_pairs, params, kind, results, lists));
}

int qb200_match_cached_mixed(qb200_handle* h, const qb200_slot_pair* pairs, int32_t n_pairs, const qb200_params* params, qb200_result* results,
                             const qb200_pair_lists* lists) {
  return run_call(h, cached_pairs(Sink::Match, Entries::Mixed, pairs, n_pairs, params, results, lists));
}

int qb200_match_cached_enqueue_mixed(qb200_handle* h, const qb200_slot_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                     qb200_result* results, const qb200_pair_lists* lists) {
  return enqueue_call(h, cached_pairs(Sink::Match, Entries::Mixed, pairs, n_pairs, params, results, lists));
}

int qb200_match_features_each(qb200_handle* h, const qb200_feature_pair* pairs, int32_t n_pairs, const qb200_params* params,
                              qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists) {
  return run_call(h, feature_pairs(Sink::Match, pairs, n_pairs, params, kind, results, lists));
}

int qb200_match_features_enqueue_each(qb200_handle* h, const qb200_feature_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                      qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists) {
  return enqueue_call(h, feature_pairs(Sink::Match, pairs, n_pairs, params, kind, results, lists));
}

// ---- caller graphs -> maximum cliques ----------------------------------------------------------------------------------------------
int qb200_max_clique_batch_each(qb200_handle* h, const qb200_graph* graphs, int32_t n_graphs, const qb200_params* params, qb200_mem_kind kind,
                                qb200_result* results, const qb200_pair_lists* lists) {
  return run_call(h, caller_graphs(graphs, n_graphs, params, kind, results, lists));
}

int qb200_max_clique_batch_enqueue_each(qb200_handle* h, const qb200_graph* graphs, int32_t n_graphs, const qb200_params* params,
                                        qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists) {
  return enqueue_call(h, caller_graphs(graphs, n_graphs, params, kind, results, lists));
}

// ---- correspondence sets -> TIM graphs ---------------------------------------------------------------------------------------------
int qb200_build_graph_batch_each(qb200_handle* h, const qb200_corr_set* sets, int32_t n_sets, const qb200_params* params,
                                 qb200_mem_kind kind, qb200_result* results, const qb200_graph_out* out) {
  return run_call(h, corr_sets(sets, n_sets, params, kind, results, out));
}

int qb200_build_graph_batch_enqueue_each(qb200_handle* h, const qb200_corr_set* sets, int32_t n_sets, const qb200_params* params,
                                         qb200_mem_kind kind, qb200_result* results, const qb200_graph_out* out) {
  return enqueue_call(h, corr_sets(sets, n_sets, params, kind, results, out));
}

// ---- caller inlier sets -> poses ------------------------------------------------------------------------------------------------
int qb200_solve_pose_batch_each(qb200_handle* h, const qb200_inlier_set* sets, int32_t n_sets, const qb200_params* params,
                                qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists) {
  return run_call(h, inlier_sets(sets, n_sets, params, kind, results, lists));
}

int qb200_solve_pose_batch_enqueue_each(qb200_handle* h, const qb200_inlier_set* sets, int32_t n_sets, const qb200_params* params,
                                        qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists) {
  return enqueue_call(h, inlier_sets(sets, n_sets, params, kind, results, lists));
}

// ---- registered pairs -> aligned clouds, transformed matches and good matches in caller memory -------------------------------------
int qb200_align_batch_each(qb200_handle* h, const qb200_align_set* sets, int32_t n_sets, const qb200_params* params, qb200_mem_kind kind,
                           const qb200_align_out* out) {
  return run_call(h, align_sets(sets, n_sets, params, kind, out));
}

int qb200_align_batch_enqueue_each(qb200_handle* h, const qb200_align_set* sets, int32_t n_sets, const qb200_params* params,
                                   qb200_mem_kind kind, const qb200_align_out* out) {
  return enqueue_call(h, align_sets(sets, n_sets, params, kind, out));
}

int qb200_cache_copy(qb200_handle* h, int32_t from_slot, int32_t to_slot) {
  if (int rc = enter(h)) return rc;
  if (from_slot < 0 || to_slot < 0 || from_slot >= h->c_slots || to_slot >= h->c_slots) return QB200_ERR_BAD_ARG;
  if (from_slot == to_slot) return QB200_OK;
  const cudaStream_t st = h->lane[0]->stream;
  const size_t V = h->cfg.max_voxel_points;
  QB_CUDA_TRY(h, cudaMemcpyAsync(h->c_vox + to_slot * V, h->c_vox + from_slot * V, V * sizeof(float4), cudaMemcpyDeviceToDevice, st));
  QB_CUDA_TRY(h, cudaMemcpyAsync(h->c_nrm + to_slot * V, h->c_nrm + from_slot * V, V * sizeof(float4), cudaMemcpyDeviceToDevice, st));
  QB_CUDA_TRY(h, cudaMemcpyAsync(h->c_desc + to_slot * kDescK * V, h->c_desc + from_slot * kDescK * V, kDescK * V * sizeof(float), cudaMemcpyDeviceToDevice, st));
  QB_CUDA_TRY(h, cudaMemcpyAsync(h->c_n + to_slot, h->c_n + from_slot, sizeof(int), cudaMemcpyDeviceToDevice, st));
  QB_CUDA_TRY(h, cudaMemcpyAsync(h->c_status + to_slot, h->c_status + from_slot, sizeof(int), cudaMemcpyDeviceToDevice, st));
  memcpy(h->c_sig.get() + 4 * (size_t)to_slot, h->c_sig.get() + 4 * (size_t)from_slot, 4 * sizeof(float));
  QB_CUDA_TRY(h, cudaStreamSynchronize(st));
  return QB200_OK;
}

int qb200_cache_read(qb200_handle* h, int32_t slot, float* vox4, float* normals4, float* desc33, int32_t cap, int32_t* n_out) {
  if (int rc = enter(h)) return rc;
  if (!n_out || slot < 0 || slot >= h->c_slots || cap < 0) return QB200_ERR_BAD_ARG;
  Lane* L = h->lane[0].get();
  int n = 0;
  QB_CUDA_TRY(h, cudaMemcpyAsync(&n, h->c_n + slot, sizeof(int), cudaMemcpyDeviceToHost, L->stream));
  QB_CUDA_TRY(h, cudaStreamSynchronize(L->stream));
  *n_out = n;
  const int m = n < cap ? n : cap;
  const size_t V = L->V;
  if (m > 0) {
    if (vox4) QB_CUDA_TRY(h, cudaMemcpyAsync(vox4, h->c_vox + slot * V, (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost, L->stream));
    if (normals4) QB_CUDA_TRY(h, cudaMemcpyAsync(normals4, h->c_nrm + slot * V, (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost, L->stream));
    if (desc33) {
      if (int rc = export_desc_rows(L, h->c_desc + slot * kDescK * V, h->c_n + slot, m)) return rc;
      QB_CUDA_TRY(h, cudaMemcpyAsync(desc33, L->aos_scratch, (size_t)m * kDescDim * sizeof(float), cudaMemcpyDeviceToHost, L->stream));
    }
    QB_CUDA_TRY(h, cudaStreamSynchronize(L->stream));
  }
  return n > cap ? QB200_CAPACITY_EXCEEDED : QB200_OK;
}

int qb200_get_kernel_ms(qb200_handle* h, float* ms, int32_t* launches, int32_t n) {
  if (!h || !ms || n < 0) return QB200_ERR_BAD_ARG;
  for (int i = 0; i < n && i < 2; ++i) {
    ms[i] = h->kernel_ms[i];
    if (launches) launches[i] = h->kernel_calls[i];
  }
  return QB200_OK;
}

}  // extern "C"

namespace qb {
// Prologue of every entry point that uses lane 0's buffers or stream: a handle, its device current, and no wave of
// qb200_register_batch_enqueue in flight any more (their records are completed first).
int enter(qb200_handle* h) {
  if (!h) return QB200_ERR_BAD_ARG;
  cudaSetDevice(h->cfg.device);
  return h->lanes_active ? batch_flush(h) : QB200_OK;
}

int collect_batch(qb200_handle* h, const qb200_result* dst) {
  cudaSetDevice(h->cfg.device);
  return collect_waves(h, dst);
}

bool device_array_of(const qb200_handle* h, const void* a, size_t align) {
  if (!a) return true;
  if ((uintptr_t)a % align) return false;
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, a) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return at.device == h->cfg.device && (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged);
}
}  // namespace qb
