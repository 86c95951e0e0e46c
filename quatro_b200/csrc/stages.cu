// stages.cu -- the single-pair C-ABI: stage entry points, getters, debug hooks.  A stage call is a wave of one on lane 0 that runs the
// batch kernels: it enqueues uploads, counter writes, launches and ONE counter-block copy, and waits again only for counter-sized copies.
#include <math.h>
#include <vector>

#include "handle.cuh"

using namespace qb;

namespace {

// Lane L's counter block into its pinned mirror L->hctr, one copy and no wait: the counts are there after the stream's next sync.
int read_counters(Lane* L) {
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->hctr_block, L->ctr_block, L->ctr_ints * sizeof(int), cudaMemcpyDeviceToHost, L->stream));
  return QB200_OK;
}

// value into a slot of the mirror and from there into the same slot of the device block, no wait.  The copy reads the mirror
// when the stream reaches it, so the caller holds a MirrorHold across it.
int write_counter(Lane* L, int* host_slot, int value) {
  *host_slot = value;
  QB_CUDA_TRY(L, cudaMemcpyAsync(L->ctr_block + (host_slot - L->hctr_block), host_slot, sizeof(int), cudaMemcpyHostToDevice, L->stream));
  return QB200_OK;
}

// A call that has written the counter mirror returns only once lane L's stream is idle: a counter copy still pending would read
// the mirror after the next call has rewritten it.  sync() is the call's own wait; a return on an error waits in the destructor.
struct MirrorHold {
  Lane* L; bool idle = false;
  ~MirrorHold() { if (!idle) cudaStreamSynchronize(L->stream); }
  cudaError_t sync() { idle = true; return cudaStreamSynchronize(L->stream); }
};

// tc_stats[first, first + n) summed over the lanes (then zeroed on every lane if reset): the qb200_debug_* counter hooks
int read_tc_stats(qb200_handle* h, int first, int n, uint64_t* out, int reset) {
  if (int rc = enter(h)) return rc;
  if (!out) return QB200_ERR_BAD_ARG;
  for (int i = 0; i < n; ++i) out[i] = 0;
  for (const auto& L : h->lane) {
    if (!L) continue;
    uint64_t o[32];
    QB_CUDA_TRY(L, cudaStreamSynchronize(L->stream));
    QB_CUDA_TRY(L, cudaMemcpy(o, L->tc_stats + first, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    if (reset) QB_CUDA_TRY(L, cudaMemset(L->tc_stats + first, 0, n * sizeof(unsigned long long)));
    for (int i = 0; i < n; ++i) out[i] += o[i];
  }
  return QB200_OK;
}

}  // namespace

extern "C" {

// ---- stage: voxelize ----------------------------------------------------------------------------
int qb200_voxelize(qb200_handle* h, const float* pts4, int32_t n, float leaf, int32_t skip_flagged, float* out4, int32_t cap,
                   int32_t* n_out) {
  if (int rc = enter(h)) return rc;
  if (!n_out || n < 0 || (n > 0 && !pts4) || !(leaf > 0) || cap < 0 || (cap > 0 && !out4)) return QB200_ERR_BAD_ARG;
  *n_out = 0;
  Lane* L = h->lane[0].get();
  if (n > L->R) { h->fail(__FILE__, __LINE__, "n exceeds max_raw_points"); return QB200_ERR_BAD_ARG; }
  if (n == 0) return QB200_OK;
  int rc = wave_reset(L, 1);
  if (rc) return rc;
  L->h_cloud_ptr[0] = reinterpret_cast<const float4*>(pts4);
  L->h_cloud_n[0] = n;
  MirrorHold hold{L};
  front_voxel(&L->h_front[0], leaf, skip_flagged);  // a one-entry front-end table
  if ((rc = upload_front(L, 1)) || (rc = stage_raw(L, 1, QB200_MEM_HOST, L->stream))) return rc;
  if ((rc = launch_voxel(L, 1)) || (rc = read_counters(L))) return rc;
  QB_CUDA_TRY(h, hold.sync());
  const int nv = L->hctr.n_vox[0], st = L->hctr.cloud_status[0];
  if (st == QB200_ERR_VOXEL_OVERFLOW) {
    // [EXT] pcl::VoxelGrid: "leaf size is too small ... integer indices would overflow" -> output = input
    int m = 0;
    for (int i = 0; i < n; ++i) {
      const float* p = pts4 + 4 * (size_t)i;
      if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2])) || (skip_flagged && p[3] < 0.0f)) continue;
      if (m < cap) memcpy(out4 + 4 * (size_t)m, p, 4 * sizeof(float));
      ++m;
    }
    *n_out = m;
    return m > cap ? QB200_CAPACITY_EXCEEDED : QB200_ERR_VOXEL_OVERFLOW;
  }
  *n_out = nv;
  const int m = nv < cap ? nv : cap;
  if (m > 0) {
    QB_CUDA_TRY(h, cudaMemcpyAsync(out4, L->vox_pts, (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost, L->stream));
    QB_CUDA_TRY(h, cudaStreamSynchronize(L->stream));
  }
  return st == QB200_CAPACITY_EXCEEDED || nv > cap ? QB200_CAPACITY_EXCEEDED : QB200_OK;
}

// ---- stage: normals + FPFH ------------------------------------------------------------------------
int qb200_compute_fpfh(qb200_handle* h, const float* pts4, int32_t n, float normal_radius, float fpfh_radius, float grid_cell,
                       float* normals4, float* desc33) {
  if (int rc = enter(h)) return rc;
  if (n < 0 || (n > 0 && !pts4) || !(normal_radius > 0) || !(fpfh_radius > 0) || !(grid_cell > 0)) return QB200_ERR_BAD_ARG;
  if (normal_radius > fpfh_radius) return QB200_ERR_BAD_ARG;  // fpfh_manager.hpp:99-102
  if (n == 0) return QB200_OK;
  Lane* L = h->lane[0].get();
  if (n > L->V) { h->fail(__FILE__, __LINE__, "cloud exceeds max_voxel_points"); return QB200_ERR_BAD_ARG; }
  int rc = wave_reset(L, 1);
  if (rc) return rc;
  QB_CUDA_TRY(h, cudaMemcpyAsync(L->vox_pts, pts4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, L->stream));
  MirrorHold hold{L};
  front_lattice(&L->h_front[0], normal_radius, fpfh_radius, grid_cell);  // a one-entry front-end table
  if ((rc = write_counter(L, L->hctr.n_vox, n)) || (rc = upload_front(L, 1)) || (rc = launch_fpfh(L, 1))) return rc;
  if (normals4) QB_CUDA_TRY(h, cudaMemcpyAsync(normals4, L->normals, (size_t)n * sizeof(float4), cudaMemcpyDeviceToHost, L->stream));
  if (desc33) {
    if ((rc = export_desc_rows(L, L->desc_t, L->ctr.n_vox, n))) return rc;
    QB_CUDA_TRY(h, cudaMemcpyAsync(desc33, L->aos_scratch, (size_t)n * kDescDim * sizeof(float), cudaMemcpyDeviceToHost, L->stream));
  }
  QB_CUDA_TRY(h, hold.sync());
  stamp_last(h, {kLastFeatures});
  return QB200_OK;
}

// ---- stage: matching (both calls hand out pair 0's correspondences as qb200_get_last_correspondences does) ----------
int qb200_match(qb200_handle* h, const float* src4, int32_t n_src, const float* src_desc33, const float* tgt4, int32_t n_tgt,
                const float* tgt_desc33, const qb200_params* p, int32_t* corr, int32_t cap, int32_t* n_corr, int32_t* n_mutual) {
  if (int rc = enter(h)) return rc;
  if (!p || !n_corr || n_src < 0 || n_tgt < 0 || cap < 0) return QB200_ERR_BAD_ARG;
  if ((n_src > 0 && (!src4 || !src_desc33)) || (n_tgt > 0 && (!tgt4 || !tgt_desc33))) return QB200_ERR_BAD_ARG;
  if (!p->use_crosscheck) return QB200_ERR_UNSUPPORTED;
  *n_corr = 0;
  if (n_mutual) *n_mutual = 0;
  Lane* L = h->lane[0].get();
  if (n_src > L->V || n_tgt > L->V) { h->fail(__FILE__, __LINE__, "cloud exceeds max_voxel_points"); return QB200_ERR_BAD_ARG; }
  h->last_match_n[0] = h->last_match_n[1] = 0;
  h->last_n_corr = 0;
  stamp_last(h, {kLastCorr, kLastNn});
  if (n_src == 0 || n_tgt == 0) return QB200_OK;
  int rc = wave_reset(L, 2);
  if (rc) return rc;
  h->last_match_n[0] = n_src; h->last_match_n[1] = n_tgt;
  stamp_last(h, {kLastNn});
  MirrorHold hold{L};
  // the features as a feature wave of one pair imports them (the import writes the clouds' counts)
  L->h_feat[0] = fpfh_src(L, 0, src4, src_desc33, n_src);
  L->h_feat[1] = fpfh_src(L, 1, tgt4, tgt_desc33, n_tgt);
  if ((rc = stage_features(L, 2, QB200_MEM_HOST, L->stream)) || (rc = launch_feature_import(L, 2))) return rc;
  memset(&L->h_solve[0], 0, sizeof(PairSolve));  // a one-entry pair table: p's tuple test
  match_fields(&L->h_solve[0], *p);
  if ((rc = upload_solve(L, 1)) || (rc = launch_match(L, 1, 0)) || (rc = read_counters(L))) return rc;
  QB_CUDA_TRY(h, hold.sync());
  if (n_mutual) *n_mutual = L->hctr.n_mutual[0];
  h->last_n_corr = L->hctr.n_corr[0];
  stamp_last(h, {kLastCorr});
  if ((rc = qb200_get_last_correspondences(h, corr, nullptr, nullptr, cap, n_corr))) return rc;
  return L->hctr.cloud_status[0] == QB200_CAPACITY_EXCEEDED ? QB200_CAPACITY_EXCEEDED : QB200_OK;
}

int qb200_match_and_pack(qb200_handle* h, const float* src4, int32_t n_src, const float* tgt4, int32_t n_tgt, const qb200_params* p,
                         int32_t* corr, float* src_matched4, float* tgt_matched4, int32_t cap, int32_t* n_corr) {
  if (int rc = enter(h)) return rc;
  if (!n_corr || !params_ok(p) || n_src < 0 || n_tgt < 0 || cap < 0) return QB200_ERR_BAD_ARG;
  if (!p->use_crosscheck) return QB200_ERR_UNSUPPORTED;
  *n_corr = 0;
  Lane* L = h->lane[0].get();
  if (n_src > L->V || n_tgt > L->V) { h->fail(__FILE__, __LINE__, "cloud exceeds max_voxel_points"); return QB200_ERR_BAD_ARG; }
  if (n_src == 0 || n_tgt == 0) return QB200_OK;
  int rc = wave_reset(L, 2);
  if (rc) return rc;
  QB_CUDA_TRY(h, cudaMemcpyAsync(L->vox_pts, src4, (size_t)n_src * sizeof(float4), cudaMemcpyHostToDevice, L->stream));
  QB_CUDA_TRY(h, cudaMemcpyAsync(L->vox_pts + L->V, tgt4, (size_t)n_tgt * sizeof(float4), cudaMemcpyHostToDevice, L->stream));
  MirrorHold hold{L};
  if ((rc = write_counter(L, L->hctr.n_vox, n_src)) || (rc = write_counter(L, L->hctr.n_vox + 1, n_tgt))) return rc;
  L->h_front[0] = L->h_front[1] = front_entry(*p);  // one-entry tables: p's front end and tuple test
  memset(&L->h_solve[0], 0, sizeof(PairSolve));
  match_fields(&L->h_solve[0], *p);
  if ((rc = upload_front(L, 2)) || (rc = upload_solve(L, 1)) || (rc = launch_fpfh(L, 2))) return rc;
  if ((rc = launch_match(L, 1, 0)) || (rc = read_counters(L))) return rc;
  QB_CUDA_TRY(h, hold.sync());
  h->last_n_corr = L->hctr.n_corr[0];
  stamp_last(h, {kLastCorr, kLastFeatures});
  if ((rc = qb200_get_last_correspondences(h, corr, src_matched4, tgt_matched4, cap, n_corr))) return rc;
  return L->hctr.cloud_status[0] == QB200_CAPACITY_EXCEEDED ? QB200_CAPACITY_EXCEEDED : QB200_OK;
}

// ---- stage: graph ---------------------------------------------------------------------------------
int qb200_build_graph(qb200_handle* h, const float* a4, const float* b4, int32_t L, double noise_bound, double cbar2, uint32_t* adj,
                      int32_t words_per_row, int32_t* degree, int64_t* n_edges) {
  if (int rc = enter(h)) return rc;
  if (L < 0 || (L > 0 && (!a4 || !b4 || !adj)) || words_per_row < (L + 31) / 32 || !(noise_bound > 0) || !(cbar2 > 0))
    return QB200_ERR_BAD_ARG;
  if (n_edges) *n_edges = 0;
  if (L == 0) return QB200_OK;
  Lane* ln = h->lane[0].get();
  if (L > ln->Lc) { h->fail(__FILE__, __LINE__, "L exceeds max_corr"); return QB200_ERR_BAD_ARG; }
  int rc = wave_reset(ln, 2);
  if (rc) return rc;
  QB_CUDA_TRY(h, cudaMemcpyAsync(ln->ma, a4, (size_t)L * sizeof(float4), cudaMemcpyHostToDevice, ln->stream));
  QB_CUDA_TRY(h, cudaMemcpyAsync(ln->mb, b4, (size_t)L * sizeof(float4), cudaMemcpyHostToDevice, ln->stream));
  MirrorHold hold{ln};
  // a one-entry solver table: this beta (the mode only has to be one that builds a graph)
  memset(&ln->h_solve[0], 0, sizeof(PairSolve));
  ln->h_solve[0].gc = graph_const(noise_bound, cbar2);
  ln->h_solve[0].mode = QB200_PMC_HEU;
  if ((rc = write_counter(ln, ln->hctr.n_corr, L)) || (rc = upload_solve(ln, 1)) || (rc = launch_graph(ln, 1))) return rc;
  const int nb = (L + 31) / 32;
  memset(adj, 0, (size_t)L * words_per_row * sizeof(uint32_t));
  QB_CUDA_TRY(h, cudaMemcpy2DAsync(adj, (size_t)words_per_row * 4, ln->adj, (size_t)ln->W * 4, (size_t)nb * 4, L, cudaMemcpyDeviceToHost, ln->stream));
  if (degree) QB_CUDA_TRY(h, cudaMemcpyAsync(degree, ln->deg, (size_t)L * sizeof(int), cudaMemcpyDeviceToHost, ln->stream));
  if ((rc = read_counters(ln))) return rc;
  QB_CUDA_TRY(h, hold.sync());
  if (n_edges) *n_edges = *ln->hctr.n_edges / 2;
  return QB200_OK;
}

// ---- stage: max clique ------------------------------------------------------------------------------
int qb200_max_clique_ex(qb200_handle* h, const uint32_t* adj, int32_t L, int32_t words_per_row, int32_t mode, double kcore_thr,
                        int64_t node_limit, int32_t* clique, int32_t* n_clique, int32_t* kcore, int32_t* kcore_order, int32_t* max_core,
                        int32_t* flags) {
  if (int rc = enter(h)) return rc;
  if (!n_clique || L < 0 || (L > 0 && (!adj || !clique)) || words_per_row < (L + 31) / 32) return QB200_ERR_BAD_ARG;
  if (mode != QB200_PMC_EXACT && mode != QB200_PMC_HEU && mode != QB200_KCORE_HEU) return QB200_ERR_BAD_ARG;
  if (node_limit < 0) return QB200_ERR_BAD_ARG;
  if (flags) *flags = 0;
  *n_clique = 0;
  if (max_core) *max_core = 0;
  Lane* ln = h->lane[0].get();
  if (L > ln->Lc) { h->fail(__FILE__, __LINE__, "L exceeds max_corr"); return QB200_ERR_BAD_ARG; }
  if (L == 0) return QB200_OK;
  int rc = wave_reset(ln, 2);
  if (rc) return rc;
  const int nb = (L + 31) / 32;
  QB_CUDA_TRY(h, cudaMemsetAsync(ln->adj, 0, (size_t)L * ln->W * 4, ln->stream));
  QB_CUDA_TRY(h, cudaMemcpy2DAsync(ln->adj, (size_t)ln->W * 4, adj, (size_t)words_per_row * 4, (size_t)nb * 4, L, cudaMemcpyHostToDevice, ln->stream));
  MirrorHold hold{ln};
  memset(&ln->h_solve[0], 0, sizeof(PairSolve));  // a one-entry solver table: this mode, threshold and node limit
  ln->h_solve[0].mode = mode;
  ln->h_solve[0].kcore_thr = kcore_thr;
  ln->h_solve[0].node_limit = node_limit > 0 ? node_limit : (long long)QB200_DEFAULT_CLIQUE_NODE_LIMIT;
  // the rows just copied, masked in place like a batch graph's host rows: bits at columns >= L are ignored
  ln->h_graph[0] = GraphSrc{nullptr, ln->adj, 0, L, ln->W};
  QB_CUDA_TRY(h, cudaMemcpyAsync(ln->d_graph, ln->h_graph, sizeof(GraphSrc), cudaMemcpyHostToDevice, ln->stream));
  if ((rc = write_counter(ln, ln->hctr.n_corr, L)) || (rc = upload_solve(ln, 1)) || (rc = launch_row_import(ln, 1, L)) ||
      (rc = launch_degree(ln, 1)))
    return rc;
  if ((rc = launch_clique(ln, 1, mode == QB200_PMC_EXACT)) || (rc = read_counters(ln))) return rc;
  QB_CUDA_TRY(h, hold.sync());
  const int nc = ln->hctr.n_clique[0];
  if (flags) *flags = ln->hctr.flags[0];
  *n_clique = nc;
  if (max_core) *max_core = ln->hctr.max_core[0];
  if (nc > 0) QB_CUDA_TRY(h, cudaMemcpyAsync(clique, ln->clique, (size_t)nc * sizeof(int), cudaMemcpyDeviceToHost, ln->stream));
  if (kcore) QB_CUDA_TRY(h, cudaMemcpyAsync(kcore, ln->kcore, (size_t)L * sizeof(int), cudaMemcpyDeviceToHost, ln->stream));
  if (kcore_order) QB_CUDA_TRY(h, cudaMemcpyAsync(kcore_order, ln->korder, (size_t)L * sizeof(int), cudaMemcpyDeviceToHost, ln->stream));
  QB_CUDA_TRY(h, cudaStreamSynchronize(ln->stream));
  h->last_n_clique = nc;
  stamp_last(h, {kLastClique});
  return QB200_OK;
}

int qb200_max_clique(qb200_handle* h, const uint32_t* adj, int32_t L, int32_t words_per_row, int32_t mode, double kcore_thr,
                     int32_t* clique, int32_t* n_clique, int32_t* kcore, int32_t* kcore_order, int32_t* max_core) {
  return qb200_max_clique_ex(h, adj, L, words_per_row, mode, kcore_thr, 0, clique, n_clique, kcore, kcore_order, max_core, nullptr);
}

// ---- stage: pose given the clique -------------------------------------------------------------------
int qb200_solve_pose(qb200_handle* h, const float* a4, const float* b4, int32_t L, const int32_t* clique, int32_t n_clique,
                     const qb200_params* p, qb200_result* res, uint8_t* rot_inlier_mask, uint8_t* trans_inlier_mask) {
  if (int rc = enter(h)) return rc;
  if (!res || !params_ok(p) || L < 0 || (L > 0 && (!a4 || !b4)) || n_clique < 0 || n_clique > L || (n_clique > 0 && !clique))
    return QB200_ERR_BAD_ARG;
  Lane* ln = h->lane[0].get();
  if (L > ln->Lc) { h->fail(__FILE__, __LINE__, "L exceeds max_corr"); return QB200_ERR_BAD_ARG; }
  // pose_kernel reads a4[clique[j]] / b4[clique[j]] unchecked: an entry outside [0, L) would read past the pair's points
  for (int j = 0; j < n_clique; ++j)
    if (clique[j] < 0 || clique[j] >= L) { h->fail(__FILE__, __LINE__, "clique entry outside [0, L)"); return QB200_ERR_BAD_ARG; }
  int rc = wave_reset(ln, 2);
  if (rc) return rc;
  if (L > 0) QB_CUDA_TRY(h, cudaMemcpyAsync(ln->ma, a4, (size_t)L * sizeof(float4), cudaMemcpyHostToDevice, ln->stream));
  if (L > 0) QB_CUDA_TRY(h, cudaMemcpyAsync(ln->mb, b4, (size_t)L * sizeof(float4), cudaMemcpyHostToDevice, ln->stream));
  if (n_clique > 0) QB_CUDA_TRY(h, cudaMemcpyAsync(ln->clique, clique, (size_t)n_clique * sizeof(int), cudaMemcpyHostToDevice, ln->stream));
  MirrorHold hold{ln};
  if ((rc = write_counter(ln, ln->hctr.n_corr, L)) || (rc = write_counter(ln, ln->hctr.n_clique, n_clique))) return rc;
  ln->h_solve[0] = solve_entry(resolve_params(h, *p));
  if ((rc = upload_solve(ln, 1)) || (rc = launch_fill_counters(ln, 1, 0)) || (rc = launch_pose(ln, 1))) return rc;
  QB_CUDA_TRY(h, cudaMemcpyAsync(ln->h_results, ln->d_results, sizeof(qb200_result), cudaMemcpyDeviceToHost, ln->stream));
  QB_CUDA_TRY(h, hold.sync());
  *res = ln->h_results[0];
  set_last(h, *res);
  stamp_last(h, {kLastClique, kLastFinal});  // the points are the caller's: no correspondences were packed
  if (res->status < 0) return res->status;
  if (res->valid) {
    const int nc = res->clique_size;
    if (rot_inlier_mask) QB_CUDA_TRY(h, cudaMemcpyAsync(rot_inlier_mask, ln->rot_mask, (size_t)nc, cudaMemcpyDeviceToHost, ln->stream));
    if (trans_inlier_mask) QB_CUDA_TRY(h, cudaMemcpyAsync(trans_inlier_mask, ln->trans_mask, (size_t)nc, cudaMemcpyDeviceToHost, ln->stream));
    QB_CUDA_TRY(h, cudaStreamSynchronize(ln->stream));
  }
  return res->status;
}

// ---- Quatro::computeTransformation: a qb200_solve_batch of one set ------------------------------------
int qb200_solve_correspondences(qb200_handle* h, const float* a4, const float* b4, int32_t L, const qb200_params* p, qb200_result* res) {
  if (!res) return QB200_ERR_BAD_ARG;
  const qb200_corr_set set = {a4, b4, L, 0};
  const int rc = qb200_solve_batch(h, &set, 1, p, QB200_MEM_HOST, res);
  if (rc != QB200_OK) return rc;
  return res->status;
}

// ---- introspection ----------------------------------------------------------------------------------
// Slot 0 of lane 0 holds a single-pair call's lists only until the next wave on lane 0 rewrites it.  Each getter hands out its list
// only if the most recent single-pair call that produced it was also the last call to run a wave on lane 0 (stamp_last); otherwise
// it refuses (QB200_ERR_BAD_ARG, n = 0) rather than pair that call's count with another wave's entries.
int qb200_get_last_clique(qb200_handle* h, int32_t* idx, int32_t cap, int32_t* n) {
  if (int rc = enter(h)) return rc;
  if (!n || cap < 0) return QB200_ERR_BAD_ARG;
  Lane* L = h->lane[0].get();
  *n = 0;
  if (!last_is_live(h, kLastClique)) return QB200_ERR_BAD_ARG;
  *n = h->last_n_clique;
  const int m = *n < cap ? *n : cap;
  if (m > 0 && idx) {
    QB_CUDA_TRY(h, cudaMemcpyAsync(idx, L->clique, (size_t)m * sizeof(int), cudaMemcpyDeviceToHost, L->stream));
    QB_CUDA_TRY(h, cudaStreamSynchronize(L->stream));
  }
  return *n > cap ? QB200_CAPACITY_EXCEEDED : QB200_OK;
}

int qb200_get_last_final_inliers(qb200_handle* h, int32_t* idx, int32_t cap, int32_t* n) {
  if (int rc = enter(h)) return rc;
  if (!n || cap < 0) return QB200_ERR_BAD_ARG;
  Lane* L = h->lane[0].get();
  *n = 0;
  if (!last_is_live(h, kLastFinal)) return QB200_ERR_BAD_ARG;
  *n = h->last_n_final;
  const int m = *n < cap ? *n : cap;
  if (m > 0 && idx) {
    QB_CUDA_TRY(h, cudaMemcpyAsync(idx, L->final_inl, (size_t)m * sizeof(int), cudaMemcpyDeviceToHost, L->stream));
    QB_CUDA_TRY(h, cudaStreamSynchronize(L->stream));
  }
  return *n > cap ? QB200_CAPACITY_EXCEEDED : QB200_OK;
}

// the first min(n, cap) correspondences of pair 0: index pairs (src, tgt) and matched points, any of them may be NULL
int qb200_get_last_correspondences(qb200_handle* h, int32_t* corr, float* src_matched4, float* tgt_matched4, int32_t cap, int32_t* n) {
  if (int rc = enter(h)) return rc;
  if (!n || cap < 0) return QB200_ERR_BAD_ARG;
  Lane* L = h->lane[0].get();
  *n = 0;
  if (!last_is_live(h, kLastCorr)) return QB200_ERR_BAD_ARG;
  *n = h->last_n_corr;
  const int m = *n < cap ? *n : cap;
  if (m > 0) {
    std::vector<int> s(m), t(m);
    QB_CUDA_TRY(h, cudaMemcpyAsync(s.data(), L->corr_src, (size_t)m * sizeof(int), cudaMemcpyDeviceToHost, L->stream));
    QB_CUDA_TRY(h, cudaMemcpyAsync(t.data(), L->corr_tgt, (size_t)m * sizeof(int), cudaMemcpyDeviceToHost, L->stream));
    if (src_matched4) QB_CUDA_TRY(h, cudaMemcpyAsync(src_matched4, L->ma, (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost, L->stream));
    if (tgt_matched4) QB_CUDA_TRY(h, cudaMemcpyAsync(tgt_matched4, L->mb, (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost, L->stream));
    QB_CUDA_TRY(h, cudaStreamSynchronize(L->stream));
    if (corr)
      for (int i = 0; i < m; ++i) { corr[2 * i] = s[i]; corr[2 * i + 1] = t[i]; }
  }
  return *n > cap ? QB200_CAPACITY_EXCEEDED : QB200_OK;
}

int qb200_get_last_features(qb200_handle* h, int32_t which, float* normals4, float* desc33, int32_t cap, int32_t* n_out) {
  if (int rc = enter(h)) return rc;
  if (!n_out || which < 0 || which > 1 || cap < 0) return QB200_ERR_BAD_ARG;
  Lane* L = h->lane[0].get();
  *n_out = 0;
  if (!last_is_live(h, kLastFeatures)) return QB200_ERR_BAD_ARG;
  if (int rc = read_counters(L)) return rc;
  QB_CUDA_TRY(h, cudaStreamSynchronize(L->stream));
  const int n = L->hctr.n_vox[which];
  *n_out = n;
  const int m = n < cap ? n : cap;
  if (m > 0) {
    if (normals4) QB_CUDA_TRY(h, cudaMemcpyAsync(normals4, L->normals + (size_t)which * L->V, (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost, L->stream));
    if (desc33) {
      if (int rc = export_desc_rows(L, L->desc_t + (size_t)which * kDescK * L->V, L->ctr.n_vox + which, m)) return rc;
      QB_CUDA_TRY(h, cudaMemcpyAsync(desc33, L->aos_scratch, (size_t)m * kDescDim * sizeof(float), cudaMemcpyDeviceToHost, L->stream));
    }
    QB_CUDA_TRY(h, cudaStreamSynchronize(L->stream));
  }
  return n > cap ? QB200_CAPACITY_EXCEEDED : QB200_OK;
}

// QB200_TC_VERIFY=1: every batch is matched by BOTH K6 implementations and the packed (distance, index) results are compared;
// out2[0] = nearest-neighbour entries compared, out2[1] = entries that differ (must stay 0: the tensor-core filter is exact).
int qb200_debug_match_verify(qb200_handle* h, uint64_t* out2, int32_t reset) { return read_tc_stats(h, 4, 2, out2, reset); }

// QB200_TC_PROF=1: clock64 accounting of tc_nn_kernel's roles (cycles summed over CTAs / warps), stats[8..31] -> out24
int qb200_debug_tc_profile(qb200_handle* h, uint64_t* out24, int32_t reset) { return read_tc_stats(h, 8, 24, out24, reset); }

int qb200_debug_match_stats(qb200_handle* h, uint64_t* out4, int32_t reset) { return read_tc_stats(h, 0, 4, out4, reset); }

// Nearest-neighbour tables of the most recent qb200_match or one-pair qb200_match_descriptors_each (pair 0 of the handle, point
// order): what match_mutual_kernel read
int qb200_debug_nn_tables(qb200_handle* h, uint64_t* rowbest, int32_t cap_rows, uint64_t* colbest, int32_t cap_cols) {
  if (int rc = enter(h)) return rc;
  if (cap_rows < 0 || cap_cols < 0) return QB200_ERR_BAD_ARG;
  Lane* L = h->lane[0].get();
  if (!last_is_live(h, kLastNn)) return QB200_ERR_BAD_ARG;
  QB_CUDA_TRY(h, cudaStreamSynchronize(L->stream));
  const int nr = cap_rows < h->last_match_n[0] ? cap_rows : h->last_match_n[0];
  const int nc = cap_cols < h->last_match_n[1] ? cap_cols : h->last_match_n[1];
  if (rowbest && nr > 0) QB_CUDA_TRY(h, cudaMemcpy(rowbest, L->rowbest, (size_t)nr * 8, cudaMemcpyDeviceToHost));
  if (colbest && nc > 0) QB_CUDA_TRY(h, cudaMemcpy(colbest, L->colbest, (size_t)nc * 8, cudaMemcpyDeviceToHost));
  return QB200_OK;
}

// Footprint of the tensor-core nearest-neighbour kernel as it is launched: out5 = threads per CTA, dynamic and static shared
// bytes, registers per thread, resident CTAs per SM (occupancy calculator at that shared-memory size)
int qb200_debug_tc_footprint(qb200_handle* h, int32_t* out5) {
  if (!h || !out5) return QB200_ERR_BAD_ARG;
  cudaSetDevice(h->cfg.device);
  return tc_footprint(h->lane[0].get(), out5);
}

// Validation hook: tensor-core (3xTF32) approximate squared distances between up to 128 source and 128 target
// descriptors -> out[128*128] (row = source).  Lets tests measure the filter's error against the exact chain.
int qb200_debug_tc_distances(qb200_handle* h, const float* a33, int32_t na, const float* b33, int32_t nb, float* out) {
  if (int rc = enter(h)) return rc;
  if (!a33 || !b33 || !out || na < 1 || nb < 1 || na > 128 || nb > 128) return QB200_ERR_BAD_ARG;
  Lane* L = h->lane[0].get();
  int rc = wave_reset(L, 2);
  if (rc) return rc;
  MirrorHold hold{L};
  // the descriptors as a feature wave imports them, without keypoints: the import's staging is in spfh, which
  // the stream has passed before the memset below reuses it
  L->h_feat[0] = fpfh_src(L, 0, nullptr, a33, na);
  L->h_feat[1] = fpfh_src(L, 1, nullptr, b33, nb);
  if ((rc = stage_features(L, 2, QB200_MEM_HOST, L->stream)) || (rc = launch_feature_import(L, 2))) return rc;
  float* d_out = L->spfh;  // not the sort scratch: K6 sorts the descriptors by norm first
  QB_CUDA_TRY(h, cudaMemsetAsync(d_out, 0, 128 * 128 * sizeof(float), L->stream));
  if ((rc = launch_tc_debug_tile(L, d_out))) return rc;
  QB_CUDA_TRY(h, cudaMemcpyAsync(out, d_out, 128 * 128 * sizeof(float), cudaMemcpyDeviceToHost, L->stream));
  QB_CUDA_TRY(h, hold.sync());
  return QB200_OK;
}

}  // extern "C"
