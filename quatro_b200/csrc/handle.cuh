// handle.cuh -- the opaque qb200_handle and its lanes: one device, per lane one stream and the device workspaces for one wave of
// max_batch_slots pairs.  Replaces the reference's process-global state (function-local statics at
// include/quatro.hpp:53,64,469-470,660 and include/fpfh_manager.hpp:110) with per-handle state.
#pragma once
#include <string.h>

#include <initializer_list>
#include <memory>
#include <vector>

#include "common.cuh"
#include "owners.cuh"

namespace qb {

// K8's constants of one β = 2 noise_bound sqrt(cbar2) (graph.cu: graph_const)
struct GraphConst {
  float b2, hb2q, twob2, b4;   // beta^2, beta^2/4, 2 beta^2, beta^4 (fp32)
  float c1, c2, c3;            // q = c1 M |D| + (c2 M + c3) M
  float two_b2_slack;          // 2 beta^2 (1 + 1e-5): part of M
  double beta;
};

// K10/11's parameters of one pair (pose.cu)
struct PoseParams {
  double rot_noise_bound, cote_range, gnc_factor, cost_threshold;
  int max_iterations, cote_median, use_rot_inliers, use_RyRx;
  double RyRx[9];
};

// One pair's solver configuration, as K7..K11 read it from the lane's table (DESIGN §5.4): the matcher and solver fields of its
// qb200_params, resolved on the host.  mode == QB200_INLIER_NONE: the pair skips K8 / K9 and gets the identity clique.
struct PairSolve {
  GraphConst gc;
  PoseParams pp;
  double kcore_thr;
  long long node_limit;      // PMC_EXACT nodes (0 already resolved to QB200_DEFAULT_CLIQUE_NODE_LIMIT)
  int mode;                  // QB200_PMC_EXACT .. QB200_INLIER_NONE
  int use_tuple;             // K7's tuple test runs for this pair: use_tuple_test and tuple_scale != 0 (match_fields)
  float tuple_scale;
  int tuple_trials;          // trials per mutual correspondence
  unsigned long long seed;
};

// One cloud's front-end configuration, as K1..K5 read it from the lane's table d_front (DESIGN §5.4): the voxel and lattice fields of
// its qb200_params, resolved on the host by front_voxel / front_lattice.  A kernel loads its cloud's entry once, at its start.
struct CloudFront {
  float inv_leaf;            // 1 / voxel_size
  int skip_flagged;
  float inv_cell;            // 1 / lattice cell
  int mn, mf;                // lattice reach of the normal / FPFH radius, in cells
  float rn2, rf2;            // squared normal / FPFH radius
  int list_usable;           // K3 may read K2c's neighbour list (the normal neighbourhood is a subsequence of it)
};

struct PpScan;   // one scan's pre-processing entry (preprocess.cu)

// Where feature_import_kernel reads one cloud of a feature or descriptor wave (frontend.cu): n keypoints and n descriptor rows of
// `stride` floats, of which the first `dim` are the descriptor, in the caller's device memory or in the lane's staging areas;
// desc == nullptr: keypoints only (a describe-points wave, described by K2..K5).  The import writes the cloud's descriptors
// dimension-major, row d at out + d * ld: an FPFH-33 cloud into its block of desc_t (ld = V, fpfh_src), a cloud of another length
// into the lane's dd_buf, which nn_dim_kernel reads through this same table.
struct FeatureSrc {
  const float4* pts;
  const float* desc;
  float* out;
  int n, dim, stride, ld;
};

// What feature_export_kernel reads (frontend.cu): cloud c's voxel points, normals and dimension-major descriptors at c * V points
// (c * kDescK * V floats) past these pointers, and its count; status == nullptr: every cloud is written, else only the clouds whose
// front-end status is QB200_OK.  n_kept != nullptr (a voxelize wave): QB200_CAPACITY_EXCEEDED clouds are written too, and a
// QB200_ERR_VOXEL_OVERFLOW cloud reports n_kept[c], its kept raw points, and gets no entries here (passthrough_kernel writes them)
struct ExportSrc {
  const float4* vox;
  const float4* nrm;
  const float* desc;
  const int* n;
  const int* status;
  const int* n_kept;
};

// Where feature_export_kernel writes cloud c: c * stride keypoints past each array (nullptr = not asked for), at most cap of them; and,
// when counts / status are set, its reported count and status (a refused cloud: count 0, nothing written)
struct ExportDst {
  float4* vox;
  float4* nrm;
  float* desc;
  long long stride;
  int cap;
  int* counts;
  int* status;
  // the caller's arrays of qb200_feature_out from scan `first` on
  static ExportDst caller(const qb200_feature_out& o, long long first);
  // the requested arrays of o, placed in a staging block of n clouds of `cap` keypoints each (base == nullptr: only the size), with
  // counts and status behind them
  static size_t carve(unsigned char* base, int n, int cap, const qb200_feature_out& o, ExportDst* out);
};

// Where the import kernels of a graph wave read one caller graph (graph.cu): its edge list (n_edges {u, v} pairs, in the caller's
// device memory or the lane's staging; nullptr = none, or streamed in chunks after the wave's launch) or its adjacency rows (stride
// words apart, in the caller's device memory or already copied into the graph's slot of adj; nullptr = none), and its vertex count
struct GraphSrc {
  const int2* edges;
  const uint32_t* rows;
  long long n_edges;
  int L, stride;
};

// Where a graph wave's device-kind outputs go (graph.cu: graph_export_kernel): set g's rows at adj + g * rows_per_set * words_per_row
// and its degrees at degree + g * rows_per_set, from the wave's first set on (nullptr = not asked for)
struct GraphDst {
  uint32_t* adj;
  int* degree;
  long long rows_per_set;
  int words_per_row;
};

// Where inlier_import_kernel reads one caller inlier set's correspondence ids (pose.cu): n ids in the caller's device memory or in
// the lane's staging (corr_src, the set's slot)
struct InlierSrc {
  const int* ids;
  int n, pad;
};

// One set of an align wave (align.cu), as the host resolved it: where its cloud, keypoints and correspondences are read (the caller's
// device memory or the lane's staging), where its outputs go (the caller's device arrays from the set's first entry on, or the lane's
// staging; nullptr = not asked for) and how many entries each receives, rows 0..2 of its pose and its good-match threshold.  blk0:
// the set's first block of align_points_kernel.
struct AlignSrc {
  const float4* cloud;
  const float4* src_kp;
  const float4* tgt_kp;
  const int2* corr;
  float4* aligned;
  float4* matched;
  int* good_ids;
  float4* good;
  double T[12];              // T(r, c) at T[4 r + c]
  double thr;                // 3.0 * (double)voxel_size
  int n_points, n_src, n_tgt, n_corr;
  int cap_points, cap_corr;
  int blk0, pad;
};

// What a batch call reads (api.cu: BatchCall), per input: a pair of raw scans, a pair of cached scans (slots), a pair of caller
// keypoint clouds with their FPFH-33 rows, a pair of caller keypoint clouds with descriptor rows of any length, a correspondence set, one raw scan, one caller keypoint cloud, one caller graph, a
// correspondence set with the caller's inlier ids, or a registered pair to align (a cloud, keypoints, correspondences and a pose)
enum class Source { RawPairs, CachedPairs, FeaturePairs, DescriptorPairs, CorrSets, RawScans, KeypointClouds, Graphs, InlierSets, AlignSets };
// What a batch call produces: solved records (and lists), the matcher's records (and lists), cache slots, front-end features in
// caller memory, max-clique records (and clique lists), TIM graphs in caller memory (and records), or poses of given inlier sets
// (records and lists), or aligned clouds and good matches in caller memory.  The valid (source, sink) pairs:
//   RawPairs, CachedPairs, FeaturePairs,
//   DescriptorPairs                      x  Solve, Match   qb200_register_batch*, _cached*, _features*, _descriptors*; qb200_match_*
//   CorrSets                             x  Solve, Graph   qb200_solve_batch*, qb200_build_graph_batch*
//   RawScans                             x  CacheSlots     qb200_cache_scans*
//   RawScans, KeypointClouds             x  Export         qb200_describe_batch*, qb200_describe_points*
//   RawScans                             x  Voxels         qb200_voxelize_batch*
//   Graphs                               x  Clique         qb200_max_clique_batch*
//   InlierSets                           x  Pose           qb200_solve_pose_batch*
//   AlignSets                            x  AlignOut       qb200_align_batch*
// Voxels is Export without K2..K5: the voxel centroids alone, with qb200_voxelize's capacity and pass-through outputs
enum class Sink { Solve, Match, CacheSlots, Export, Voxels, Clique, Graph, Pose, AlignOut };

// One lane: a stream and every device buffer of DESIGN §4 for one wave of S pairs.  Lane 0 is created with the handle; batches
// of several waves rotate over up to 8 lanes, so the H2D copies and the latency-bound solver tail of one wave overlap the dense
// kernels of the others.  The lane owns its stream, buffers and events: deleting it releases them.
struct Lane {
  int S, R, V, Lc, W;        // slots, raw cap / cloud, voxel cap / cloud, corr cap / pair, words per adjacency row
  int NS;                    // match stripes per pair = V / kMatchTile
  int device;
  int n_sm;                  // multiprocessors of the device (grid size of the persistent kernels)
  int force_exact_match;     // 0 (default): tensor-core filter + exact evaluation; 1 (QB200_MATCH_EXACT=1): exact CUDA-core K6 only
  int tc_verify;             // 1 (QB200_TC_VERIFY=1): every batch is matched again by the exact K6 and compared (stats[4..5])
  int tc_prof;               // 1 (QB200_TC_PROF=1): tc_nn_kernel with clock64 accounting of every role's waits (stats[8..31])
  Stream own_stream;
  cudaStream_t stream;       // own_stream, or the caller's stream of qb200_set_stream (lane 0)
  char* err;                 // the handle's message buffer (qb200_last_error)
  int64_t launches;
  uint64_t waves;            // waves started on this lane (wave_reset): lane 0's count tells the getters whether slot 0 was reused

  // ---- wave description (host-known inputs) ----
  DeviceMem<const float4*> d_cloud_ptr; // [2S]
  DeviceMem<int> d_cloud_n;   // [2S]
  DeviceMem<int> d_raw_off;   // [2S+1] offsets into the concatenated sort arrays
  PinnedMem<const float4*> h_cloud_ptr; PinnedMem<int> h_cloud_n, h_raw_off;  // pinned mirrors
  DeviceMem<float4> raw_stage; // [2S*R] staging for host inputs
  DeviceMem<int> d_slot_of_cloud; PinnedMem<int> h_slot_of_cloud;  // [2S] cache slot of every cloud of the wave, and its pinned mirror
  DeviceMem<FeatureSrc> d_feat; PinnedMem<FeatureSrc> h_feat;  // [2S] where a feature wave's clouds are read, and its pinned mirror
  DeviceMem<GraphSrc> d_graph; PinnedMem<GraphSrc> h_graph;   // [S] where a graph wave's graphs are read, and its pinned mirror
  DeviceMem<InlierSrc> d_inl; PinnedMem<InlierSrc> h_inl;     // [S] where a pose wave's inlier ids are read, and its pinned mirror
  DeviceMem<AlignSrc> d_aln; PinnedMem<AlignSrc> h_aln;       // [S] an align wave's sets, and its pinned mirror
  DeviceMem<float> dd_buf; size_t dd_cap;  // a descriptor wave's clouds of other lengths than 33: dimension-major rows (FeatureSrc::out),
                                           // then host-kind rows staged packed; grown to the largest wave so far, allocated on first use
  DeviceMem<unsigned char> aln_stage;  // an align wave's host-kind correspondences and correspondence outputs, [S][Lc] of each
                                       // (AlignStage), allocated on first use
  int pend_w0, pend_np;       // wave in flight on this lane (pend_np == 0: none)
  unsigned pend_stages;      // ... the stage-time slots it reports (bit i: qb200_get_stage_ms slot i)
  Sink pend_sink;             // ... what wave_collect hands on for it: the fields below of its sink
  qb200_result* pend_dst;     // ... (Solve, Match, Clique, Graph, Pose) the caller's record array of its batch, nullptr for the other sinks
  bool pend_host_lists;       // ... (Solve, Match, Clique, Pose) its batch has host-kind lists, which wave_collect hands on from lst_stage
  qb200_pair_lists pend_lists; // ... and then a copy of their descriptor
  qb200_feature_out pend_out; // ... (Export, Voxels) a copy of its batch's output descriptor, whose counts and status (and, in host
                              // kind, entries) wave_collect hands on from exp_stage (and a Voxels wave's pass-through from raw_stage)
  qb200_graph_out pend_graph; // ... (Graph) a copy of its batch's output descriptor, whose host-kind arrays wave_collect writes
  qb200_align_out pend_align; // ... (AlignOut) a copy of its batch's output descriptor, whose counts, status and host-kind arrays
                              // wave_collect writes
  // ... and the cache slots it reads (cached pairs) or writes (CacheSlots), ascending and unique; empty: it does not touch the
  // cache.  A wave reads the cache only in its copy-in and writes it only in its copy-out, so other lanes order their conflicting
  // copies after those events (api.cu: cache_waits)
  std::vector<int> pend_slots;
  int pend_writes;
  Event ev_cache_in, ev_cache_out;

  // ---- sort workspace (voxel sort, then lattice sort) ----
  DeviceMem<uint64_t> key_a, key_b;  // [2S*max(R,V)]
  DeviceMem<uint32_t> val_a, val_b;  // [2S*max(R,V)]; val_a also holds the voxel sort's digit histograms
  DeviceMem<void> cub_temp; size_t cub_bytes;  // library radix sort of up to 2S*V items (lattice / norm sorts of clouds too large for sort.cu)
  DeviceMem<float> aos_scratch;  // [2*V*33] AoS descriptors handed out by qb200_compute_fpfh / _get_last_features / _cache_read

  // ---- front end ----
  DeviceMem<int> vox_start;   // [2S*(V+1)] position (in the sorted raw array) of each voxel's first point
  DeviceMem<float4> vox_pts;  // [2S*V] centroids, ascending (k,j,i)
  DeviceMem<uint64_t> cell_key; // [2S*V] occupied lattice cells, ascending
  DeviceMem<int> cell_start;  // [2S*(V+1)]
  DeviceMem<float4> normals;  // [2S*V]; a feature or describe-points wave stages host keypoints here (packed, [sum n]), and the
                              // import has read them before K3 writes the normals
  DeviceMem<float> spfh;      // [2S*V*36] rows padded to 36 floats; a feature wave stages host descriptors here (packed, [sum n][33])
  DeviceMem<uint32_t> nbr_list; // [2S][kNbrGlobalCap][V] fpfh_radius neighbour indices found by K2c (lattice order), read by K3..K5
  DeviceMem<int> nbr_cnt;     // [2S*V] neighbour count (self included); > kNbrGlobalCap: K5 walks the lattice itself
  DeviceMem<float> desc_t;    // [2S*40*V] FPFH, dimension-major per cloud (row d = bin d over all points; rows 33..39 zero)
  DeviceMem<float> desc_tiles; // [2S*(V/64)*3*2560] per 64-point block: centred TF32 hi | lo | exact fp32 images in the wgmma
                              // shared-memory operand layout (one bulk copy per column tile, one per 128-row stripe)
  DeviceMem<float> desc_norm; // [2S*V] squared norms (fp32 fma chain)
  DeviceMem<int> tc_fallback; // [S] 1 = too many exact ties for the filter to pay off: pair re-done by the exact fp32 kernel
  DeviceMem<unsigned long long> tc_stats; // [32] diagnostics, cumulative: [0..3] exact evaluations, tiles drained, 0 (unused), aborted stripes; [4..5] QB200_TC_VERIFY; [8..31] QB200_TC_PROF
  // ---- matching ----
  DeviceMem<unsigned long long> rowbest; // [S*V] packed (dist bits << 32 | tgt idx) per source point
  DeviceMem<unsigned long long> colpart; // [colpart_count()] tensor-core K6 scratch: class results [2][S][V] and the tile-max cache
                                         // ([S][V/64][2] 32-bit maxima of 32-column groups)
  DeviceMem<unsigned long long> colbest; // [S*V] packed (dist bits << 32 | src idx) per target point (the exact K6 atomicMins into it)
  DeviceMem<int> mut_i, mut_j; // [S*V] mutual NN list (larger-cloud idx, smaller-cloud idx)
  DeviceMem<unsigned char> mark; // [S*V] tuple-test survivors
  DeviceMem<int> partner;     // [S*V] tgt partner per source index (-1)
  DeviceMem<float> mean;      // [2S*4]
  DeviceMem<int> corr_src, corr_tgt; // [S*Lc]
  DeviceMem<float4> ma, mb;   // [S*Lc] matched points (src, tgt)
  // ---- graph / clique ----
  DeviceMem<uint32_t> adj, adjp; // [S*Lc*W] adjacency bits, and the same in (core, id)-rank space
  DeviceMem<int> deg;         // [S*Lc]
  DeviceMem<int> kcore, korder, rank_of, by_rank, kbin; // [S*(Lc+2)]
  DeviceMem<int> clique;      // [S*Lc] ascending ids
  DeviceMem<uint32_t> ex_stack, ex_pool; // PMC_EXACT scratch, allocated on first use: [min(S,64)*1024*W] candidate sets per level, [min(S,64)*2^17] list entries
  DeviceMem<int> ex_lvl;      // [2*min(S,64)*1024] list segment (begin | remaining) per level
  DeviceMem<unsigned short> ex_cur; // [min(S,64)*1024] clique under construction (ranks)
  DeviceMem<unsigned char> kcore_ws; // [S * kcore_ws_bytes(Lc)] k-core arrays of graphs above kKcoreSmemVerts vertices (Lc > kKcoreSmemVerts only)
  DeviceMem<unsigned short> chain_ws; // [S*8*Lc] descent chains of those graphs (Lc > kKcoreSmemVerts only)
  DeviceMem<unsigned char> pose_ws; // [S * pose_ws_bytes(Lc)] pose workspace of cliques above kPoseSmemClique members (Lc > kPoseSmemClique only)
  DeviceMem<int> final_inl;   // [S*Lc]
  DeviceMem<unsigned char> rot_mask, trans_mask; // [S*Lc]
  DeviceMem<PairSolve> d_solve; PinnedMem<PairSolve> h_solve;  // [S] solver table of the wave, and its pinned mirror (upload_solve copies it)
  DeviceMem<CloudFront> d_front; PinnedMem<CloudFront> h_front;  // [2S] front-end table of the wave, and its pinned mirror (upload_front)
  // ---- pre-processing (preprocess.cu), allocated on first use for the largest wave so far (pw_scans / ip_cap) ----
  DeviceMem<int> pp_cnt; PinnedMem<int> pp_hcnt;  // [2S][8] per-scan counts and status of a wave, and its pinned mirror
  DeviceMem<PpScan> d_pp; PinnedMem<PpScan> h_pp; // [2S] per-scan parameter table of a wave, and its pinned mirror (one H2D per wave)
  DeviceMem<int> pw_ints;     // [pw_scans] x (patch id / rank per point, per-patch counters and offsets)
  DeviceMem<float4> pw_out;   // [pw_scans][R] ground | non-ground
  int pw_scans;
  DeviceMem<void> ip_buf; size_t ip_cap;  // range-image scratch (per scan and pixel: winner, parent, size, range, row set, output)
  // ---- results ----
  DeviceMem<qb200_result> d_results; // [S]
  PinnedMem<qb200_result> h_results; // [S]
  PinnedMem<unsigned char> lst_stage; int lst_cap;  // host-kind pair lists, grown on first use: [S][lst_cap] entries of every list
                                                    // (ListDst::carve), written by pack_lists_kernel through the mapped address
  PinnedMem<unsigned char> exp_stage; size_t exp_bytes;  // a describe wave's counts and status, and in host kind its entries
                                                         // (ExportDst::carve over 2S clouds), written by feature_export_kernel through
                                                         // the mapped address; grown on first use
  WaveCounters ctr, hctr;     // the counter block, and the same layout over its pinned mirror (stage calls read it back whole)
  DeviceMem<int> ctr_block; PinnedMem<int> hctr_block; size_t ctr_ints;

  Event ev[9];                // stage boundaries of the last wave: start, h2d, voxel, fpfh, match, graph, clique, pose, d2h
  Event kev[4];               // [0,1] around match_stripe_kernel, [2,3] around tim_graph_kernel (last wave)
  int kev_armed[2];

  void fail(const char* file, int line, const char* msg) { snprintf(err, kErrLen, "%s:%d: %s", file, line, msg); }
  static constexpr int kErrLen = 512;

  // colpart: class-indexed column results [S][V], row results [S][V], then the tile-max cache ([S][V/64][2] u32) and two spare words
  size_t colpart_count() const { return (size_t)2 * S * V + (size_t)S * (V >> 7) * 2 + 2; }
  unsigned long long* colpart_col() const { return colpart; }
  unsigned long long* colpart_row() const { return colpart + (size_t)S * V; }
  unsigned* colpart_tile_cmax() const { return reinterpret_cast<unsigned*>(colpart + (size_t)2 * S * V); }
  // the duplicate-class tables K6 keeps in key_a once the norm sort is done with it: class of every rank [2S][V], then the unique
  // count of every cloud [2S]
  uint32_t* class_of() const { return reinterpret_cast<uint32_t*>(key_a.get()); }
  int* n_unique() const { return reinterpret_cast<int*>(class_of() + (size_t)2 * S * V); }
};

// The lists of lane 0's slot 0 that the single-pair getters hand out: correspondences and matched points, clique, final inliers,
// normals and descriptors (qb200_get_last_*), and the nearest-neighbour tables (qb200_debug_nn_tables)
enum LastList { kLastCorr, kLastClique, kLastFinal, kLastFeatures, kLastNn, kLastLists };

}  // namespace qb

struct qb200_handle {
  qb200_config cfg;
  char err[qb::Lane::kErrLen];
  std::unique_ptr<qb::Lane> lane[8];  // lane[0] is created with the handle, the others on first use
  int max_lanes;              // 1..8 (QB200_LANES, default 4)
  int timeline;               // 1 (QB200_TIMELINE=1): stage boundaries of every raw-scan wave on stderr
  int lanes_active, lane_cursor;  // lanes of the rotation in use (0 = nothing in flight), next lane = busy longest
  qb::Event ev_fork;
  qb::Stream copy_stream;     // host scans of a multi-wave batch cross PCIe on ONE stream, wave after wave (api.cu: wave_submit)
  qb::Event ev_copied;        // a wave's scans have arrived (recorded on the copy stream)

  // ---- scan cache (qb200_cache_*): front-end results of whole scans, resident on the device.  Waves of every lane read it (each
  // through its lane's slot table), and cache-write waves write it; qb200_cache_reserve / _copy flush first ----
  int c_slots;
  qb::DeviceMem<float4> c_vox, c_nrm;  // [slots*V]
  qb::DeviceMem<float> c_desc;         // [slots*40*V] dimension-major like desc_t
  qb::DeviceMem<int> c_n, c_status;    // [slots]
  std::unique_ptr<float[]> c_sig;      // host [slots*4]: (voxel, normal_r, fpfh_r, cell) a slot was computed with (set when the
                                       // write is queued, so the checks of the calls after it see the new signature)

  // ---- multi-GPU gather of the result records (comm.cu) ----
  void* comm;                 // ncclComm_t
  int comm_world, comm_rank, comm_cap;   // cap: records per rank the staging buffers hold
  qb::Stream comm_stream;
  qb::Event comm_done;
  qb::DeviceMem<qb200_result> d_send, d_recv;  // device staging
  qb::PinnedMem<qb200_result> h_send, h_recv;  // pinned host staging (h_recv is rank-major)
  int pend_gather_n;          // > 0: a deferred gather is in flight (records per rank)
  qb200_result* pend_gather_dst;
  int pipe_n, pipe_buf;       // pipelined rank mode: local batch queued, gather not started yet (records per rank, half of h_send)
  qb200_result* pipe_dst;

  // ---- state mirrored from the reference's statics ----
  double rot_noise_bound_latched;  // quatro.hpp:469-470 (0 = not latched yet)
  int last_n_corr, last_n_clique, last_n_final;  // slot 0 of the most recent single-pair call
  int last_match_n[2];        // source / target points of the most recent qb200_match (qb200_debug_nn_tables)
  // per list (qb::LastList): lane 0's wave count right after the most recent single-pair call that produced it.  Every later wave on
  // lane 0 rewrites slot 0's buffers but not the counts above, so a getter hands out its list only while the count is unchanged.
  uint64_t last_wave[qb::kLastLists];

  float stage_ms[8];
  float kernel_ms[2];
  int kernel_calls[2];

  void fail(const char* file, int line, const char* msg) { snprintf(err, sizeof(err), "%s:%d: %s", file, line, msg); }
};

namespace qb {

// Per-pair choice between shared memory and global scratch (clique.cu, pose.cu): a graph of up to kKcoreSmemVerts vertices keeps its
// k-core and clique arrays in shared memory, a clique of up to kPoseSmemClique members its pose workspace.  The layouts are sized
// for min(Lc, limit), so a wide handle launches with about the shared memory of an 8192 handle and its small pairs keep their arrays
// in shared memory.
constexpr int kKcoreSmemVerts = 8192;
constexpr int kPoseSmemClique = 4096;
constexpr int kCliqueWarps = 8;
// bin (int x (Lc + 2)) | deg, pos, vert, mrk (u16 x Lc) | nbl [4][Lc] u16, 16-byte aligned
__host__ __device__ inline size_t kcore_ws_bytes(int Lc) { return ((size_t)(Lc + 2) * 4 + (size_t)8 * Lc * 2 + 15) & ~(size_t)15; }
size_t pose_ws_bytes(int Lc);

// Stage launchers (each enqueues kernels on the lane's stream for clouds/pairs [0, n) of its current wave).  K1..K5 read every cloud's
// configuration from the lane's table d_front (upload_front), K7 every pair's tuple test from d_solve (upload_solve); launch_match
// launches the tuple test only when h_solve has a pair that runs it.
int launch_voxel(Lane* h, int n_clouds);
int launch_fpfh(Lane* h, int n_clouds);
// keep_w: the matched points keep their keypoints' w (caller keypoints of a feature wave); otherwise w = 1.  dims (a descriptor
// wave, kDimsFpfh | kDimsOther): which K6 the wave's pairs need, the FPFH-33 matcher (on the counts ctr.n_fpfh) and nn_dim_kernel
// (on the pairs whose d_feat entries have another length); 0: every pair is FPFH-33 and K6 reads ctr.n_vox.
constexpr int kDimsFpfh = 1, kDimsOther = 2;
int launch_match(Lane* h, int n_pairs, int keep_w, int dims = 0);
// A match wave's records (pairs [0, n), after launch_match), in place of the solver tail: the matcher's counters, status and flags
// from the counter block, and the values of a pair that was not solved
int launch_match_records(Lane* h, int n_pairs);
// a cloud's front-end entry: its voxel fields (frontend.cu), its lattice fields for these radii and this lattice cell (frontend.cu),
// or both (lattice_only: the lattice fields alone, the voxel fields zero) from p (api.cu)
void front_voxel(CloudFront* e, float leaf, int skip_flagged);
void front_lattice(CloudFront* e, float normal_radius, float fpfh_radius, float cell);
CloudFront front_entry(const qb200_params& p, bool lattice_only = false);
// the entries [0, n) of h_front to d_front on the lane's stream: one copy (h_front must stay as it is until the stream passed it)
int upload_front(Lane* h, int n);
void match_fields(PairSolve* e, const qb200_params& p);  // K7's fields of a pair's entry (match.cu)
// The solver stages read every pair's configuration from the lane's table d_solve (upload_solve): K8 skips the pairs in
// QB200_INLIER_NONE, K9 runs each pair in its own mode (the exact search only when the table has a PMC_EXACT pair: any_exact),
// iota_clique_kernel fills only the QB200_INLIER_NONE pairs.
int launch_graph(Lane* h, int n_pairs);
int launch_clique(Lane* h, int n_pairs, bool any_exact);
int launch_pose(Lane* h, int n_pairs);
int launch_fill_counters(Lane* h, int n_pairs, int have_frontend);
int launch_finalize_status(Lane* h, int n_pairs);
int launch_iota_clique(Lane* h, int n_pairs);
GraphConst graph_const(double noise_bound, double cbar2);
PoseParams pose_params(const qb200_params& p);  // p's rotation noise bound already resolved
PairSolve solve_entry(const qb200_params& p);   // the same, every matcher and solver field
// the entries [0, n) of h_solve to d_solve on the lane's stream: one copy (h_solve must stay as it is until the stream passed it)
int upload_solve(Lane* h, int n);
// Where pack_lists_kernel writes pair s's lists: each array (nullptr = not asked for) + s * stride entries, at most cap of them.
struct ListDst {
  int2* corr; float4* sm; float4* tm; int* clique; int* fin; unsigned char* rm; unsigned char* tmask;
  long long stride;
  int cap;
  // the caller's arrays from pair `first` on (stride = cap_per_pair)
  static ListDst caller(const qb200_pair_lists& d, long long first);
  // lists' arrays, placed in a staging block of S pairs of `cap` entries each (base == nullptr: only the size); only requested lists
  // get a non-null pointer
  static size_t carve(unsigned char* base, int S, int cap, const qb200_pair_lists& d, ListDst* out);
};
int launch_pack_lists(Lane* h, int n_pairs, const ListDst& dst);
// entries of a list of `count` entries that a pair's stride of `cap` receives (counts never exceed the lane's Lc)
__host__ __device__ inline int list_entries(int count, int Lc, int cap) {
  const int n = count < 0 ? 0 : count > Lc ? Lc : count;
  return n < cap ? n : cap;
}
// the FPFH-33 K6 of pairs [0, n), on the clouds' counts n_pts (ctr.n_vox, or ctr.n_fpfh in a descriptor wave: a pair with a count
// of 0 is skipped and its rowbest / colbest entries are left to nn_dim_kernel)
int launch_match_nn(Lane* h, int n_pairs, const int* n_pts);
int launch_match_exact(Lane* h, int n_pairs, const int* only, const int* n_pts);
// nn_dim_kernel's K6 of the pairs of a descriptor wave whose d_feat entries have another length than 33 (match.cu)
int launch_match_dim(Lane* h, int n_pairs);
int launch_tc_debug_tile(Lane* h, float* d_out);
int tc_footprint(Lane* h, int* out5);
// Clouds [0, n_clouds) of src to dst in one launch: keypoints, normals and 33-float descriptor rows (pcl::FPFHSignature33) of each
// cloud's first min(n, dst.cap) points.  max_n: a host bound of the entries any cloud writes (the launch's tile count).
int launch_feature_export(Lane* h, int n_clouds, const ExportSrc& src, const ExportDst& dst, int max_n);
// Voxelize waves, after launch_voxel: PCL's pass-through of every cloud [0, n_clouds) refused with QB200_ERR_VOXEL_OVERFLOW, its kept
// raw points (raw_point_kept) in input order.  dst != nullptr: the first `cap` of them at dst + c * stride (the caller's device array);
// dst == nullptr: all of them at raw_stage + raw_off[c], the cloud's own region (in place for host scans), from where wave_collect
// copies them to the caller's host array.
int launch_passthrough(Lane* h, int n_clouds, float4* dst, long long stride, int cap);
// the first min(*n, m) descriptor rows of one cloud (its dimension-major block desc, its count at the device address n) into aos_scratch
int export_desc_rows(Lane* h, const float* desc, const int* n, int m);
// Feature waves (api.cu: stage_features, frontend.cu): h_feat[0, n) holds every cloud's caller pointers and count.  stage_features
// copies host-kind inputs into the staging areas (inputs back to back in the caller's memory as one copy) and uploads the table, on
// stream cs; launch_feature_import then fills vox_pts, desc_t and n_vox on the lane's stream (after wave_reset).
int stage_features(Lane* L, int n_clouds, qb200_mem_kind kind, cudaStream_t cs);
int launch_feature_import(Lane* h, int n_clouds);
// the table entry of an FPFH-33 cloud: n rows of 33 floats (or none) into cloud c's block of desc_t
inline FeatureSrc fpfh_src(const Lane* L, int c, const float* pts4, const float* desc, int n) {
  return FeatureSrc{reinterpret_cast<const float4*>(pts4), desc, L->desc_t + (size_t)c * kDescK * L->V, n, kDescDim, kDescDim, L->V};
}
size_t sort_temp_bytes(int max_items);
void comm_release(qb200_handle* h);
int collect_batch(qb200_handle* h, const qb200_result* dst);  // api.cu: wait for every wave in flight that writes into dst[...]
// api.cu, shared with the single-pair entry points of stages.cu
int enter(qb200_handle* h);  // entry prologue: a handle, its device current, no enqueued batch in flight
// a caller's array of QB200_MEM_DEVICE kind: device or managed memory of the handle's device, `align`-byte aligned (nullptr passes)
bool device_array_of(const qb200_handle* h, const void* a, size_t align);
int wave_reset(Lane* L, int n_clouds);
int stage_raw(Lane* L, int ncl, qb200_mem_kind kind, cudaStream_t cs);
int launch_degree(Lane* h, int n_pairs);
// Graph waves (graph.cu): the adjacency of graphs [0, n) from the table d_graph into their slots of adj.  launch_row_import writes the
// L rows (ceil(L / 32) words each) of every graph: its caller rows with the bits at columns >= L cleared, or zeros for an edge list.
// launch_edge_import then sets both bits of every edge: of every graph whose table entry has edges (only < 0), or of the n edges at
// `edges` of graph `only` alone (a chunk of a host edge list).  launch_symmetry_check compares every 32 x 32 tile of a row graph
// with its transpose.  An invalid edge, an asymmetric pair of tiles or a diagonal bit gives the graph status QB200_ERR_BAD_ARG in
// ctr.cloud_status and the mode QB200_INLIER_NONE in d_solve, so that K9 skips it.  max_L: the largest L of the graphs (grid size).
int launch_row_import(Lane* h, int n_graphs, int max_L);
int launch_edge_import(Lane* h, int n_graphs, long long max_edges, int only, const int2* edges);
int launch_symmetry_check(Lane* h, int n_graphs, int max_L);
// a graph wave's records (graphs [0, n), after K9): status, L, edges, max core, clique size and flags; the rest as a match record
int launch_clique_records(Lane* h, int n_graphs);
// TIM graph waves (graph.cu), after launch_graph on sets [0, n): launch_graph_export writes every set's L rows (words ceil(L / 32) ..
// words_per_row - 1 as zero) and degrees to d.  launch_edge_offsets finds where each row's edges (i, j), j > i, start in its set's
// list (korder, Lc + 2 ints per set, is the scratch: K9 does not run in these waves).  launch_edge_emit then writes the edges whose
// list index lies in [e0, e1) at out + index - e0: of every set (only < 0; set g's window at out + g * out_stride) or of set `only`.
// launch_graph_records writes the records: status QB200_OK, L, n_edges, QB200_FLAG_LISTS_TRUNCATED past cap_edges (> 0: an edge list
// was asked for), the rest as a match record.
int launch_graph_export(Lane* h, int n_sets, const GraphDst& d);
int launch_edge_offsets(Lane* h, int n_sets);
int launch_edge_emit(Lane* h, int n_sets, int only, long long e0, long long e1, int2* out, long long out_stride);
int launch_graph_records(Lane* h, int n_sets, long long cap_edges);
// Pose waves (pose.cu): launch_inlier_import writes the ids of every set of the table d_inl into its slot of clique and their count
// into ctr.n_clique, and refuses a set with an id outside [0, n_corr): status QB200_ERR_BAD_ARG in ctr.cloud_status[set] and n_clique
// 0, so that pose_kernel reads no point through it.  After pose_kernel, launch_pose_records turns every refused set's record into a
// QB200_ERR_BAD_ARG record: valid 0, identity T, n_corr = L, the rest 0.
int launch_inlier_import(Lane* h, int n_sets);
int launch_pose_records(Lane* h, int n_sets);
// Align waves (align.cu), sets [0, n) of the table d_aln: launch_align_good checks every set's correspondence indices (a set with one
// outside [0, n_src) x [0, n_tgt) gets QB200_ERR_BAD_ARG in ctr.cloud_status and no output), writes the transformed source keypoints
// and the good matches, and their count into ctr.n_final.  launch_align_points then transforms the clouds of the sets it did not
// refuse; n_blocks: the blocks of every set (AlignSrc::blk0).
int launch_align_good(Lane* h, int n_sets);
int launch_align_points(Lane* h, int n_blocks, int n_sets);
constexpr int kAlignPts = 1024;  // points per block of align_points_kernel
// The lane's align staging (aln_stage), per set Lc entries of each array
struct AlignStage {
  int2* corr; float4* matched; float4* good; int* ids;
  static size_t bytes(int S, int Lc) { return (size_t)S * Lc * (sizeof(int2) + 2 * sizeof(float4) + sizeof(int)); }
  static AlignStage carve(unsigned char* base, int S, int Lc) {
    const size_t n = (size_t)S * Lc;
    AlignStage a;
    a.matched = reinterpret_cast<float4*>(base);
    a.good = a.matched + n;
    a.corr = reinterpret_cast<int2*>(a.good + n);
    a.ids = reinterpret_cast<int*>(a.corr + n);
    return a;
  }
};
// the checks every entry of a registering call passes; solver = false: the front-end and matcher fields only (a match call)
bool params_ok(const qb200_params* p, bool solver = true);
float lattice_cell(const qb200_params& p);
qb200_params resolve_params(qb200_handle* h, const qb200_params& p);
void set_last(qb200_handle* h, const qb200_result& r);
// the lists `lists` of lane 0's slot 0 are those of the single-pair call that just ended: the getters hand them out until lane 0
// starts another wave
void stamp_last(qb200_handle* h, std::initializer_list<LastList> lists);
// whether lane 0 has started no wave since `list` was stamped; if it has, the message for qb200_last_error
bool last_is_live(qb200_handle* h, LastList list);
// Raise a kernel's dynamic shared-memory opt-in to at least `bytes` on `device`.  The attribute is a property of the
// (function, device), not of a handle: handles of different capacities share it, so it is only ever raised (process-wide maximum).
cudaError_t ensure_dyn_smem(int device, const void* kernel, size_t bytes);
int sort_pairs(Lane* h, int n_items, int end_bit);
int launch_voxel_sort(Lane* h, int n_clouds, int idx_bits);
int launch_cloud_sort(Lane* h, int n_clouds, const int* n_items, int f1, int f2);

}  // namespace qb
