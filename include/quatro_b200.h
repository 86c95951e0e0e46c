/*
 * quatro_b200.h -- C-ABI of the H100-native (sm_90a) global-registration hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  Every entry point replaces one stage
 * boundary of the reference (url-kaist/Quatro, paths relative to the reference root):
 *
 *   qb200_patchwork             <- PatchWork<PointT>::estimate_ground   include/patchwork.hpp:329-455 (pre-processing, 8f-1)
 *   qb200_segment_cloud         <- ImageProjection::segmentCloud        include/imageProjection.hpp:273-294 (pre-processing, 8f-1)
 *   qb200_voxelize              <- voxelize<T>()                    include/quatro.hpp:49-57
 *   qb200_compute_fpfh          <- FPFHEstimation::computeFPFHFeatures  src/teaser_utils/fpfh.cc:44-75
 *   qb200_match                 <- Matcher::calculateCorrespondences    include/teaser_utils/feature_matcher.h:42-74
 *                                  + Matcher::advancedMatching          src/teaser_utils/feature_matcher.cc:77-265
 *   qb200_build_graph           <- Quatro::computeTIMs + solveForScale + inlier_graph_.addEdge loop
 *                                  include/quatro.hpp:307-386, 784-789
 *   qb200_max_clique            <- teaser::MaxCliqueSolver::findMaxClique   src/graph.cc:12-130
 *   qb200_solve_pose            <- chain TIMs + GNC-TLS yaw + COTE      include/quatro.hpp:817-936
 *   qb200_solve_correspondences <- Quatro::computeTransformation(Eigen::Matrix4d&)  include/quatro.hpp:769-936
 *   qb200_match_and_pack        <- FPFHManager::setFeaturePair          include/fpfh_manager.hpp:98-153
 *   qb200_register_pair/_batch  <- examples/run_global_registration.cpp:206-246 (voxelize .. computeTransformation)
 *   qb200_register_batch_sharded / _rank  <- the same loop over a list of pairs, sharded over the GPUs of one box
 *   qb200_pair_lists (_ex forms) <- FPFHManager::getCorrespondences, Quatro::getMaxCliques / getFinalInliersIndices for every
 *                                  pair of a batch (examples/run_global_registration.cpp:268, 292)
 *   qb200_*_each                <- one Quatro object per pair: Quatro::reset(Params) + setPreEstaimatedRyRx for every pair of a batch
 *   qb200_*_mixed               <- the same, plus voxelize / FPFHManager / matcher flags and seed per pair
 *                                  (examples/run_global_registration.cpp:206-209)
 *   qb200_register_features_*   <- Matcher::calculateCorrespondences + Quatro::computeTransformation for every pair of a batch
 *                                  of caller keypoints and FPFH-33 descriptors (include/fpfh_manager.hpp:125-127)
 *   qb200_voxelize_batch_*      <- voxelize<T>() for every scan of a batch (include/quatro.hpp:49-57)
 *   qb200_describe_batch_*      <- voxelize<T>() + FPFHEstimation::computeFPFHFeatures + FPFHManager::getObjDescriptor /
 *                                  getTgtNormals for every scan of a batch (include/fpfh_manager.hpp:161-177)
 *   qb200_describe_points_*     <- FPFHEstimation::computeFPFHFeatures for every caller keypoint cloud of a batch
 *                                  (src/teaser_utils/fpfh.cc:44-75)
 *   qb200_match_*               <- FPFHManager::setFeaturePair + getCorrespondences / getSrcMatched / getTgtMatched for every pair
 *                                  of a batch, without the solve (include/fpfh_manager.hpp:98-153, 234-236)
 *   qb200_max_clique_batch_*    <- teaser::Graph + MaxCliqueSolver::findMaxClique for every caller graph of a batch
 *                                  (include/teaser/graph.h:29-274, src/graph.cc:12-130)
 *   qb200_build_graph_batch_*   <- Quatro::computeTIMs + solveForScale + inlier_graph_.addEdge loop for every correspondence set of
 *                                  a batch, the graph handed out (include/quatro.hpp:307-386, 784-789)
 *   qb200_solve_pose_batch_*    <- the tail of Quatro::computeTransformation (chain TIMs + GNC-TLS yaw + COTE + final inliers) for
 *                                  every caller inlier set of a batch (include/quatro.hpp:806-936)
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no C++/torch types.  All pointers are HOST pointers
 *     unless a function takes a qb200_mem_kind (then QB200_MEM_DEVICE pointers are accepted).
 *   - Points are 16-byte records {x, y, z, w} (pcl::PointXYZ layout, include/utility.h:109;
 *     KITTI .bin records, examples/run_global_registration.cpp:384-399).
 *   - Every function returns a qb200_status (0 = ok, <0 = bad argument / CUDA failure,
 *     >0 = per-pair degenerate result).  Nothing throws across this boundary.
 *   - There is NO CPU fallback: if no CUDA device is usable qb200_create() fails with
 *     QB200_ERR_NO_DEVICE and no other entry point can be called.
 *   - One handle = one device + one stream; a handle is not thread-safe, several handles are.
 */
#ifndef QUATRO_B200_H_
#define QUATRO_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define QB200_VERSION 100

typedef enum qb200_status {
  QB200_OK = 0,
  /* >0: the call worked, the pair is degenerate (mirrors solution_.valid=false, quatro.hpp:809-813) */
  QB200_DEGENERATE_CLIQUE = 1,   /* max clique size <= 1 */
  QB200_DEGENERATE_INPUT = 2,    /* fewer than 2 correspondences / empty cloud */
  QB200_CAPACITY_EXCEEDED = 3,   /* a per-pair buffer (voxels / correspondences) overflowed; result invalid */
  /* <0: errors */
  QB200_ERR_BAD_ARG = -1,
  QB200_ERR_NO_DEVICE = -2,
  QB200_ERR_CUDA = -3,
  QB200_ERR_UNSUPPORTED = -4,    /* e.g. use_crosscheck = 0, libnccl absent */
  QB200_ERR_VOXEL_OVERFLOW = -5  /* PCL's voxel index would not fit an int: the truncated spans dx*dy*dz > INT_MAX (PCL warns and
                                    returns the input unfiltered), a kept point's floor(p / leaf) outside int32, or the floor-based
                                    grid div_b[0]*div_b[1]*div_b[2] > INT_MAX, or a largest linear index above INT_MAX (PCL's
                                    float subtraction can round a cell coordinate up to div_b); the input is returned
                                    unfiltered in every case */
} qb200_status;

/* qb200_result.flags */
enum { QB200_FLAG_CLIQUE_TRUNCATED = 1 /* PMC_EXACT stopped at max_clique_node_limit: the clique is the best found, not proven maximum */ };
#define QB200_DEFAULT_CLIQUE_NODE_LIMIT 262144

/* Quatro::INLIER_SELECTION_MODE, include/quatro.hpp:184-189 */
enum { QB200_PMC_EXACT = 0, QB200_PMC_HEU = 1, QB200_KCORE_HEU = 2, QB200_INLIER_NONE = 3 };
/* Params::cote_mode, include/quatro.hpp:209 */
enum { QB200_COTE_MEDIAN = 0, QB200_COTE_WEIGHTED_MEAN = 1 };
typedef enum qb200_mem_kind { QB200_MEM_HOST = 0, QB200_MEM_DEVICE = 1 } qb200_mem_kind;

/* One POD for every knob on the path.  Defaults (qb200_default_params) = config/params.yaml:22-44
 * + the hard-coded matcher flags of include/fpfh_manager.hpp:126-127. */
typedef struct qb200_params {
  /* front end */
  float voxel_size;              /* 0.3   voxelize leaf                      params.yaml:22 */
  float normal_radius;           /* 0.5                                      params.yaml:24 */
  float fpfh_radius;             /* 0.75                                     params.yaml:25 */
  float grid_cell;               /* 0 -> (1 + 2^-9) fpfh_radius. Cell of the neighbour-search lattice; the neighbour SETS do not
                                    depend on it, only the (cell,index) order in which they are accumulated. */
  float tuple_scale;             /* 0.95                                     fpfh_manager.hpp:127 */
  int32_t use_crosscheck;        /* 1 */
  int32_t use_tuple_test;        /* 1 */
  int32_t tuple_trials_per_corr; /* 100                                      feature_matcher.cc:195 */
  int32_t skip_flagged;          /* 1: voxelize drops points with w < 0 (stand-in for the reference's
                                    ground/sub-cluster removal, which is out of scope; PCL itself only
                                    drops non-finite points) */
  int32_t reserved0;
  uint64_t seed;                 /* tuple-test RNG seed (replaces srand(time(NULL)), feature_matcher.cc:189) */
  /* solver, include/quatro.hpp:202-268 */
  double noise_bound;            /* 0.3   */
  double cbar2;                  /* 1.0   */
  double rot_noise_bound;        /* 0 -> 2*noise_bound (the value the reference's function-local static
                                    latches on its first call, quatro.hpp:469-470 after :851) */
  double cote_noise_bound;       /* 0.3   Quatro::noise_bound_ ctor constant, quatro.hpp:115,601 */
  double rotation_gnc_factor;    /* 1.4   */
  double rotation_cost_threshold;/* 1.1e-4 */
  double kcore_heuristic_threshold; /* 0.5 */
  int32_t rotation_max_iterations;  /* 50 */
  int32_t inlier_selection_mode;    /* QB200_PMC_HEU */
  int32_t cote_mode;                /* QB200_COTE_MEDIAN */
  int32_t using_rot_inliers_when_estimating_cote; /* 0 */
  int32_t use_pre_estimated_RyRx;   /* 0 */
  int32_t max_clique_node_limit;    /* PMC_EXACT: branch-and-bound nodes per pair before the search returns its best clique so far
                                       (deterministic stand-in for pmc's wall-clock time_limit, src/graph.cc:44); 0 -> QB200_DEFAULT_CLIQUE_NODE_LIMIT */
  double RyRx[9];                   /* row-major 3x3, setPreEstaimatedRyRx, quatro.hpp:276-279 */
} qb200_params;

/* Largest max_voxel_points qb200_create accepts (2^18): dense indoor scans at a 0.05 m voxel reach 100-150 k points per cloud.
 * The handle's device memory grows linearly with it, about 1.2 KB per voxel point and cloud: a one-slot handle with 262144 voxel and
 * 524288 raw points per cloud allocates 0.74 GB. */
#define QB200_MAX_VOXEL_POINTS 262144

/* Largest max_corr qb200_create accepts (2^15): correspondence ids, ranks and degrees fit 16 bits and the 2 x 32768 COTE events
 * of a pair are tagged 0..65535.  A slot's two adjacency copies take max_corr^2 / 4 bytes (256 MB at 32768), so a handle of
 * this capacity wants few slots.  Graphs and cliques above 8192 vertices keep their per-vertex k-core / clique arrays in a
 * global-memory scratch of about 1.2 MB per slot, cliques above 4096 members the pose workspace (42 bytes per member). */
#define QB200_MAX_CORR 32768

/* Handle configuration: device and per-pair capacities (device workspaces are sized once). */
typedef struct qb200_config {
  int32_t device;            /* CUDA ordinal */
  int32_t max_batch_slots;   /* pairs resident in one wave of the batch pipeline (default 64) */
  int32_t max_raw_points;    /* per cloud (default 131072) */
  int32_t max_voxel_points;  /* per cloud (default 16384; multiple of 128, <= QB200_MAX_VOXEL_POINTS) */
  int32_t max_corr;          /* per pair  (default 4096; multiple of 32, <= QB200_MAX_CORR; cliques of any size up to max_corr) */
  int32_t reserved[3];
} qb200_config;

/* Fixed-size per-pair record (also the unit gathered across GPUs). */
typedef struct qb200_result {
  int32_t valid;             /* solution_.valid */
  int32_t status;            /* qb200_status for this pair */
  int32_t n_src_vox, n_tgt_vox;
  int32_t n_mutual;          /* mutual nearest neighbours before the tuple test */
  int32_t n_corr;            /* L: correspondences after tuple test + dedupe */
  int32_t max_core;          /* pmc max core number (graph.cc:60) */
  int32_t clique_size;
  int32_t gnc_iters;
  int32_t n_rot_inliers;     /* getNumRotaionInliers */
  int32_t n_final_inliers;
  int32_t flags;             /* QB200_FLAG_* bits */
  int64_t n_edges;
  double cost;               /* Quatro::cost_ */
  double T[16];              /* column-major 4x4 (Eigen::Matrix4d memory order); identity when !valid */
} qb200_result;

typedef struct qb200_pair {
  const float* src; /* n_src x 4 floats */
  const float* tgt;
  int32_t n_src, n_tgt;
} qb200_pair;

typedef struct qb200_handle qb200_handle;

void qb200_default_params(qb200_params* p);
void qb200_default_config(qb200_config* c);
int qb200_version(void);

/* Every QB200_* environment switch (QB200_LANES, QB200_MATCH_EXACT, QB200_TC_VERIFY, QB200_TC_PROF, QB200_TIMELINE) is read here,
 * when the handle is created: a switch applies to the handles created while it is set, and changing the environment later does
 * not affect an existing handle. */
int qb200_create(const qb200_config* cfg, qb200_handle** out);
void qb200_destroy(qb200_handle* h);
/* Run on a caller-owned CUDA stream (cudaStream_t as void*); NULL restores the handle's own stream. */
int qb200_set_stream(qb200_handle* h, void* cuda_stream);
const char* qb200_last_error(const qb200_handle* h);
/* Number of kernels this handle has launched so far (bench.py's gpu_launches). */
int64_t qb200_launch_count(const qb200_handle* h);

/* --- stage boundaries (host pointers) ------------------------------------------------------ */

/* pcl::VoxelGrid semantics: centroid per occupied leaf cube, output ordered by ascending
 * (k,j,i) cell; non-finite points (and w<0 points when skip_flagged) are dropped. */
int qb200_voxelize(qb200_handle* h, const float* pts4, int32_t n, float leaf, int32_t skip_flagged,
                   float* out4, int32_t cap, int32_t* n_out);

/* --- pre-processing before the path: ground removal (SURVEY.md 8f-1) ------------------------------
 * qb200_patchwork <- PatchWork<PointT>::estimate_ground, include/patchwork.hpp:329-455 (concentric zone model
 * :512-543, region-wise ground plane fit :278-324,548-590, ground likelihood estimation :386-440), de-ROS-ed: the
 * parameters the reference reads from the ROS parameter server (patchwork.hpp:50-95, config/patchwork_params.yaml)
 * travel in this POD. */
#define QB200_PW_MAX_ZONES 4
#define QB200_PW_MAX_THRESHOLDS 8
typedef struct qb200_patchwork_params {
  double sensor_height;                   /* 1.723   patchwork_params.yaml:1 */
  double th_seeds;                        /* 0.25 */
  double th_dist;                         /* 0.125 */
  double max_range;                       /* 80.0 */
  double min_range;                       /* 2.7 (= min_ranges_each_zone[0]) */
  double uprightness_thr;                 /* 0.707 */
  double adaptive_seed_selection_margin;  /* -1.1 */
  double global_elevation_threshold;      /* -0.5 */
  double min_ranges_each_zone[QB200_PW_MAX_ZONES];       /* 2.7, 12.3625, 22.025, 41.35 */
  double elevation_thresholds[QB200_PW_MAX_THRESHOLDS];  /* -1.2, -0.9984, -0.851, -0.605 */
  double flatness_thresholds[QB200_PW_MAX_THRESHOLDS];   /* 0.0001, 0.000125, 0.000185, 0.000185 */
  int32_t num_iter;                       /* 3 */
  int32_t num_lpr;                        /* 20 */
  int32_t num_min_pts;                    /* 80 */
  int32_t using_global_elevation;         /* 0 */
  int32_t num_zones;                      /* 4 (the reference's binning is written for exactly four zones, patchwork.hpp:520-539) */
  int32_t num_thresholds;                 /* 4 = rings of interest (elevation_thresholds.size()) */
  int32_t num_sectors_each_zone[QB200_PW_MAX_ZONES];     /* 16, 32, 54, 32 */
  int32_t num_rings_each_zone[QB200_PW_MAX_ZONES];       /* 2, 4, 4, 4 */
} qb200_patchwork_params;
void qb200_default_patchwork_params(qb200_patchwork_params* p);

/* ground4 / nonground4: room for n points each (either may be NULL: only the counts are returned).  Point order of both
 * outputs = the reference's: patches in (zone, ring, sector) order, inside a patch ascending (z, input index); a patch whose
 * plane is rejected hands its ground part, then its non-ground part, to the non-ground output (patchwork.hpp:399-436).
 * Points outside (min_range, max_range], below -1.8 sensor_height, non-finite, or in patches of <= num_min_pts points appear in
 * neither output (as in the reference).  QB200_CAPACITY_EXCEEDED: a patch holds more than 16384 points. */
int qb200_patchwork(qb200_handle* h, const float* pts4, int32_t n, const qb200_patchwork_params* p,
                    float* ground4, int32_t* n_ground, float* nonground4, int32_t* n_nonground);

/* qb200_segment_cloud <- ImageProjection::segmentCloud in "Patchwork" mode, include/imageProjection.hpp:273-294: range-image
 * projection (:308-352), connected components of the range image under the LeGO-LOAM angle criterion (labelComponents, :483-579)
 * and the extraction of the valid segments / outliers (:424-481, getValidSegments :214-216, getOutliers :230-232).
 * The constructor's per-sensor constants (:86-131) travel in this POD; qb200_default_segment_params = "Velodyne-64-HDE",
 * "4CrossNeighbor" (examples/run_global_registration.cpp:53-55). */
enum { QB200_NEIGHBORS_4 = 0, QB200_NEIGHBORS_8 = 1, QB200_NEIGHBORS_4_CROSS = 2 };
typedef struct qb200_segment_params {
  int32_t n_scan;                     /* 64   (<= 64) */
  int32_t horizon_scan;               /* 1800 */
  float ang_res_x;                    /* 360 / 1800 */
  float ang_res_y;                    /* 26.9 / 63 */
  float ang_bottom;                   /* 25.0 */
  float segment_theta;                /* 60 deg in radians */
  int32_t neighbor_mode;              /* QB200_NEIGHBORS_4_CROSS */
  int32_t min_pts_for_subclustering;  /* 30 */
  int32_t segment_valid_point_num;    /* 5 */
  int32_t segment_valid_line_num;     /* 3 */
} qb200_segment_params;
void qb200_default_segment_params(qb200_segment_params* p);

/* valid4 / outlier4: room for n_scan * horizon_scan points each (either may be NULL).  Both outputs are in row-major pixel
 * order; a pixel holds the LAST input point projected into it (:340-346); w = 1. */
int qb200_segment_cloud(qb200_handle* h, const float* pts4, int32_t n, const qb200_segment_params* p,
                        float* valid4, int32_t* n_valid, float* outlier4, int32_t* n_outlier);

/* qb200_preprocess_batch: the example's pre-processing (examples/run_global_registration.cpp:136-162) for many scans in one call.
 * For every scan i each output array and each count is byte-identical to qb200_patchwork(scan i) followed by
 * qb200_segment_cloud on that scan's non-ground output, on the same handle; nothing depends on the batch size or the scan's
 * position in it.  Scans are processed in waves of 2 * max_batch_slots; the non-ground clouds stay on the device between the two
 * steps.  scans4[i]: n_points[i] x {x,y,z,w} in `kind` memory (n_points[i] <= max_raw_points).  sp == NULL: ground removal only
 * (valid and outlier counts are 0 and their arrays are not touched).
 * Bad arguments fail the whole call with QB200_ERR_BAD_ARG before any work starts. */
typedef struct qb200_preprocess_out {
  int32_t cap_per_scan;  /* >= 1: points reserved per scan in every point array below */
  int32_t kind;          /* qb200_mem_kind of the four point arrays (QB200_MEM_DEVICE: memory of the handle's device, 16-byte aligned) */
  float* ground4;        /* [n][cap][4] or NULL */
  float* nonground4;     /* [n][cap][4] or NULL */
  float* valid4;         /* [n][cap][4] valid segments of the non-ground cloud, or NULL */
  float* outlier4;       /* [n][cap][4] or NULL */
  int32_t* counts;       /* host [n][4] ground, non-ground, valid, outlier: full counts, never clipped */
  int32_t* status;       /* host [n] what qb200_patchwork returns for that scan (QB200_OK / QB200_CAPACITY_EXCEEDED) */
} qb200_preprocess_out;  /* scan i's entries start at i * cap_per_scan; it gets min(count, cap_per_scan) of them, and nothing past
                            that is written: a count above cap_per_scan shows the clipping */
int qb200_preprocess_batch(qb200_handle* h, const float* const* scans4, const int32_t* n_points, int32_t n_scans,
                           qb200_mem_kind kind, const qb200_patchwork_params* pp,
                           const qb200_segment_params* sp /* NULL: ground removal only */, const qb200_preprocess_out* out);

/* qb200_preprocess_batch with one parameter entry per scan: pp[i] (and sp[i]) pre-process scan i.  pp and sp point to n_scans
 * entries (NULL is fine when n_scans == 0); sp == NULL: ground removal only for every scan.  A batch of mixed sensors (each scan's
 * own range image, as the reference builds one ImageProjection per cloud) or of per-scan mounting heights runs in one call.
 * For every scan i each output array, count and status is byte-identical to qb200_preprocess_batch called on scan i alone with
 * pp[i] / sp[i], on the same handle; nothing depends on the batch, the wave, the scan's position or the memory kinds.
 * Every entry must pass the checks of qb200_preprocess_batch: a bad entry fails the whole call with QB200_ERR_BAD_ARG before any
 * work starts (no count, status or output entry is written) and qb200_last_error names the entry.  cap_per_scan, the output
 * descriptor, the memory kinds and QB200_CAPACITY_EXCEEDED behave as in qb200_preprocess_batch.  The parameter arrays are
 * copied by the call. */
int qb200_preprocess_batch_each(qb200_handle* h, const float* const* scans4, const int32_t* n_points, int32_t n_scans,
                                qb200_mem_kind kind, const qb200_patchwork_params* pp, const qb200_segment_params* sp,
                                const qb200_preprocess_out* out);

/* normals4: n x {nx,ny,nz,curvature}; desc33: n x 33 floats (pcl::FPFHSignature33). Either may be NULL. */
int qb200_compute_fpfh(qb200_handle* h, const float* pts4, int32_t n, float normal_radius,
                       float fpfh_radius, float grid_cell, float* normals4, float* desc33);

/* corr: n_corr x {src_idx, tgt_idx}, sorted lexicographically, unique. */
int qb200_match(qb200_handle* h, const float* src4, int32_t n_src, const float* src_desc33,
                const float* tgt4, int32_t n_tgt, const float* tgt_desc33, const qb200_params* p,
                int32_t* corr, int32_t cap, int32_t* n_corr, int32_t* n_mutual);

/* adj: L rows x words_per_row uint32, bit j of row i set iff edge (i,j); full symmetric matrix.
 * words_per_row >= ceil(L/32).  degree (L) and n_edges may be NULL. */
int qb200_build_graph(qb200_handle* h, const float* a4, const float* b4, int32_t L,
                      double noise_bound, double cbar2, uint32_t* adj, int32_t words_per_row,
                      int32_t* degree, int64_t* n_edges);

/* clique: ascending vertex ids.  kcore (L, pmc's core number + 1) and kcore_order (L) may be NULL.  Bits at columns >= L of adj
 * (the last used word's high bits and any padding words) are ignored.  QB200_KCORE_HEU compares max_core with
 * (int)(kcore_heuristic_threshold * L) as x86-64 computes that cast: INT_MIN for NaN and for products outside int range. */
int qb200_max_clique(qb200_handle* h, const uint32_t* adj, int32_t L, int32_t words_per_row,
                     int32_t mode, double kcore_heuristic_threshold, int32_t* clique, int32_t* n_clique,
                     int32_t* kcore, int32_t* kcore_order, int32_t* max_core);
/* The same with the PMC_EXACT knobs: node_limit (0 = default) and the QB200_FLAG_* bits of the search (flags may be NULL).
 * PMC_EXACT = the heuristic clique as the incumbent, then a bit-parallel branch and bound with greedy-colouring bounds
 * (src/graph.cc:106-127 -> [EXT] pmc::pmcx_maxclique::search_dense); the clique SIZE is the maximum, membership follows the
 * canonical sequential order of DESIGN.md 5.3 (pmc's own choice among equal maximum cliques depends on thread timing). */
int qb200_max_clique_ex(qb200_handle* h, const uint32_t* adj, int32_t L, int32_t words_per_row,
                        int32_t mode, double kcore_heuristic_threshold, int64_t node_limit, int32_t* clique, int32_t* n_clique,
                        int32_t* kcore, int32_t* kcore_order, int32_t* max_core, int32_t* flags);

/* rotation + translation given the (sorted) clique. inlier_mask (n_clique bytes) may be NULL.
 * A clique entry outside [0, L) is refused with QB200_ERR_BAD_ARG before anything reaches the device. */
int qb200_solve_pose(qb200_handle* h, const float* a4, const float* b4, int32_t L,
                     const int32_t* clique, int32_t n_clique, const qb200_params* p,
                     qb200_result* res, uint8_t* rot_inlier_mask, uint8_t* trans_inlier_mask);

/* = Quatro::computeTransformation on matched point pairs. */
int qb200_solve_correspondences(qb200_handle* h, const float* a4, const float* b4, int32_t L,
                                const qb200_params* p, qb200_result* res);

/* voxelized clouds in -> correspondences + matched point copies (FPFHManager::setFeaturePair). */
int qb200_match_and_pack(qb200_handle* h, const float* src4, int32_t n_src, const float* tgt4,
                         int32_t n_tgt, const qb200_params* p, int32_t* corr, float* src_matched4,
                         float* tgt_matched4, int32_t cap, int32_t* n_corr);

/* Batch of precomputed correspondence sets (matched point pairs a[i] <-> b[i], xyzw records): graph -> max clique ->
 * GNC-TLS yaw + COTE for every set, = Quatro::computeTransformation (include/quatro.hpp:769-936) called once per set
 * with setInputSource / setInputTarget already given matched clouds.  Sets are processed in waves of
 * max_batch_slots; kind says where a / b live; results is a host array of n records. */
typedef struct qb200_corr_set {
  const float* a;   /* L x 4 floats (source side) */
  const float* b;   /* L x 4 floats (target side) */
  int32_t L;        /* <= max_corr */
  int32_t reserved;
} qb200_corr_set;
int qb200_solve_batch(qb200_handle* h, const qb200_corr_set* sets, int32_t n_sets, const qb200_params* p,
                      qb200_mem_kind kind, qb200_result* results);

/* --- per-pair lists of the batch entry points: correspondences, max clique, final inliers, inlier masks -------------------------
 * The single-pair getters (qb200_get_last_*) read slot 0 after a single-pair call; the _ex forms of the batch entry points hand out
 * the same lists for every pair of a batch.  The caller owns every array; pair i's entries start at i * cap_per_pair whatever wave or
 * lane ran it.  Pair i gets min(count, cap_per_pair) entries of each list, count taken from its record: n_corr for corr and the
 * matched points, clique_size for the clique and both masks, n_final_inliers for the final inliers.  Entries past that count are
 * left untouched, and a pair whose status is QB200_CAPACITY_EXCEEDED gets no entries.  A pair whose clique has at most one member
 * is not solved: its mask entries are 0.  When a list that was asked for (a non-NULL array) held more than cap_per_pair entries,
 * the pair's record carries QB200_FLAG_LISTS_TRUNCATED; records of calls without lists never do.  The lists never depend on the
 * wave size, the lane count, the destination kind, or whether the pair came through the scan cache.
 * QB200_MEM_HOST arrays are complete when the call returns (enqueue: when the flush returns).  QB200_MEM_DEVICE arrays (memory of
 * the handle's device; corr 8-byte, matched points 16-byte aligned) are written by the call's stream work and are complete when it
 * is done, under the same rule.  The descriptor itself is copied by the call. */
typedef struct qb200_pair_lists {
  int32_t cap_per_pair;       /* 1 .. max_corr: entries reserved per pair in every array below */
  int32_t kind;               /* qb200_mem_kind of every array below (QB200_MEM_DEVICE: memory of the handle's device) */
  int32_t* corr;              /* [n][cap][2] (source voxel idx, target voxel idx), same order as qb200_get_last_correspondences */
  float* src_matched4;        /* [n][cap][4] matched points (getSrcKps), aligned with corr */
  float* tgt_matched4;        /* [n][cap][4] */
  int32_t* clique;            /* [n][cap] ascending correspondence ids = qb200_get_last_clique (getMaxCliques) */
  int32_t* final_inliers;     /* [n][cap] = qb200_get_last_final_inliers (getFinalInliersIndices) */
  uint8_t* rot_inlier_mask;   /* [n][cap] per clique member, as qb200_solve_pose writes it */
  uint8_t* trans_inlier_mask; /* [n][cap]; a translation estimated from the rotation inliers only leaves 0 past n_rot_inliers */
} qb200_pair_lists;           /* any array may be NULL: nothing is written to it */
enum { QB200_FLAG_LISTS_TRUNCATED = 2 /* a list of this pair had more than cap_per_pair entries */ };

/* qb200_solve_batch + the lists (Quatro::getMaxCliques / getFinalInliersIndices, include/quatro.hpp:949-972).  The caller supplied
 * the correspondences, so corr, src_matched4 and tgt_matched4 must be NULL (else QB200_ERR_BAD_ARG). */
int qb200_solve_batch_ex(qb200_handle* h, const qb200_corr_set* sets, int32_t n_sets, const qb200_params* p, qb200_mem_kind kind,
                         qb200_result* results, const qb200_pair_lists* lists);

/* Pipelined form of qb200_register_batch for a stream of batches: _enqueue queues the batch and returns (it collects a lane's
 * earlier wave only when it needs that lane again), so the single-warp tail of one batch runs under the PCIe copies and front-end
 * kernels of the next; _flush waits for everything queued and completes the record arrays.  The scans (host kind) and `results` of
 * every queued batch must stay valid until a flush (or qb200_register_batch, = enqueue + flush) returns.  Other entry points flush
 * implicitly.  Raw, cached, caller-feature and correspondence-set batches (qb200_register_cached_enqueue_mixed,
 * qb200_register_features_enqueue_each, qb200_solve_batch_enqueue_each), scan-cache writes (qb200_cache_scans_enqueue_each) and describe
 * calls (qb200_describe_batch_enqueue_each, qb200_describe_points_enqueue_each), voxelize calls (qb200_voxelize_batch_enqueue_each)
 * and match calls (qb200_match_*_enqueue_*) may be queued
 * in one stream and completed by a single flush; every access to a
 * cache slot follows enqueue order, so a queued cached batch registers the slot contents it was enqueued against.  qb200_cache_reserve,
 * qb200_cache_copy, qb200_cache_read and the pre-processing calls flush first, so they see every write queued before them. */
int qb200_register_batch_enqueue(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* p, qb200_mem_kind kind,
                                 qb200_result* results);
int qb200_register_batch_flush(qb200_handle* h);
/* qb200_register_batch_enqueue + the lists of qb200_register_batch_ex; the arrays must stay valid until the flush, as results must */
int qb200_register_batch_enqueue_ex(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* p,
                                    qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists);

/* raw scans in -> pose out. */
int qb200_register_pair(qb200_handle* h, const float* src4, int32_t n_src, const float* tgt4,
                        int32_t n_tgt, const qb200_params* p, qb200_result* res);

/* Batch of independent pairs.  kind says where pairs[i].src/tgt live; results is a host array.
 * The batch is processed in waves of max_batch_slots pairs.  Batches larger than one wave rotate over up to
 * 4 lanes (each further lane -- same buffers again, own stream -- is allocated on first use) so that one wave's
 * host->device copies and solver tail overlap the other waves' dense kernels; QB200_LANES=n (1..8, default 4) in
 * the environment sets the lane count (1 = strictly one wave at a time).  Results never depend on the wave size
 * or the lane.  Every batch call (raw, cached or correspondence-set input, any form) goes through the same checks and the same
 * wave driver, and its waves rotate over the same lanes; only raw host scans cross PCIe on the shared copy stream and open a
 * multi-wave batch with a quarter wave.  A call with n = 0 pairs does no work and
 * latches no rotation noise bound.  A kind other than QB200_MEM_HOST / QB200_MEM_DEVICE is QB200_ERR_BAD_ARG. */
int qb200_register_batch(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs,
                         const qb200_params* p, qb200_mem_kind kind, qb200_result* results);
/* qb200_register_batch + every pair's lists: FPFHManager::getCorrespondences / getSrcKps / getTgtKps (include/fpfh_manager.hpp:
 * 234-236), Quatro::getMaxCliques / getFinalInliersIndices (include/quatro.hpp:949-972).  lists == NULL: = qb200_register_batch.
 * With one pair it also sets what qb200_get_last_* read. */
int qb200_register_batch_ex(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* p, qb200_mem_kind kind,
                            qb200_result* results, const qb200_pair_lists* lists);

/* --- scan cache: one scan against many (loop-closure sweeps) and odometry chains -------------------------------------------------
 * FPFHManager keeps the previous target's cloud and descriptors and reuses them as the next source (swapTgt2Src / is_odometry_test_,
 * include/fpfh_manager.hpp:74-77, 111-118) and hands its descriptors out (getObjDescriptor / getSceneDescriptor / getTgtNormals,
 * :161-177).  The cache keeps voxel points, normals and FPFH-33 of a scan resident on the DEVICE, so the front end runs once per
 * scan instead of once per pair.  Slots are indexed 0 .. n_slots-1; results never depend on whether a scan came from the cache
 * (tests/test_gpu_parity.py::test_scan_cache_*). */
typedef struct qb200_slot_pair { int32_t src_slot, tgt_slot; } qb200_slot_pair;
int qb200_cache_reserve(qb200_handle* h, int32_t n_slots);   /* (re)allocates; 0 frees.  192 B per voxel point and slot: ~3.1 MB at
                                                                 max_voxel_points = 16384, ~50 MB at 262144 */
/* voxelize + normals + FPFH of n_scans raw scans (scans4[i]: n_points[i] x {x,y,z,w}) into slots slot_ids[i] (a slot named twice
 * ends with the last scan that names it); = qb200_cache_scans_enqueue_each with p repeated + qb200_register_batch_flush */
int qb200_cache_scans(qb200_handle* h, const float* const* scans4, const int32_t* n_points, const int32_t* slot_ids, int32_t n_scans,
                      const qb200_params* p, qb200_mem_kind kind);
/* match + graph + clique + pose for pairs of cached scans (= qb200_register_batch without its front end); p's front-end parameters
 * must be the ones the slots were cached with */
int qb200_register_cached(qb200_handle* h, const qb200_slot_pair* pairs, int32_t n_pairs, const qb200_params* p, qb200_result* results);
/* qb200_register_cached + the lists of qb200_register_batch_ex (getCorrespondences, getMaxCliques, getFinalInliersIndices); corr
 * indexes the voxel order qb200_cache_read returns */
int qb200_register_cached_ex(qb200_handle* h, const qb200_slot_pair* pairs, int32_t n_pairs, const qb200_params* p,
                             qb200_result* results, const qb200_pair_lists* lists);
int qb200_cache_copy(qb200_handle* h, int32_t from_slot, int32_t to_slot);   /* swapTgt2Src */

/* --- per-pair solver parameters: one batch, N independently configured Quatro objects ---------------------------------------------
 * The reference configures each Quatro object on its own (reset(Params), include/quatro.hpp:202-268, 755-765) and gives it the IMU
 * roll/pitch of its scan (setPreEstaimatedRyRx, :276-279, applied at :419-426 and :891-893).  The _each forms take the same arguments
 * as their _ex siblings, except that `params` points to n entries, one per pair (or correspondence set) in the order of the input
 * array.  The array is copied by the call; `lists` may be NULL.
 *   Solver fields (noise_bound .. RyRx: noise_bound, cbar2, rot_noise_bound, cote_noise_bound, rotation_gnc_factor,
 *     rotation_cost_threshold, kcore_heuristic_threshold, rotation_max_iterations, inlier_selection_mode, cote_mode,
 *     using_rot_inliers_when_estimating_cote, use_pre_estimated_RyRx, max_clique_node_limit, RyRx) may differ from pair to pair.
 *   Front-end fields (voxel_size .. seed: the FPFHManager / voxelize configuration) must be bit-identical in every entry of
 *     qb200_register_batch_each, _enqueue_each and qb200_register_cached_each (cached slots are bound to one set of them);
 *     qb200_solve_batch_each ignores them.
 *   Every entry must pass the checks of the _ex call; a bad entry or a front-end mismatch fails the whole call with QB200_ERR_BAD_ARG
 *     before any work starts, and no record or list is written.
 *   Pair i's record and lists are byte-identical to pair i of the _ex call made with params[i] for the whole batch (results never
 *     depend on the batch, the wave or the lane).
 *   Entries with rot_noise_bound == 0 are resolved in pair order through the handle's latch, as if the single-pair calls had been made
 *     in that order: on a handle that has not latched yet, the first such entry latches 2 * its noise_bound. */
/* qb200_register_batch_ex with one params entry per pair */
int qb200_register_batch_each(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* params, qb200_mem_kind kind,
                              qb200_result* results, const qb200_pair_lists* lists);
/* qb200_register_batch_enqueue_ex with one params entry per pair; completed by qb200_register_batch_flush like every enqueue */
int qb200_register_batch_enqueue_each(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                      qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists);
/* qb200_register_cached_ex with one params entry per slot pair (front-end fields: the ones the slots were cached with) */
int qb200_register_cached_each(qb200_handle* h, const qb200_slot_pair* pairs, int32_t n_pairs, const qb200_params* params,
                               qb200_result* results, const qb200_pair_lists* lists);
/* qb200_solve_batch_ex with one params entry per correspondence set (front-end fields ignored) */
int qb200_solve_batch_each(qb200_handle* h, const qb200_corr_set* sets, int32_t n_sets, const qb200_params* params, qb200_mem_kind kind,
                           qb200_result* results, const qb200_pair_lists* lists);

/* --- per-pair front-end parameters: presets, retries and seed sweeps in one batch ---------------------------------------------------
 * The reference voxelizes and describes every registration with its own configuration: voxelize(..., voxel_size)
 * (examples/run_global_registration.cpp:206-207), a fresh FPFHManager(normal_radius, fpfh_radius) per pair (:209), the matcher's tuple
 * flags (include/fpfh_manager.hpp:125-127) and an RNG seed per run (src/teaser_utils/feature_matcher.cc:189).  The _mixed forms take
 * exactly the arguments of their _each siblings; every field of every entry may differ, the front-end fields (voxel_size .. seed)
 * included.  A pair's source and target are both voxelized and described with its entry.
 *   Pair i's record and lists are byte-identical to pair i of the _ex call made with params[i] for the whole batch; they never depend
 *     on the batch, the wave, the lane, the memory kind or the configurations of the other pairs of the wave.  A pair's size refusals
 *     (QB200_ERR_VOXEL_OVERFLOW, QB200_CAPACITY_EXCEEDED) stay its own.
 *   Checks happen before any work starts: every entry must pass the checks of the _ex call (QB200_ERR_BAD_ARG), an entry with
 *     use_crosscheck = 0 fails the call with QB200_ERR_UNSUPPORTED, and a cached pair whose entry does not match the front-end
 *     signature of one of its two slots (voxel_size, normal_radius, fpfh_radius, lattice cell) fails it with QB200_ERR_BAD_ARG.  A
 *     rejected call writes no record, list or slot, and qb200_last_error names the entry.
 *   Entries with rot_noise_bound == 0 are resolved in pair order through the handle's latch, as in the _each forms. */
/* qb200_register_batch_each whose entries may differ in their front-end fields */
int qb200_register_batch_mixed(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* params, qb200_mem_kind kind,
                               qb200_result* results, const qb200_pair_lists* lists);
/* qb200_register_batch_enqueue_each whose entries may differ in their front-end fields; completed by qb200_register_batch_flush */
int qb200_register_batch_enqueue_mixed(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                       qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists);
/* qb200_register_cached_each whose entries may differ in their front-end fields: pair i's entry must match the signature of its own
 * two slots (not that of entry 0) */
int qb200_register_cached_mixed(qb200_handle* h, const qb200_slot_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                qb200_result* results, const qb200_pair_lists* lists);
/* Pipelined forms of qb200_register_cached_mixed and qb200_solve_batch_each, completed by qb200_register_batch_flush like every
 * enqueue (a loop-closure back end queues candidate batches as keyframes arrive).  A narrower form is one of these with the entry
 * repeated and lists = NULL.
 *   The argument checks are those of the blocking call and run before anything is queued: a rejected call queues and writes nothing,
 *     and the batches already queued still complete on the flush.
 *   The params array and the list descriptor are copied by the call; the slot pairs, host-kind correspondence sets, `results` and
 *     the list arrays must stay valid until the flush returns.
 *   Entries with rot_noise_bound == 0 latch in enqueue order, as in the raw enqueue forms.
 *   Records and lists are byte-identical to those of the blocking call. */
int qb200_register_cached_enqueue_mixed(qb200_handle* h, const qb200_slot_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                        qb200_result* results, const qb200_pair_lists* lists);
int qb200_solve_batch_enqueue_each(qb200_handle* h, const qb200_corr_set* sets, int32_t n_sets, const qb200_params* params,
                                   qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists);
/* qb200_cache_scans with one params entry per scan: scan i is voxelized and described with params[i] and slot_ids[i] records that
 * entry's front-end signature (qb200_cache_copy carries it).  Slot s's voxels, normals and descriptors (qb200_cache_read) are
 * byte-identical to qb200_cache_scans of that scan alone with its entry.  A bad entry fails the call with QB200_ERR_BAD_ARG before
 * any slot is written, and qb200_last_error names it. */
int qb200_cache_scans_each(qb200_handle* h, const float* const* scans4, const int32_t* n_points, const int32_t* slot_ids, int32_t n_scans,
                           const qb200_params* params, qb200_mem_kind kind);
/* qb200_cache_scans_each, queued: completed by qb200_register_batch_flush like every enqueue (a SLAM back end caches each keyframe and
 * queues its candidate batches without draining the stream).  A narrower form is this call with the entry repeated.
 *   The argument checks are those of qb200_cache_scans_each and run before anything is queued: a rejected call queues nothing, writes
 *     no slot and no slot signature, names the bad entry or scan in qb200_last_error, and the batches already queued still complete
 *     on the flush.
 *   Order: every access to a slot follows enqueue order.  A cached batch enqueued before the write registers the slot's old contents,
 *     one enqueued after it the new ones; two queued writes to one slot land in enqueue order; a slot named twice in one call ends
 *     with the last scan that names it, as in the blocking call.
 *   Each written slot's front-end signature is recorded when the call is queued, so a cached batch enqueued after it is checked
 *     against the new signature.
 *   The scans4, n_points, slot_ids and params arrays are read by the call; host-kind scans must stay valid until the flush returns.
 *   Slot contents (qb200_cache_read), and everything registered from them, are byte-identical to the blocking calls made in the
 *     same order. */
int qb200_cache_scans_enqueue_each(qb200_handle* h, const float* const* scans4, const int32_t* n_points, const int32_t* slot_ids,
                                   int32_t n_scans, const qb200_params* params, qb200_mem_kind kind);
/* read a cached scan back: voxel points (n x 4), normals (n x {nx,ny,nz,curvature}), descriptors (n x 33); any may be NULL */
int qb200_cache_read(qb200_handle* h, int32_t slot, float* vox4, float* normals4, float* desc33, int32_t cap, int32_t* n);

/* --- caller keypoints and FPFH-33 descriptors: the matcher boundary in batches ---------------------------------------------------
 * Matcher::calculateCorrespondences(source_points, target_points, source_features, target_features, ...)
 * (include/teaser_utils/feature_matcher.h:42-74, called by FPFHManager::setFeaturePair, include/fpfh_manager.hpp:125-127) followed by
 * Quatro::computeTransformation, for a batch of pairs whose keypoints and descriptors the caller already holds: PCL's
 * FPFHEstimationOMP output, a map database, or qb200_cache_read of another handle.  Pair i is matched and solved with params[i], as
 * qb200_match followed by qb200_solve_correspondences would; the waves rotate over the lanes like every batch call.
 *   Matcher fields (use_tuple_test, tuple_scale, tuple_trials_per_corr, seed) and solver fields may differ from pair to pair.  The
 *     voxel and lattice fields (voxel_size, normal_radius, fpfh_radius, grid_cell, skip_flagged) are ignored; no slot signature is
 *     involved.
 *   Pair i's record and lists are byte-identical to those of this call on pair i alone with params[i]; they never depend on the batch,
 *     the wave, the lane, the memory kind or the other pairs of the wave.
 *   n_src_vox / n_tgt_vox are n_src / n_tgt.  corr indexes the caller's keypoint arrays; src_matched4 / tgt_matched4 are the caller's
 *     keypoint records, w included.
 *   An empty side gives QB200_DEGENERATE_INPUT, as a raw pair with an empty cloud does; more than max_corr correspondences give
 *     QB200_CAPACITY_EXCEEDED.
 *   Checks run before anything starts or is queued.  n < 0, n > max_voxel_points, or a NULL array on a non-empty side give
 *     QB200_ERR_BAD_ARG, and so does, in QB200_MEM_DEVICE kind, an array that is not memory of the handle's device or is misaligned
 *     (keypoints 16-byte, descriptors 4-byte aligned).  A params entry that fails the checks of the _each forms gives QB200_ERR_BAD_ARG,
 *     use_crosscheck = 0 QB200_ERR_UNSUPPORTED.  A rejected call writes no record or list and queues nothing, qb200_last_error names
 *     the entry, and the batches already queued still complete on the flush.
 *   Entries with rot_noise_bound == 0 latch in pair order (enqueue order for the queued form), as in the other _each forms.
 *   qb200_get_stage_ms reports the features' copy and import under [0] (h2d); [1] and [2] (voxel, fpfh) stay zero; [3] .. [7] as usual.
 * A narrower call is this one with the entry repeated and lists = NULL.  The params array and the list descriptor are copied by the
 * call. */
typedef struct qb200_feature_pair {
  const float* src;       /* n_src x {x,y,z,w}: keypoints (e.g. voxel centroids) */
  const float* src_desc;  /* n_src x 33: pcl::FPFHSignature33 rows, the layout qb200_match takes */
  const float* tgt;
  const float* tgt_desc;
  int32_t n_src, n_tgt;
} qb200_feature_pair;
int qb200_register_features_each(qb200_handle* h, const qb200_feature_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                 qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists);
/* qb200_register_features_each, queued: completed by qb200_register_batch_flush like every enqueue, in one stream with raw, cached and
 * correspondence-set batches and cache writes.  Host-kind keypoints and descriptors, `results` and the list arrays must stay valid until
 * the flush returns.  Records and lists are byte-identical to those of the blocking call. */
int qb200_register_features_enqueue_each(qb200_handle* h, const qb200_feature_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                         qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists);

/* --- matching in batches: correspondences and matched points of many pairs, not solved -------------------------------------------
 * FPFHManager::setFeaturePair followed by getCorrespondences / getSrcMatched / getTgtMatched (include/fpfh_manager.hpp:98-153,
 * 234-236) for every pair of a batch: what a caller needs who picks the pairs worth solving from n_mutual / n_corr (a loop-closure
 * pre-filter), hands the correspondences to another estimator, solves one match under several solver settings, or fills a cache of
 * matched pairs.  Each call takes the arguments of its register counterpart and honours the same per-pair fields:
 *   qb200_match_batch_mixed / _enqueue_mixed     raw pairs, as qb200_register_batch_mixed: front-end and matcher fields
 *   qb200_match_cached_mixed / _enqueue_mixed    slot pairs, as qb200_register_cached_mixed: matcher fields, and the entry must match
 *                                                the front-end signature of both slots
 *   qb200_match_features_each / _enqueue_each    caller features, as qb200_register_features_each: matcher fields
 * Contract:
 *   Lists.  Only corr, src_matched4 and tgt_matched4 may be non-NULL; a clique, final-inlier or mask array gives QB200_ERR_BAD_ARG.
 *     lists == NULL gives the records only.  Pair i's corr, src_matched4 and tgt_matched4 are byte-identical to the lists of the
 *     register counterpart on the same inputs and params; they never depend on the batch, the wave, the lane, the memory kinds or the
 *     other pairs.
 *   Records.  status, n_src_vox, n_tgt_vox, n_mutual, n_corr and the matcher's flags (with QB200_FLAG_LISTS_TRUNCATED) equal the register
 *     counterpart's.  Nothing is solved: valid = 0, T is the identity, and max_core, clique_size, gnc_iters, n_rot_inliers,
 *     n_final_inliers, n_edges and cost are 0.
 *   Status.  QB200_DEGENERATE_INPUT for an empty side, QB200_CAPACITY_EXCEEDED for more voxels or correspondences than the handle
 *     holds, or the front-end status the register counterpart gives the pair.  Every other pair is QB200_OK, one with 0 or 1
 *     correspondences included: the caller has its list and decides.
 *   Params.  The solver fields (noise_bound .. RyRx) are ignored and not checked.  The front-end and matcher fields pass the checks of
 *     the register counterpart, and use_crosscheck = 0 gives QB200_ERR_UNSUPPORTED.  Nothing is latched: entries with
 *     rot_noise_bound == 0 stay unresolved, so a match followed by qb200_solve_batch_each latches as the register call would.
 *   Rejections cover the whole call and are decided before anything is queued: no record or list entry is written, qb200_last_error
 *     names the bad pair, entry or array, and the batches already queued still complete on the flush.
 *   The queued forms share the stream and the single flush of every other enqueue form; a queued cached match sees the slot contents
 *     it was enqueued against.  Host-kind inputs, `results` and the list arrays must stay valid until the flush returns.
 *   qb200_get_stage_ms reports the stages that ran: h2d, voxel and fpfh as the input has them, match and d2h; graph, clique and pose
 *     are 0.
 * The params array and the list descriptor are copied by the call.  src_matched4 + i * cap_per_pair * 4 with L = n_corr is pair i's
 * qb200_corr_set for qb200_solve_batch_each, device arrays included. */
int qb200_match_batch_mixed(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* params, qb200_mem_kind kind,
                            qb200_result* results, const qb200_pair_lists* lists);
int qb200_match_batch_enqueue_mixed(qb200_handle* h, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* params, qb200_mem_kind kind,
                                    qb200_result* results, const qb200_pair_lists* lists);
int qb200_match_cached_mixed(qb200_handle* h, const qb200_slot_pair* pairs, int32_t n_pairs, const qb200_params* params, qb200_result* results,
                             const qb200_pair_lists* lists);
int qb200_match_cached_enqueue_mixed(qb200_handle* h, const qb200_slot_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                     qb200_result* results, const qb200_pair_lists* lists);
int qb200_match_features_each(qb200_handle* h, const qb200_feature_pair* pairs, int32_t n_pairs, const qb200_params* params,
                              qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists);
int qb200_match_features_enqueue_each(qb200_handle* h, const qb200_feature_pair* pairs, int32_t n_pairs, const qb200_params* params,
                                      qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists);

/* --- the front end in batches: voxel keypoints, normals and FPFH-33 of many scans into caller memory ----------------------------------
 * voxelize<T> (include/quatro.hpp:49-57) + FPFHEstimation::computeFPFHFeatures (src/teaser_utils/fpfh.cc:44-75), handed out as
 * FPFHManager::getObjDescriptor / getSceneDescriptor / getTgtNormals do (include/fpfh_manager.hpp:161-177), for a batch of raw scans:
 * a descriptor database, a map of keyframe features, or FPFH for another solver.  The output goes straight into the caller's arrays,
 * and qb200_register_features_each of any handle takes it back as keypoints and descriptors.
 *   Scan i (scans4[i]: n_points[i] x {x,y,z,w} in `kind` memory) is voxelized and described with the front-end fields of params[i]
 *     (voxel_size, normal_radius, fpfh_radius, grid_cell, skip_flagged); the other fields are ignored.
 *   Scan i's entries start at i * cap_per_scan in every array; min(counts[i], cap_per_scan) of them are written and nothing past them,
 *     so a count above cap_per_scan shows the clipping.  The arrays are byte-identical to qb200_cache_scans_each of that scan alone
 *     with params[i] followed by qb200_cache_read; they never depend on the batch, the wave, the lane, the memory kinds or the other
 *     scans.
 *   A scan refused on its own gets its status in status[i]: QB200_CAPACITY_EXCEEDED (more occupied voxels than max_voxel_points) or
 *     QB200_ERR_VOXEL_OVERFLOW (PCL's voxel index would overflow; qb200_voxelize hands such a scan back unfiltered, this call does
 *     not).  Its count is 0, nothing is written for it, and the other scans are unaffected.  Every other scan gets QB200_OK, an
 *     empty one (or one whose points are all skipped) with count 0.
 *   Checks run before anything starts or is queued: those of qb200_cache_scans_each (without the slots), cap_per_scan >= 1, non-NULL
 *     counts and status, a known output kind, and in QB200_MEM_DEVICE output kind arrays of the handle's device, vox4 / normals4
 *     16-byte and desc33 4-byte aligned.  A rejected call gives QB200_ERR_BAD_ARG, writes no count, status or entry, queues nothing,
 *     and qb200_last_error names the bad scan, entry or array; batches already queued still complete on the flush.
 *   The scans run in waves of 2 * max_batch_slots over the lanes, as cache writes do.  Host-kind output is complete when the call
 *     returns, device-kind output when the call's stream work is done (the call itself waits for it).
 *   Like a cache write, this is a batch call that registers nothing: qb200_get_stage_ms and qb200_get_kernel_ms report zeros after it.
 * The params array and the output descriptor are copied by the call. */
typedef struct qb200_feature_out {
  int32_t cap_per_scan;  /* >= 1: keypoints reserved per scan in every array below */
  int32_t kind;          /* qb200_mem_kind of the three arrays (QB200_MEM_DEVICE: the handle's device; vox4 / normals4 16-byte,
                            desc33 4-byte aligned) */
  float* vox4;           /* [n][cap][4] voxel centroids in the order qb200_voxelize / qb200_cache_read return, or NULL */
  float* normals4;       /* [n][cap][4] {nx,ny,nz,curvature}, or NULL */
  float* desc33;         /* [n][cap][33] pcl::FPFHSignature33 rows, or NULL */
  int32_t* counts;       /* host [n]: voxel points of scan i, never clipped */
  int32_t* status;       /* host [n]: that scan's own front-end status */
} qb200_feature_out;
int qb200_describe_batch_each(qb200_handle* h, const float* const* scans4, const int32_t* n_points, int32_t n_scans,
                              const qb200_params* params, qb200_mem_kind kind, const qb200_feature_out* out);
/* qb200_describe_batch_each, queued: completed by qb200_register_batch_flush like every enqueue, in one stream with raw, cached,
 * caller-feature and correspondence-set batches and cache writes.  Host-kind scans and every output array (counts and status
 * included) must stay valid until the flush returns, which completes them.  The outputs are byte-identical to the blocking call's. */
int qb200_describe_batch_enqueue_each(qb200_handle* h, const float* const* scans4, const int32_t* n_points, int32_t n_scans,
                                      const qb200_params* params, qb200_mem_kind kind, const qb200_feature_out* out);

/* --- the voxel filter in batches: VoxelGrid centroids of many scans into caller memory -----------------------------------------------
 * voxelize<T> (include/quatro.hpp:49-57, pcl::VoxelGrid) for a batch of raw scans, each with its own leaf, and nothing after it: keyframes
 * stored at a voxel size, another descriptor or registration back end, qb200_describe_points_each at radii chosen later.
 *   Scan i (scans4[i]: n_points[i] x {x,y,z,w} in `kind` memory, 0 <= n_points[i] <= max_raw_points) is filtered with
 *     params[i].voxel_size as the leaf and params[i].skip_flagged.  Every other field is ignored and not checked.
 *   The output descriptor is qb200_feature_out with normals4 and desc33 NULL; vox4 may be NULL (counts and status only).
 *   Scan i's outputs are byte-identical to qb200_voxelize(scan i, voxel_size, skip_flagged) on the same handle:
 *     counts[i] is that call's *n_out given unlimited room, never clipped to cap_per_scan;
 *     scan i's entries start at i * cap_per_scan, and the first min(counts[i], cap_per_scan) of the entries qb200_voxelize writes are
 *     written, nothing past them;
 *     status[i] is the scan's own filter status:
 *       QB200_OK (an empty scan, or one whose points are all skipped, with count 0);
 *       QB200_CAPACITY_EXCEEDED: more occupied voxels than max_voxel_points; the count is max_voxel_points and the entries are the
 *         first centroids, as qb200_voxelize gives them;
 *       QB200_ERR_VOXEL_OVERFLOW: PCL's pass-through.  The count is the number of kept points (finite x, y, z, and w >= 0 when
 *         skip_flagged is set) and the entries are those input records, verbatim and in input order.  This count may exceed
 *         max_voxel_points, up to max_raw_points.
 *     Clipping by cap_per_scan shows only as counts[i] > cap_per_scan, never as a status: the one place where the call differs from
 *     qb200_voxelize's return code.  No output depends on the batch, the wave, the lane, the memory kinds or the other scans.
 *   Checks run before anything starts or is queued: n, the arrays and the kind; every scan's count and pointer (in QB200_MEM_DEVICE
 *     kind memory of the handle's device, 16-byte aligned); every entry's voxel_size (> 0, as qb200_voxelize accepts a leaf; NaN is
 *     refused); the output checks of qb200_describe_batch_each (cap_per_scan >= 1, counts and status, output kind, device vox4 on the
 *     handle's device and 16-byte aligned); and NULL normals4 and desc33.  A rejected call gives QB200_ERR_BAD_ARG, writes no count,
 *     status or entry, queues nothing, and qb200_last_error names the bad scan, entry or array; batches already queued still complete
 *     on the flush.
 *   The scans run in waves of 2 * max_batch_slots over the lanes, as describe calls do, and no normals or FPFH are computed.  Like
 *     them it registers nothing: qb200_get_stage_ms and qb200_get_kernel_ms report zeros after it.
 * The params array and the output descriptor are copied by the call. */
int qb200_voxelize_batch_each(qb200_handle* h, const float* const* scans4, const int32_t* n_points, int32_t n_scans,
                              const qb200_params* params, qb200_mem_kind kind, const qb200_feature_out* out);
/* qb200_voxelize_batch_each, queued: completed by qb200_register_batch_flush like every enqueue, in one stream with every other
 * enqueue form.  Host-kind scans and every output array (counts and status included) must stay valid until the flush returns, which
 * completes them.  The outputs are byte-identical to the blocking call's. */
int qb200_voxelize_batch_enqueue_each(qb200_handle* h, const float* const* scans4, const int32_t* n_points, int32_t n_scans,
                                      const qb200_params* params, qb200_mem_kind kind, const qb200_feature_out* out);

/* --- FPFH of caller keypoint clouds in batches: normals and FPFH-33 of many clouds, without the voxel filter ------------------------
 * FPFHEstimation::computeFPFHFeatures (src/teaser_utils/fpfh.cc:44-75) takes whatever cloud it is handed; this call does the same for a
 * batch of clouds whose keypoints the caller chose: a PCL VoxelGrid run elsewhere, uniform or random sampling, a keypoint detector,
 * a map database that stores keypoints but not descriptors, or the same keypoints described again at other radii.  The output goes
 * straight into the caller's arrays, and qb200_register_features_each of any handle takes it back with the caller's keypoints.
 *   Cloud i (pts4[i]: n_points[i] x {x,y,z,w} in `kind` memory) gets normals and FPFH-33 computed with the lattice fields of params[i]:
 *     normal_radius, fpfh_radius and grid_cell (<= 0 resolves, as everywhere else, to (1 + 2^-9) fpfh_radius).  Every other field is
 *     ignored.  The points are taken in the caller's order, as they are: no voxel filter, no dropping of w < 0, no merging of
 *     duplicates.
 *   normals4[i] and desc33[i] are byte-identical to qb200_compute_fpfh on that cloud alone with the resolved radii and cell, clouds
 *     with points the lattice drops (non-finite, outside the lattice) and coincident duplicates included.  They never depend on the
 *     batch, the wave, the lane, the memory kinds or the other clouds.
 *   The output descriptor is qb200_feature_out, with vox4 NULL (the keypoints are the caller's own).  counts[i] = n_points[i] and
 *     status[i] = QB200_OK, since every refusal is decided for the whole call.  cap_per_scan and the clipping behave as in
 *     qb200_describe_batch_each: cloud i's entries start at i * cap_per_scan, min(n_points[i], cap_per_scan) of them are written.
 *   Checks run before anything starts or is queued.  QB200_ERR_BAD_ARG for n_points[i] < 0 or > max_voxel_points (the rule of
 *     qb200_compute_fpfh and qb200_register_features_each), a NULL cloud with n_points[i] > 0, in QB200_MEM_DEVICE kind a cloud that
 *     is not memory of the handle's device or not 16-byte aligned, a params entry whose radii are not finite and positive, whose
 *     normal_radius exceeds its fpfh_radius or whose grid_cell is not finite, a non-NULL vox4, and the output checks of
 *     qb200_describe_batch_each (cap_per_scan >= 1, counts and status, output kind, device arrays and their alignment).  A rejected
 *     call writes no count, status or entry, queues nothing, and qb200_last_error names the bad cloud, entry or array; batches already
 *     queued still complete on the flush.
 *   The clouds run in waves of 2 * max_batch_slots over the lanes, as describe calls do.  Like them it registers nothing:
 *     qb200_get_stage_ms and qb200_get_kernel_ms report zeros after it.
 * The params array and the output descriptor are copied by the call. */
int qb200_describe_points_each(qb200_handle* h, const float* const* pts4, const int32_t* n_points, int32_t n_clouds,
                               const qb200_params* params, qb200_mem_kind kind, const qb200_feature_out* out);
/* qb200_describe_points_each, queued: completed by qb200_register_batch_flush like every enqueue, in one stream with every other
 * enqueue form.  Host-kind clouds and every output array (counts and status included) must stay valid until the flush returns,
 * which completes them.  The outputs are byte-identical to the blocking call's. */
int qb200_describe_points_enqueue_each(qb200_handle* h, const float* const* pts4, const int32_t* n_points, int32_t n_clouds,
                                       const qb200_params* params, qb200_mem_kind kind, const qb200_feature_out* out);

/* --- maximum cliques of caller graphs in batches -------------------------------------------------------------------------------------
 * teaser::Graph (include/teaser/graph.h:29-207) + teaser::MaxCliqueSolver::findMaxClique (graph.h:219-274, src/graph.cc:12-130) for a
 * batch of graphs the library did not build: complete TIM graphs, consistency tests of the caller's own, pairwise-consistency outlier
 * rejection across sessions.  Each graph runs the k-core peel and the clique search of qb200_max_clique_ex, in waves of max_batch_slots
 * graphs over the lanes like every batch call.
 *   Graph i is an edge list or an adjacency matrix in `kind` memory (below) and is solved with params[i].  Only inlier_selection_mode
 *     (QB200_PMC_EXACT, QB200_PMC_HEU or QB200_KCORE_HEU), kcore_heuristic_threshold and max_clique_node_limit are read; every other
 *     field is ignored.  QB200_INLIER_NONE, an unknown mode or a negative node limit gives QB200_ERR_BAD_ARG.
 *   Edge lists have teaser::Graph::addEdge semantics: (u, v) and (v, u) are one edge, a repeated edge is ignored, and edge order never
 *     matters.  In adjacency rows, bits at columns >= L are ignored.
 *   Invalid graphs: a self-loop, a vertex outside [0, L), an adjacency matrix that is not symmetric or one with a diagonal bit gives
 *     that graph the status QB200_ERR_BAD_ARG, in either memory kind.  This is decided on the device; the graph gets no clique and no
 *     list entries, and the other graphs are unaffected.
 *   Records.  status (QB200_OK for every valid graph), n_corr = L, n_edges (distinct undirected edges = Graph::numEdges()), max_core,
 *     clique_size and flags (QB200_FLAG_CLIQUE_TRUNCATED, QB200_FLAG_LISTS_TRUNCATED).  Nothing is registered: valid = 0, T is the
 *     identity, and n_src_vox, n_tgt_vox, n_mutual, gnc_iters, n_rot_inliers, n_final_inliers and cost are 0.
 *   Lists.  Only clique may be non-NULL; any other list array gives QB200_ERR_BAD_ARG.  The clique is in ascending vertex ids, clipped
 *     to cap_per_pair as in every _ex call.
 *   Equality.  For every valid graph the record fields above and the clique are byte-identical to qb200_max_clique_ex on the same
 *     adjacency with the same mode, threshold and node limit.  They never depend on the batch, the wave, the lane, the memory kinds,
 *     edge list versus adjacency input, or the other graphs.
 *   Checks run before anything starts or is queued: n < 0, L < 0 or L > max_corr, edges and adj both non-NULL, neither of them while
 *     L > 0 and n_edges > 0, n_edges < 0, words_per_row < ceil(L / 32) with adj, a NULL results array, a bad params entry, a bad list
 *     descriptor, and in QB200_MEM_DEVICE kind an array that is not memory of the handle's device or is misaligned (edges 8-byte, adj
 *     4-byte).  A rejected call gives QB200_ERR_BAD_ARG, writes no record or list entry, queues nothing, and qb200_last_error names
 *     the graph, entry or array; batches already queued still complete on the flush.
 *   qb200_get_stage_ms reports [0] h2d (tables and host adjacency rows), [4] graph (the import and its checks, host edge lists
 *     included: they cross PCIe in chunks under the import), [5] clique and [7] d2h; the other stages are 0.
 * The params array and the list descriptor are copied by the call. */
typedef struct qb200_graph {
  const int32_t* edges;      /* n_edges x {u, v} (the teaser::Graph::addEdge calls), or NULL */
  const uint32_t* adj;       /* L rows x words_per_row uint32, bit j of row i = edge (i, j) (qb200_max_clique's layout), or NULL */
  int64_t n_edges;           /* edges only */
  int32_t L;                 /* vertices 0 .. L-1 (Graph::populateVertices), <= max_corr */
  int32_t words_per_row;     /* adj only: >= ceil(L / 32) */
} qb200_graph;
int qb200_max_clique_batch_each(qb200_handle* h, const qb200_graph* graphs, int32_t n_graphs, const qb200_params* params,
                                qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists);
/* qb200_max_clique_batch_each, queued: completed by qb200_register_batch_flush like every enqueue, in one stream with every other
 * enqueue form.  The graphs array is read by the call; host-kind edge lists and rows, `results` and the list arrays must stay valid
 * until the flush returns.  Records and lists are byte-identical to the blocking call's. */
int qb200_max_clique_batch_enqueue_each(qb200_handle* h, const qb200_graph* graphs, int32_t n_graphs, const qb200_params* params,
                                        qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists);

/* --- TIM consistency graphs of correspondence sets in batches -------------------------------------------------------------------------
 * Quatro::computeTIMs + solveForScale + the inlier_graph_.addEdge loop (include/quatro.hpp:307-386, 784-789) for every set of a batch,
 * handed out instead of solved: for a clique or outlier solver of the caller's own, graph statistics as a loop-closure pre-filter, or
 * one graph solved in several modes by qb200_max_clique_batch_each without building it again.  Sets run in waves of max_batch_slots
 * over the lanes like every batch call.
 *   Params.  Set i is built with params[i].noise_bound and params[i].cbar2 (beta = 2 noise_bound sqrt(cbar2)), which must be > 0 as
 *     qb200_build_graph requires.  Every other field is ignored, inlier_selection_mode included: a QB200_INLIER_NONE entry still gets
 *     its graph.  Nothing is latched (rot_noise_bound is neither read nor resolved).
 *   Adjacency.  Set i's L rows at adj + i * rows_per_set * words_per_row are byte-identical to qb200_build_graph on that set alone with
 *     the same noise_bound, cbar2 and words_per_row: words ceil(L / 32) .. words_per_row - 1 are written as zero.  Rows L ..
 *     rows_per_set - 1 are left untouched.
 *   Degrees.  Set i's L entries at degree + i * rows_per_set are qb200_build_graph's degree; entries past L are left untouched.
 *   Edges.  Set i's list at edges + 2 * i * cap_edges is every edge {u, v}, u < v, in ascending (u, v) order: the sequence of the
 *     reference's inlier_graph_.addEdge calls.  min(n_edges, cap_edges) entries are written and nothing past them; a clipped list sets
 *     QB200_FLAG_LISTS_TRUNCATED in the record.
 *   Records.  status = QB200_OK for every set (L = 0 or 1 included: the graph is empty), n_corr = L, n_edges = qb200_build_graph's count,
 *     flags as above.  Nothing is solved: valid = 0, T is the identity, and every other counter and cost are 0.
 *   Equality.  No output depends on the batch, the wave, the lane, QB200_LANES, the input or output memory kinds, or the other sets.
 *   Checks run before anything starts or is queued: the set checks of qb200_solve_batch_each (L outside 0 .. max_corr, null points), a
 *     bad params entry, a NULL results or out, an unknown kind or out->kind, rows_per_set below some set's L while adj or degree is
 *     given, words_per_row < ceil(rows_per_set / 32) with adj, cap_edges < 1 with edges, and in QB200_MEM_DEVICE output kind an array
 *     that is not memory of the handle's device or is misaligned (adj and degree 4-byte, edges 8-byte).  A rejected call gives
 *     QB200_ERR_BAD_ARG, writes no record or output entry, queues nothing, and qb200_last_error names the set, entry or array; batches
 *     already queued still complete on the flush.
 *   qb200_get_stage_ms reports [0] h2d, [4] graph (K8, the degrees and the device-kind outputs) and [7] d2h; the other stages are 0.
 *   qb200_get_kernel_ms[1] counts tim_graph_kernel as a solve batch does.
 * QB200_MEM_HOST outputs are complete when the call returns (enqueue: when the flush returns); QB200_MEM_DEVICE outputs are written by the
 * call's stream work under the same rule.  The params array and the output descriptor are copied by the call.
 * {edges + 2 * i * cap_edges, NULL, n_edges, L, 0} (when n_edges <= cap_edges) and {NULL, adj + i * rows_per_set * words_per_row, 0, L,
 * words_per_row} are set i's qb200_graph for qb200_max_clique_batch_each in the same memory kind, device arrays included. */
typedef struct qb200_graph_out {
  int32_t kind;            /* qb200_mem_kind of the three arrays (QB200_MEM_DEVICE: memory of the handle's device) */
  int32_t rows_per_set;    /* adj, degree: rows reserved per set (>= every set's L when either is given) */
  int32_t words_per_row;   /* adj: >= ceil(rows_per_set / 32) */
  int32_t reserved;
  int64_t cap_edges;       /* edges: entries reserved per set (>= 1 when edges is given) */
  uint32_t* adj;           /* [n][rows_per_set][words_per_row], bit j of row i = edge (i, j): qb200_build_graph's layout, or NULL */
  int32_t* degree;         /* [n][rows_per_set], or NULL */
  int32_t* edges;          /* [n][cap_edges][2] {u, v}, u < v, or NULL */
} qb200_graph_out;
int qb200_build_graph_batch_each(qb200_handle* h, const qb200_corr_set* sets, int32_t n_sets, const qb200_params* params,
                                 qb200_mem_kind kind, qb200_result* results, const qb200_graph_out* out);
/* qb200_build_graph_batch_each, queued: completed by qb200_register_batch_flush like every enqueue, in one stream with every other
 * enqueue form, and returns without waiting for its own waves.  Host-kind sets, `results` and host-kind output arrays must stay valid
 * until the flush returns; host-kind outputs are written when their wave is collected.  Records and outputs are byte-identical to the
 * blocking call's. */
int qb200_build_graph_batch_enqueue_each(qb200_handle* h, const qb200_corr_set* sets, int32_t n_sets, const qb200_params* params,
                                         qb200_mem_kind kind, qb200_result* results, const qb200_graph_out* out);

/* --- poses of caller inlier sets in batches ------------------------------------------------------------------------------------------
 * The tail of Quatro::computeTransformation (include/quatro.hpp:806-936: chain TIMs, GNC-TLS yaw, COTE translation, the final inlier
 * list) for every set of a batch whose inliers the caller supplies: a clique of qb200_max_clique_batch_each as it lies in device
 * memory, the inliers of a clique solver or consistency filter of the caller's own, or one clique solved under several solver settings
 * (with and without the roll/pitch prior, both COTE modes, other noise bounds) without building the graph or searching the clique
 * again.  qb200_solve_pose_batch_each is qb200_solve_pose for a batch; sets run in waves of max_batch_slots over the lanes like every
 * batch call.
 *   Equality.  For every set that is not refused, the record (T, cost, gnc_iters, n_rot_inliers, n_final_inliers, clique_size, n_corr,
 *     status, valid and every other field) is byte-identical to qb200_solve_pose on that set alone with the same list and params,
 *     except for QB200_FLAG_LISTS_TRUNCATED.  The rotation and translation masks are byte-identical to what qb200_solve_pose writes,
 *     the final inliers to qb200_get_last_final_inliers after that call.  No output depends on the batch, the wave, the lane,
 *     QB200_LANES, the input or list memory kinds, or the other sets.
 *   Order.  The list is taken in the caller's order and is not sorted; duplicates are accepted, as qb200_solve_pose accepts them.  The
 *     chain TIMs follow the order of the list.  The reference sorts its clique first, so a caller who wants the reference's result
 *     passes ascending ids (qb200_max_clique_batch_each writes them ascending).
 *   Params.  Every entry must pass the checks of qb200_solve_pose.  The pose reads rot_noise_bound (0 resolves through the handle's
 *     latch in set order, enqueue order for the queued form, as in every _each form), noise_bound (for that latch), cbar2 and
 *     cote_noise_bound, rotation_gnc_factor, rotation_cost_threshold, rotation_max_iterations, cote_mode,
 *     using_rot_inliers_when_estimating_cote, use_pre_estimated_RyRx and RyRx.  The front-end, matcher and clique fields are
 *     ignored, inlier_selection_mode included: the caller supplied the inliers.
 *   Degenerate sets follow qb200_solve_pose: L < 2 gives QB200_DEGENERATE_INPUT, at most one inlier QB200_DEGENERATE_CLIQUE; the pose
 *     is the identity and the mask entries are 0.
 *   Invalid sets.  An inlier id outside [0, L) refuses that set with status QB200_ERR_BAD_ARG, in either memory kind.  This is decided
 *     on the device before the pose runs, so no point is read through such an id.  The refused set's record has valid = 0, an identity
 *     T, n_corr = L and every other field 0; it gets no list entries, and the other sets are unaffected.  (qb200_solve_pose refuses
 *     such an id for the whole call.)
 *   Lists.  As in qb200_solve_batch_ex: corr, src_matched4 and tgt_matched4 must be NULL; clique echoes the list the pose used,
 *     final_inliers and the masks are as above; clipping to cap_per_pair sets QB200_FLAG_LISTS_TRUNCATED.
 *   Checks run before anything starts or is queued: n < 0, L < 0 or L > max_corr, n_inliers < 0 or n_inliers > L, NULL points with
 *     L > 0, a NULL list with n_inliers > 0, a NULL results array, an unknown kind, a bad params entry, a bad list descriptor, and in
 *     QB200_MEM_DEVICE kind points that are not memory of the handle's device or not 16-byte aligned, or ids that are not 4-byte
 *     aligned.  A rejected call gives QB200_ERR_BAD_ARG, writes no record or list entry, queues nothing, and qb200_last_error names
 *     the set, entry or array; batches already queued still complete on the flush.
 *   qb200_get_stage_ms reports [0] h2d (points, ids and their import), [6] pose and [7] d2h; the other stages are 0.
 *     qb200_get_kernel_ms reports zeros.
 * The params array and the list descriptor are copied by the call.  A clique list of qb200_max_clique_batch_each (clique + i *
 * cap_per_pair, n_inliers = clique_size) is set i's inlier list in the same memory kind, device arrays included. */
typedef struct qb200_inlier_set {
  const float* a;          /* L x 4 floats, source side (as qb200_corr_set) */
  const float* b;          /* L x 4 floats, target side */
  const int32_t* inliers;  /* n_inliers correspondence ids, in the order the chain TIMs take them, or NULL when n_inliers == 0 */
  int32_t L;               /* <= max_corr */
  int32_t n_inliers;       /* 0 .. L */
} qb200_inlier_set;
int qb200_solve_pose_batch_each(qb200_handle* h, const qb200_inlier_set* sets, int32_t n_sets, const qb200_params* params,
                                qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists);
/* qb200_solve_pose_batch_each, queued: completed by qb200_register_batch_flush like every enqueue, in one stream with every other
 * enqueue form.  The sets array is read by the call; host-kind points and ids, `results` and the host list arrays must stay valid until
 * the flush returns.  Records and lists are byte-identical to the blocking call's. */
int qb200_solve_pose_batch_enqueue_each(qb200_handle* h, const qb200_inlier_set* sets, int32_t n_sets, const qb200_params* params,
                                        qb200_mem_kind kind, qb200_result* results, const qb200_pair_lists* lists);

/* --- multi-GPU: batches of independent pairs shard across the GPUs of one box; the only communication is ONE all-gather (NCCL over
 * NVLink) of the fixed-size result records per batch -- north_star / SURVEY.md 8(e).  The reference has no counterpart (it is a
 * single-process CPU program: examples/run_global_registration.cpp processes one pair); these entry points are what a loop-closure
 * sweep over the reference's `quatro.computeTransformation` would call instead.  libnccl.so.2 is opened at the first call
 * (QB200_ERR_UNSUPPORTED when it is absent).
 *
 * (A) one process, several devices: handles[i] was created on device i' (any distinct devices); pair g runs on handles[g mod n_dev]
 *     (QB200_MEM_DEVICE pointers of pair g must live on that device); results come back in the order of `pairs`. */
#define QB200_UNIQUE_ID_BYTES 128
int qb200_comm_init_all(qb200_handle** handles, int32_t n_dev);
int qb200_register_batch_sharded(qb200_handle** handles, int32_t n_dev, const qb200_pair* pairs, int32_t n_pairs,
                                 const qb200_params* p, qb200_mem_kind kind, qb200_result* results);
/* (B) one process per device (torchrun / mpirun): rank 0 calls qb200_comm_unique_id and hands the 128 bytes to every rank (any
 *     out-of-band channel), every rank calls qb200_comm_init_rank.  qb200_register_batch_rank registers this rank's n_local pairs
 *     (the same n_local on every rank) and gathers all records: all_results[i * world + r] = record of rank r's i-th pair
 *     (round-robin sharding of a global list).  defer != 0: the call returns as soon as the gather is enqueued on the handle's
 *     communication stream -- all_results is complete after qb200_comm_wait (or the next qb200_register_batch_rank), so the
 *     gather overlaps the next batch and no rank waits for the slowest one inside a step.  defer == 2 (a stream of batches): the
 *     local batch is only queued (qb200_register_batch_enqueue), the call then completes the PREVIOUS batch's records and starts
 *     their gather; local_pairs' scans and all_results of a batch must stay valid until its records were delivered (two calls
 *     later, or qb200_comm_wait, which ends the stream). */
int qb200_comm_unique_id(void* id128);
int qb200_comm_init_rank(qb200_handle* h, int32_t world, int32_t rank, const void* id128);
int qb200_register_batch_rank(qb200_handle* h, const qb200_pair* local_pairs, int32_t n_local, const qb200_params* p,
                              qb200_mem_kind kind, qb200_result* all_results, int32_t defer);
int qb200_comm_wait(qb200_handle* h);
/* Bind the calling host thread to the cores of the NUMA node of the handle's GPU (kernel launches and pinned copies from the far
 * socket of a 2-socket box are slower).  Returns the number of cores bound (0: topology unknown, nothing changed). */
int qb200_bind_numa(qb200_handle* h);

/* Introspection of the most recent single-pair solve on this handle (getMaxCliques,
 * getFinalInliersIndices, getCorrespondences; quatro.hpp:949-972, fpfh_manager.hpp:234-236). */
int qb200_get_last_clique(qb200_handle* h, int32_t* idx, int32_t cap, int32_t* n);
int qb200_get_last_final_inliers(qb200_handle* h, int32_t* idx, int32_t cap, int32_t* n);
int qb200_get_last_correspondences(qb200_handle* h, int32_t* corr, float* src_matched4,
                                   float* tgt_matched4, int32_t cap, int32_t* n);

/* Normals (n x {nx,ny,nz,curvature}) and FPFH-33 descriptors (n x 33) the most recent qb200_match_and_pack (which = 0 source,
 * 1 target) or qb200_compute_fpfh (which = 0) left on the device: FPFHManager::getObjDescriptor / getSceneDescriptor /
 * getTgtNormals (include/fpfh_manager.hpp:161-177).  Either pointer may be NULL. */
int qb200_get_last_features(qb200_handle* h, int32_t which, float* normals4, float* desc33, int32_t cap, int32_t* n);

/* Per-stage device time of the last batch call in milliseconds (CUDA events); the single-pair registration and solve are batches
 * of one: [0]=h2d [1]=voxel [2]=fpfh [3]=match [4]=graph [5]=clique [6]=pose [7]=d2h; n<=8.  The times start from zero with every
 * call that finds nothing queued, and qb200_cache_scans{,_each} count as batch calls that register nothing: right after one of them
 * (or after a flush of queued cache writes alone) this and qb200_get_kernel_ms report zeros, not the previous batch's times. */
int qb200_get_stage_ms(qb200_handle* h, float* ms, int32_t n);

/* Device time (CUDA events on the handle's stream) and launch count of the two roofline kernels
 * during the last batch call: [0] = the tensor-core nearest-neighbour passes (tc_match_kernel x3),
 * [1] = tim_graph_kernel (TIM consistency graph); n <= 2.  Zeros after a cache write, as qb200_get_stage_ms. */
int qb200_get_kernel_ms(qb200_handle* h, float* ms, int32_t* launches, int32_t n);

/* Diagnostics: the tensor-core (wgmma, 3xTF32) approximate squared distances that pre-filter the 33-D
 * nearest-neighbour search, for up to 128 x 128 descriptors (out[128*128], row = a).  The matcher's results
 * never depend on these values (exact fp32 re-rank); tests use this to measure the filter's error margin. */
int qb200_debug_tc_distances(qb200_handle* h, const float* a33, int32_t na, const float* b33, int32_t nb, float* out);


/* Diagnostics: cumulative counters of the tensor-core matcher since creation / the last reset:
 * out4[0] = descriptor pairs that went through the exact fp32 chain, [1] = 128 x 64 tiles drained,
 * [2] = 0 (unused), [3] = stripes handed to the exact kernel.  Synchronises the handle's stream. */
int qb200_debug_match_stats(qb200_handle* h, uint64_t* out4, int32_t reset);
/* Diagnostics: both nearest-neighbour tables of the most recent qb200_match, in point order: rowbest[i] = packed
 * (distance bits << 32 | target index) of the best target of source point i, colbest[j] = the same for the best source of target
 * point j, ~0 = none.  min(cap_rows, n_src) and min(cap_cols, n_tgt) entries are written (either pointer may be NULL); the
 * tables are those the mutual check read, after any stripe was redone by the exact kernel.  Synchronises the handle's stream. */
int qb200_debug_nn_tables(qb200_handle* h, uint64_t* rowbest, int32_t cap_rows, uint64_t* colbest, int32_t cap_cols);
/* Handles created with QB200_TC_PROF=1 only: per-role clock64 accounting of tc_nn_kernel (24 counters, see tools/tc_profile.py) */
int qb200_debug_tc_profile(qb200_handle* h, uint64_t* out24, int32_t reset);
/* Diagnostics: footprint of the tensor-core nearest-neighbour kernel as launched: out5[0] = threads per CTA,
 * [1] = dynamic shared bytes, [2] = static shared bytes, [3] = registers per thread, [4] = resident CTAs per SM. */
int qb200_debug_tc_footprint(qb200_handle* h, int32_t* out5);

/* Diagnostics: on a handle created with QB200_TC_VERIFY=1 every batch is matched by the tensor-core path AND by the exact CUDA-core
 * kernel; out2[0] = nearest-neighbour table entries compared so far, out2[1] = entries whose packed (distance, index) differ
 * (0 unless the filter's error bound is violated).  Synchronises the handle's stream. */
int qb200_debug_match_verify(qb200_handle* h, uint64_t* out2, int32_t reset);

#ifdef __cplusplus
}
#endif
#endif /* QUATRO_B200_H_ */
