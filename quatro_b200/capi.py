"""ctypes binding of include/quatro_b200.h (one Python method per C entry point).

Used by tests/ and bench.py; mirrors the C-ABI 1:1 so the parity tests read like calls a C/C++
caller (the reference's run_global_registration.cpp) would make.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np

from . import _build

PMC_EXACT, PMC_HEU, KCORE_HEU, INLIER_NONE = 0, 1, 2, 3
FLAG_CLIQUE_TRUNCATED = 1
FLAG_LISTS_TRUNCATED = 2
COTE_MEDIAN, COTE_WEIGHTED_MEAN = 0, 1
MEM_HOST, MEM_DEVICE = 0, 1

STATUS_NAMES = {0: "OK", 1: "DEGENERATE_CLIQUE", 2: "DEGENERATE_INPUT", 3: "CAPACITY_EXCEEDED", -1: "ERR_BAD_ARG",
                -2: "ERR_NO_DEVICE", -3: "ERR_CUDA", -4: "ERR_UNSUPPORTED", -5: "ERR_VOXEL_OVERFLOW"}


class Params(C.Structure):
    _fields_ = [
        ("voxel_size", C.c_float), ("normal_radius", C.c_float), ("fpfh_radius", C.c_float), ("grid_cell", C.c_float),
        ("tuple_scale", C.c_float), ("use_crosscheck", C.c_int32), ("use_tuple_test", C.c_int32),
        ("tuple_trials_per_corr", C.c_int32), ("skip_flagged", C.c_int32), ("reserved0", C.c_int32),
        ("seed", C.c_uint64),
        ("noise_bound", C.c_double), ("cbar2", C.c_double), ("rot_noise_bound", C.c_double),
        ("cote_noise_bound", C.c_double), ("rotation_gnc_factor", C.c_double),
        ("rotation_cost_threshold", C.c_double), ("kcore_heuristic_threshold", C.c_double),
        ("rotation_max_iterations", C.c_int32), ("inlier_selection_mode", C.c_int32), ("cote_mode", C.c_int32),
        ("using_rot_inliers_when_estimating_cote", C.c_int32), ("use_pre_estimated_RyRx", C.c_int32),
        ("max_clique_node_limit", C.c_int32), ("RyRx", C.c_double * 9),
    ]


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("max_batch_slots", C.c_int32), ("max_raw_points", C.c_int32),
                ("max_voxel_points", C.c_int32), ("max_corr", C.c_int32), ("reserved", C.c_int32 * 3)]


class Result(C.Structure):
    _fields_ = [
        ("valid", C.c_int32), ("status", C.c_int32), ("n_src_vox", C.c_int32), ("n_tgt_vox", C.c_int32),
        ("n_mutual", C.c_int32), ("n_corr", C.c_int32), ("max_core", C.c_int32), ("clique_size", C.c_int32),
        ("gnc_iters", C.c_int32), ("n_rot_inliers", C.c_int32), ("n_final_inliers", C.c_int32),
        ("flags", C.c_int32), ("n_edges", C.c_int64), ("cost", C.c_double), ("T", C.c_double * 16),
    ]

    def matrix(self) -> np.ndarray:
        """4x4 pose (row/col indexing as usual); T is stored column-major."""
        return np.array(self.T[:], dtype=np.float64).reshape(4, 4).T.copy()

    def as_dict(self) -> dict:
        d = {k: getattr(self, k) for k, _ in self._fields_ if k != "T"}
        d["T"] = self.matrix()
        return d


class PatchworkParams(C.Structure):
    """qb200_patchwork_params (config/patchwork_params.yaml of the reference)."""
    _fields_ = [
        ("sensor_height", C.c_double), ("th_seeds", C.c_double), ("th_dist", C.c_double), ("max_range", C.c_double),
        ("min_range", C.c_double), ("uprightness_thr", C.c_double), ("adaptive_seed_selection_margin", C.c_double),
        ("global_elevation_threshold", C.c_double), ("min_ranges_each_zone", C.c_double * 4),
        ("elevation_thresholds", C.c_double * 8), ("flatness_thresholds", C.c_double * 8),
        ("num_iter", C.c_int32), ("num_lpr", C.c_int32), ("num_min_pts", C.c_int32), ("using_global_elevation", C.c_int32),
        ("num_zones", C.c_int32), ("num_thresholds", C.c_int32), ("num_sectors_each_zone", C.c_int32 * 4),
        ("num_rings_each_zone", C.c_int32 * 4),
    ]


class SegmentParams(C.Structure):
    """qb200_segment_params (per-sensor constants of the ImageProjection constructor)."""
    _fields_ = [("n_scan", C.c_int32), ("horizon_scan", C.c_int32), ("ang_res_x", C.c_float), ("ang_res_y", C.c_float),
                ("ang_bottom", C.c_float), ("segment_theta", C.c_float), ("neighbor_mode", C.c_int32),
                ("min_pts_for_subclustering", C.c_int32), ("segment_valid_point_num", C.c_int32), ("segment_valid_line_num", C.c_int32)]


class Pair(C.Structure):
    _fields_ = [("src", C.c_void_p), ("tgt", C.c_void_p), ("n_src", C.c_int32), ("n_tgt", C.c_int32)]


class FeaturePair(C.Structure):
    """qb200_feature_pair: one pair's keypoints ({x,y,z,w} records) and FPFH-33 descriptor rows."""
    _fields_ = [("src", C.c_void_p), ("src_desc", C.c_void_p), ("tgt", C.c_void_p), ("tgt_desc", C.c_void_p), ("n_src", C.c_int32),
                ("n_tgt", C.c_int32)]


class DescriptorPair(C.Structure):
    """qb200_descriptor_pair: one pair's keypoints ({x,y,z,w} records) and descriptor rows of `stride` floats, the first `dim` of
    which are the descriptor (1 <= dim <= DESC_DIM_MAX)."""
    _fields_ = [("src", C.c_void_p), ("src_desc", C.c_void_p), ("tgt", C.c_void_p), ("tgt_desc", C.c_void_p), ("n_src", C.c_int32),
                ("n_tgt", C.c_int32), ("dim", C.c_int32), ("stride", C.c_int32)]


DESC_DIM_MAX = 512   # QB200_MAX_DESC_DIM


class CorrSet(C.Structure):
    _fields_ = [("a", C.c_void_p), ("b", C.c_void_p), ("L", C.c_int32), ("reserved", C.c_int32)]


class Graph(C.Structure):
    """qb200_graph: one caller graph of qb200_max_clique_batch_each, as an edge list or as adjacency rows (one of the two, or neither
    for a graph without edges)."""
    _fields_ = [("edges", C.c_void_p), ("adj", C.c_void_p), ("n_edges", C.c_int64), ("L", C.c_int32), ("words_per_row", C.c_int32)]


class InlierSet(C.Structure):
    """qb200_inlier_set: one set of qb200_solve_pose_batch_each, its matched points and the caller's inlier ids (in chain order)."""
    _fields_ = [("a", C.c_void_p), ("b", C.c_void_p), ("inliers", C.c_void_p), ("L", C.c_int32), ("n_inliers", C.c_int32)]


class AlignSet(C.Structure):
    """qb200_align_set: one registered pair of qb200_align_batch_each: the cloud to align, the voxel keypoints of both sides, the
    correspondences between them and the pose (column-major, as Result.T)."""
    _fields_ = [("cloud", C.c_void_p), ("src_kp", C.c_void_p), ("tgt_kp", C.c_void_p), ("corr", C.c_void_p), ("n_points", C.c_int32),
                ("n_src", C.c_int32), ("n_tgt", C.c_int32), ("n_corr", C.c_int32), ("T", C.c_double * 16)]


class AlignOut(C.Structure):
    """qb200_align_out: caller-owned outputs of qb200_align_batch_each, cap_points aligned points and cap_corr entries of each
    correspondence array reserved per set."""
    _fields_ = [("cap_points", C.c_int32), ("cap_corr", C.c_int32), ("kind", C.c_int32), ("reserved", C.c_int32),
                ("aligned4", C.c_void_p), ("matched4", C.c_void_p), ("good_ids", C.c_void_p), ("good4", C.c_void_p),
                ("counts", C.c_void_p), ("status", C.c_void_p)]


ALIGN_ARRAYS = {"aligned4": (np.float32, (4,)), "matched4": (np.float32, (4,)), "good_ids": (np.int32, ()), "good4": (np.float32, (4,))}


class GraphOut(C.Structure):
    """qb200_graph_out: caller-owned outputs of qb200_build_graph_batch_each: adjacency rows, degrees and edge lists of every set."""
    _fields_ = [("kind", C.c_int32), ("rows_per_set", C.c_int32), ("words_per_row", C.c_int32), ("reserved", C.c_int32),
                ("cap_edges", C.c_int64), ("adj", C.c_void_p), ("degree", C.c_void_p), ("edges", C.c_void_p)]


class PairLists(C.Structure):
    """qb200_pair_lists: caller-owned per-pair lists of the batch entry points, cap_per_pair entries reserved per pair."""
    _fields_ = [("cap_per_pair", C.c_int32), ("kind", C.c_int32), ("corr", C.c_void_p), ("src_matched4", C.c_void_p),
                ("tgt_matched4", C.c_void_p), ("clique", C.c_void_p), ("final_inliers", C.c_void_p),
                ("rot_inlier_mask", C.c_void_p), ("trans_inlier_mask", C.c_void_p)]


class PreprocessOut(C.Structure):
    """qb200_preprocess_out: caller-owned outputs of qb200_preprocess_batch, cap_per_scan points reserved per scan."""
    _fields_ = [("cap_per_scan", C.c_int32), ("kind", C.c_int32), ("ground4", C.c_void_p), ("nonground4", C.c_void_p),
                ("valid4", C.c_void_p), ("outlier4", C.c_void_p), ("counts", C.c_void_p), ("status", C.c_void_p)]


PREPROCESS_ARRAYS = ("ground4", "nonground4", "valid4", "outlier4")   # in the order of the four counts


class FeatureOut(C.Structure):
    """qb200_feature_out: caller-owned outputs of qb200_describe_batch_each, qb200_describe_points_each and qb200_voxelize_batch_each,
    cap_per_scan keypoints reserved per scan or cloud."""
    _fields_ = [("cap_per_scan", C.c_int32), ("kind", C.c_int32), ("vox4", C.c_void_p), ("normals4", C.c_void_p), ("desc33", C.c_void_p),
                ("counts", C.c_void_p), ("status", C.c_void_p)]


FEATURE_ARRAYS = {"vox4": 4, "normals4": 4, "desc33": 33}   # output array -> floats per keypoint
POINT_ARRAYS = ("normals4", "desc33")   # what qb200_describe_points_each can return (the keypoints are the caller's own)
VOXEL_ARRAYS = ("vox4",)   # what qb200_voxelize_batch_each can return


# list name -> (element dtype, trailing shape, count field of the record)
LIST_LAYOUT = {
    "corr": (np.int32, (2,), "n_corr"),
    "src_matched4": (np.float32, (4,), "n_corr"),
    "tgt_matched4": (np.float32, (4,), "n_corr"),
    "clique": (np.int32, (), "clique_size"),
    "final_inliers": (np.int32, (), "n_final_inliers"),
    "rot_inlier_mask": (np.uint8, (), "clique_size"),
    "trans_inlier_mask": (np.uint8, (), "clique_size"),
}
SET_LISTS = ("clique", "final_inliers", "rot_inlier_mask", "trans_inlier_mask")   # what qb200_solve_batch_ex can return
MATCH_LISTS = ("corr", "src_matched4", "tgt_matched4")   # what the qb200_match_* calls can return
GRAPH_LISTS = ("clique",)   # what qb200_max_clique_batch_each can return


class ListBuffers:
    """The arrays of one qb200_pair_lists: zeroed numpy arrays (MEM_HOST) or CUDA tensors of `device` (MEM_DEVICE), each of shape
    (n, cap, *trailing)."""

    def __init__(self, n: int, cap: int, kind: int = MEM_HOST, lists: Sequence[str] = tuple(LIST_LAYOUT), device: int = 0):
        self.n, self.cap, self.kind = n, cap, kind
        self.arrays = {}
        for name in lists:
            dt, tail, _ = LIST_LAYOUT[name]
            shape = (max(n, 1), cap, *tail)
            if kind == MEM_HOST:
                self.arrays[name] = np.zeros(shape, dt)
            else:
                import torch
                self.arrays[name] = torch.zeros(shape, dtype=getattr(torch, np.dtype(dt).name), device=f"cuda:{device}")

    def descriptor(self) -> PairLists:
        d = PairLists(self.cap, self.kind)
        for name, a in self.arrays.items():
            setattr(d, name, a.ctypes.data if self.kind == MEM_HOST else a.data_ptr())
        return d

    def host(self, name: str) -> np.ndarray:
        a = self.arrays[name]
        return a if self.kind == MEM_HOST else a.cpu().numpy()

    def trimmed(self, records: np.ndarray) -> list:
        """Per pair a dict of its lists cut to min(count, cap) entries (numpy copies, or tensor views on the device); a pair whose status
        is CAPACITY_EXCEEDED gets empty lists."""
        out = []
        for i, r in enumerate(records):
            d = {}
            for name, a in self.arrays.items():
                m = 0 if r["status"] == 3 else min(int(r[LIST_LAYOUT[name][2]]), self.cap)
                d[name] = a[i, :m].copy() if self.kind == MEM_HOST else a[i, :m]
            out.append(d)
        return out


class GraphBuffers:
    """The arrays of one qb200_graph_out: numpy arrays (MEM_HOST) or CUDA tensors of `device` (MEM_DEVICE, adj held as int32), filled
    with `fill`: adj (n, rows_per_set, words_per_row) uint32, degree (n, rows_per_set) int32, edges (n, cap_edges, 2) int32."""
    SHAPES = {"adj": (np.uint32, lambda b: (b.rows_per_set, b.words_per_row)), "degree": (np.int32, lambda b: (b.rows_per_set,)),
              "edges": (np.int32, lambda b: (b.cap_edges, 2))}

    def __init__(self, n: int, rows_per_set: int, words_per_row: int, cap_edges: int, kind: int = MEM_HOST,
                 arrays: Sequence[str] = ("adj", "degree", "edges"), device: int = 0, fill: int = 0):
        self.n, self.rows_per_set, self.words_per_row, self.cap_edges, self.kind = n, rows_per_set, words_per_row, cap_edges, kind
        self.arrays = {}
        for name in arrays:
            dt, shape = self.SHAPES[name]
            a = np.full((max(n, 1), *shape(self)), fill, np.int64).astype(dt)
            if kind == MEM_HOST:
                self.arrays[name] = a
            else:
                import torch
                self.arrays[name] = torch.from_numpy(a.view(np.int32)).to(f"cuda:{device}")

    def descriptor(self) -> GraphOut:
        d = GraphOut(self.kind, self.rows_per_set, self.words_per_row, 0, self.cap_edges)
        for name, a in self.arrays.items():
            setattr(d, name, a.ctypes.data if self.kind == MEM_HOST else a.data_ptr())
        return d

    def host(self, name: str) -> np.ndarray:
        """the array as numpy (a copy of a device array), adj as uint32"""
        a = self.arrays[name]
        a = a if self.kind == MEM_HOST else a.cpu().numpy()
        return a.view(self.SHAPES[name][0])

    def graphs(self, records: np.ndarray, use: str = "edges") -> list:
        """Per set the Graph that qb200_max_clique_batch_each takes, in this kind: its edge list (use="edges"; a clipped list is
        refused) or its adjacency rows (use="adj")."""
        a = self.arrays[use]
        base = a.ctypes.data if self.kind == MEM_HOST else a.data_ptr()
        out = []
        for i, r in enumerate(records):
            L = int(r["n_corr"])
            if use == "edges":
                assert not r["flags"] & FLAG_LISTS_TRUNCATED, f"set {i}: its edge list was clipped to cap_edges"
                out.append(Graph(base + 8 * i * self.cap_edges, None, int(r["n_edges"]), L, 0))
            else:
                out.append(Graph(None, base + 4 * i * self.rows_per_set * self.words_per_row, 0, L, self.words_per_row))
        return out


RESULT_DTYPE = np.dtype([
    ("valid", "<i4"), ("status", "<i4"), ("n_src_vox", "<i4"), ("n_tgt_vox", "<i4"), ("n_mutual", "<i4"),
    ("n_corr", "<i4"), ("max_core", "<i4"), ("clique_size", "<i4"), ("gnc_iters", "<i4"), ("n_rot_inliers", "<i4"),
    ("n_final_inliers", "<i4"), ("flags", "<i4"), ("n_edges", "<i8"), ("cost", "<f8"), ("T", "<f8", (16,)),
])
assert RESULT_DTYPE.itemsize == C.sizeof(Result)


class QuatroB200Error(RuntimeError):
    def __init__(self, code: int, where: str, detail: str = ""):
        self.code = code
        super().__init__(f"{where}: {STATUS_NAMES.get(code, code)} {detail}")


# restype and argtypes of every function include/quatro_b200.h declares
vp, i32, i64, f32, f64, P = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_double, C.POINTER
_SIGNATURES = {
    "qb200_default_params": (None, [P(Params)]),
    "qb200_default_config": (None, [P(Config)]),
    "qb200_version": (i32, []),
    "qb200_create": (i32, [P(Config), P(vp)]),
    "qb200_destroy": (None, [vp]),
    "qb200_set_stream": (i32, [vp, vp]),
    "qb200_last_error": (C.c_char_p, [vp]),
    "qb200_launch_count": (i64, [vp]),
    "qb200_voxelize": (i32, [vp, vp, i32, f32, i32, vp, i32, P(i32)]),
    "qb200_default_patchwork_params": (None, [P(PatchworkParams)]),
    "qb200_default_segment_params": (None, [P(SegmentParams)]),
    "qb200_segment_cloud": (i32, [vp, vp, i32, P(SegmentParams), vp, P(i32), vp, P(i32)]),
    "qb200_patchwork": (i32, [vp, vp, i32, P(PatchworkParams), vp, P(i32), vp, P(i32)]),
    "qb200_compute_fpfh": (i32, [vp, vp, i32, f32, f32, f32, vp, vp]),
    "qb200_match": (i32, [vp, vp, i32, vp, vp, i32, vp, P(Params), vp, i32, P(i32), P(i32)]),
    "qb200_build_graph": (i32, [vp, vp, vp, i32, f64, f64, vp, i32, vp, P(i64)]),
    "qb200_max_clique": (i32, [vp, vp, i32, i32, i32, f64, vp, P(i32), vp, vp, P(i32)]),
    "qb200_max_clique_ex": (i32, [vp, vp, i32, i32, i32, f64, i64, vp, P(i32), vp, vp, P(i32), P(i32)]),
    "qb200_solve_pose": (i32, [vp, vp, vp, i32, vp, i32, P(Params), P(Result), vp, vp]),
    "qb200_solve_correspondences": (i32, [vp, vp, vp, i32, P(Params), P(Result)]),
    "qb200_match_and_pack": (i32, [vp, vp, i32, vp, i32, P(Params), vp, vp, vp, i32, P(i32)]),
    "qb200_register_pair": (i32, [vp, vp, i32, vp, i32, P(Params), P(Result)]),
    "qb200_register_batch": (i32, [vp, P(Pair), i32, P(Params), i32, vp]),
    "qb200_get_last_clique": (i32, [vp, vp, i32, P(i32)]),
    "qb200_get_last_final_inliers": (i32, [vp, vp, i32, P(i32)]),
    "qb200_get_last_correspondences": (i32, [vp, vp, vp, vp, i32, P(i32)]),
    "qb200_get_stage_ms": (i32, [vp, vp, i32]),
    "qb200_get_kernel_ms": (i32, [vp, vp, vp, i32]),
    "qb200_debug_tc_distances": (i32, [vp, vp, i32, vp, i32, vp]),
    "qb200_debug_match_stats": (i32, [vp, vp, i32]),
    "qb200_debug_nn_tables": (i32, [vp, vp, i32, vp, i32]),
    "qb200_register_batch_enqueue": (i32, [vp, vp, i32, vp, i32, vp]),
    "qb200_register_batch_flush": (i32, [vp]),
    "qb200_debug_tc_profile": (i32, [vp, vp, i32]),
    "qb200_debug_tc_footprint": (i32, [vp, vp]),
    "qb200_solve_batch": (i32, [vp, vp, i32, vp, i32, vp]),
    "qb200_comm_init_all": (i32, [P(vp), i32]),
    "qb200_register_batch_sharded": (i32, [P(vp), i32, P(Pair), i32, P(Params), i32, vp]),
    "qb200_comm_unique_id": (i32, [vp]),
    "qb200_comm_init_rank": (i32, [vp, i32, i32, vp]),
    "qb200_register_batch_rank": (i32, [vp, P(Pair), i32, P(Params), i32, vp, i32]),
    "qb200_comm_wait": (i32, [vp]),
    "qb200_bind_numa": (i32, [vp]),
    "qb200_debug_match_verify": (i32, [vp, vp, i32]),
    "qb200_get_last_features": (i32, [vp, i32, vp, vp, i32, P(i32)]),
    "qb200_cache_reserve": (i32, [vp, i32]),
    "qb200_cache_scans": (i32, [vp, P(vp), P(i32), P(i32), i32, P(Params), i32]),
    "qb200_register_cached": (i32, [vp, vp, i32, P(Params), vp]),
    "qb200_cache_copy": (i32, [vp, i32, i32]),
    "qb200_cache_read": (i32, [vp, i32, vp, vp, vp, i32, P(i32)]),
    "qb200_register_batch_ex": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_register_batch_enqueue_ex": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_register_cached_ex": (i32, [vp, vp, i32, P(Params), vp, P(PairLists)]),
    "qb200_solve_batch_ex": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_preprocess_batch": (i32, [vp, vp, vp, i32, i32, P(PatchworkParams), P(SegmentParams), P(PreprocessOut)]),
    "qb200_register_batch_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_register_batch_enqueue_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_register_cached_each": (i32, [vp, vp, i32, P(Params), vp, P(PairLists)]),
    "qb200_solve_batch_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_preprocess_batch_each": (i32, [vp, vp, vp, i32, i32, P(PatchworkParams), P(SegmentParams), P(PreprocessOut)]),
    "qb200_register_batch_mixed": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_register_batch_enqueue_mixed": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_register_cached_mixed": (i32, [vp, vp, i32, P(Params), vp, P(PairLists)]),
    "qb200_cache_scans_each": (i32, [vp, P(vp), P(i32), P(i32), i32, P(Params), i32]),
    "qb200_register_cached_enqueue_mixed": (i32, [vp, vp, i32, P(Params), vp, P(PairLists)]),
    "qb200_solve_batch_enqueue_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_cache_scans_enqueue_each": (i32, [vp, P(vp), P(i32), P(i32), i32, P(Params), i32]),
    "qb200_register_features_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_register_features_enqueue_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_describe_batch_each": (i32, [vp, P(vp), P(i32), i32, P(Params), i32, P(FeatureOut)]),
    "qb200_describe_batch_enqueue_each": (i32, [vp, P(vp), P(i32), i32, P(Params), i32, P(FeatureOut)]),
    "qb200_voxelize_batch_each": (i32, [vp, P(vp), P(i32), i32, P(Params), i32, P(FeatureOut)]),
    "qb200_voxelize_batch_enqueue_each": (i32, [vp, P(vp), P(i32), i32, P(Params), i32, P(FeatureOut)]),
    "qb200_describe_points_each": (i32, [vp, P(vp), P(i32), i32, P(Params), i32, P(FeatureOut)]),
    "qb200_describe_points_enqueue_each": (i32, [vp, P(vp), P(i32), i32, P(Params), i32, P(FeatureOut)]),
    "qb200_match_batch_mixed": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_match_batch_enqueue_mixed": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_match_cached_mixed": (i32, [vp, vp, i32, P(Params), vp, P(PairLists)]),
    "qb200_match_cached_enqueue_mixed": (i32, [vp, vp, i32, P(Params), vp, P(PairLists)]),
    "qb200_match_features_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_match_features_enqueue_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_match_descriptors_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_match_descriptors_enqueue_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_register_descriptors_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_register_descriptors_enqueue_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_max_clique_batch_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_max_clique_batch_enqueue_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_build_graph_batch_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(GraphOut)]),
    "qb200_build_graph_batch_enqueue_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(GraphOut)]),
    "qb200_solve_pose_batch_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_solve_pose_batch_enqueue_each": (i32, [vp, vp, i32, P(Params), i32, vp, P(PairLists)]),
    "qb200_align_batch_each": (i32, [vp, vp, i32, P(Params), i32, P(AlignOut)]),
    "qb200_align_batch_enqueue_each": (i32, [vp, vp, i32, P(Params), i32, P(AlignOut)]),
}
del vp, i32, i64, f32, f64, P
EXPORTED_SYMBOLS = list(_SIGNATURES)


_LIB: Optional[C.CDLL] = None


def _f32(a, cols=None) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.float32)
    if cols is not None:
        assert a.ndim == 2 and a.shape[1] == cols, (a.shape, cols)
    return a


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


# ---- the ctypes input arrays of the batch calls: each returns the array and what must stay alive while it is in use ----
def _pair_array(pairs: Sequence, kind: int = MEM_HOST):
    """(Pair * n) array of `pairs`: (src, tgt) numpy arrays (MEM_HOST) or (src_ptr, n_src, tgt_ptr, n_tgt) device tuples (MEM_DEVICE);
    and the contiguous scans it points to."""
    arr = (Pair * len(pairs))()
    keep = []
    for i, pr in enumerate(pairs):
        if kind == MEM_HOST:
            s, t = _f32(pr[0], 4), _f32(pr[1], 4)
            keep.append((s, t))
            arr[i].src, arr[i].n_src, arr[i].tgt, arr[i].n_tgt = s.ctypes.data, len(s), t.ctypes.data, len(t)
        else:
            arr[i].src, arr[i].n_src, arr[i].tgt, arr[i].n_tgt = pr[0], pr[1], pr[2], pr[3]
    return arr, keep


def _set_array(sets: Sequence, kind: int):
    """(CorrSet * n) array of `sets`: (a4, b4) numpy arrays (MEM_HOST) or (a_ptr, b_ptr, L) device tuples (MEM_DEVICE); and the
    contiguous points it points to."""
    arr = (CorrSet * len(sets))()
    keep = []
    for i, st in enumerate(sets):
        if kind == MEM_HOST:
            a, b = _f32(st[0], 4), _f32(st[1], 4)
            assert len(a) == len(b)
            keep.append((a, b))
            arr[i].a, arr[i].b, arr[i].L = a.ctypes.data, b.ctypes.data, len(a)
        else:
            arr[i].a, arr[i].b, arr[i].L = st[0], st[1], st[2]
    return arr, keep


def _feature_array(pairs: Sequence, kind: int = MEM_HOST):
    """(FeaturePair * n) array of `pairs`: (src4, src_desc, tgt4, tgt_desc) numpy arrays (MEM_HOST) or (src_ptr, src_desc_ptr, n_src,
    tgt_ptr, tgt_desc_ptr, n_tgt) device tuples (MEM_DEVICE); and the contiguous arrays it points to."""
    arr = (FeaturePair * max(len(pairs), 1))()
    keep = []
    for i, pr in enumerate(pairs):
        if kind == MEM_HOST:
            s, sd, t, td = _f32(pr[0], 4), _f32(pr[1], 33), _f32(pr[2], 4), _f32(pr[3], 33)
            assert len(s) == len(sd) and len(t) == len(td)
            keep.append((s, sd, t, td))
            arr[i].src, arr[i].src_desc, arr[i].n_src = s.ctypes.data, sd.ctypes.data, len(s)
            arr[i].tgt, arr[i].tgt_desc, arr[i].n_tgt = t.ctypes.data, td.ctypes.data, len(t)
        else:
            arr[i].src, arr[i].src_desc, arr[i].n_src, arr[i].tgt, arr[i].tgt_desc, arr[i].n_tgt = pr
    return arr, keep


def _descriptor_array(pairs: Sequence, kind: int = MEM_HOST):
    """(DescriptorPair * n) array of `pairs`, each a DescriptorPair (pointers of any kind, used as they are), (src4, src_rows, tgt4,
    tgt_rows[, dim]) numpy arrays with rows of `stride` = rows.shape[1] floats (dim defaults to the stride; MEM_HOST), or (src_ptr,
    src_desc_ptr, n_src, tgt_ptr, tgt_desc_ptr, n_tgt, dim, stride) device tuples (MEM_DEVICE); and the contiguous arrays it points
    to."""
    arr = (DescriptorPair * max(len(pairs), 1))()
    keep = []
    for i, pr in enumerate(pairs):
        if isinstance(pr, DescriptorPair):
            arr[i] = pr
        elif kind == MEM_HOST:
            s, t = _f32(pr[0], 4), _f32(pr[2], 4)
            sd, td = np.ascontiguousarray(pr[1], np.float32), np.ascontiguousarray(pr[3], np.float32)
            assert sd.ndim == td.ndim == 2 and sd.shape[1] == td.shape[1] and len(s) == len(sd) and len(t) == len(td)
            stride = sd.shape[1]
            keep.append((s, sd, t, td))
            arr[i].src, arr[i].src_desc, arr[i].n_src = s.ctypes.data, sd.ctypes.data, len(s)
            arr[i].tgt, arr[i].tgt_desc, arr[i].n_tgt = t.ctypes.data, td.ctypes.data, len(t)
            arr[i].dim, arr[i].stride = (pr[4] if len(pr) > 4 else stride), stride
        else:
            (arr[i].src, arr[i].src_desc, arr[i].n_src, arr[i].tgt, arr[i].tgt_desc, arr[i].n_tgt, arr[i].dim, arr[i].stride) = pr
    return arr, keep


def _graph_array(graphs: Sequence):
    """(Graph * n) array of `graphs`: each a Graph (pointers of any kind, used as they are), a (L, wpr) uint32 adjacency array, or an
    (L, edges) tuple with an (m, 2) int32 edge array; and the contiguous host arrays it points to."""
    arr = (Graph * max(len(graphs), 1))()
    keep = []
    for i, g in enumerate(graphs):
        if isinstance(g, Graph):
            arr[i] = g
        elif isinstance(g, tuple):
            L, e = g
            e = np.ascontiguousarray(np.asarray(e, np.int32).reshape(-1, 2))
            keep.append(e)
            arr[i].edges, arr[i].n_edges, arr[i].L = (e.ctypes.data if len(e) else None), len(e), L
        else:
            a = np.ascontiguousarray(g, np.uint32)
            keep.append(a)
            arr[i].adj, arr[i].L, arr[i].words_per_row = (a.ctypes.data if a.size else None), a.shape[0], a.shape[1]
    return arr, keep


def _inlier_array(sets: Sequence, inliers: Sequence, kind: int):
    """(InlierSet * n) array of `sets` (as _set_array takes them) with inliers[i] as set i's ids: an int array (MEM_HOST) or a
    (ids_ptr, n_inliers) device tuple (MEM_DEVICE); and the contiguous host arrays it points to."""
    assert len(inliers) == len(sets)
    arr = (InlierSet * max(len(sets), 1))()
    pts, keep = _set_array(sets, kind)
    for i, ids in enumerate(inliers):
        arr[i].a, arr[i].b, arr[i].L = pts[i].a, pts[i].b, pts[i].L
        if kind == MEM_HOST:
            ids = np.ascontiguousarray(ids, np.int32).reshape(-1)
            keep.append(ids)
            arr[i].inliers, arr[i].n_inliers = (ids.ctypes.data if len(ids) else None), len(ids)
        else:
            arr[i].inliers, arr[i].n_inliers = ids[0], ids[1]
    return arr, keep


def _align_array(sets: Sequence, kind: int):
    """(AlignSet * n) array of `sets`: each a dict with cloud, src_kp, tgt_kp ((n,4) float32), corr ((m,2) int32) and T (4x4, row-major
    as Result.matrix() gives it) for MEM_HOST, or with (device_ptr, n) tuples in place of the arrays for MEM_DEVICE (cloud may be None);
    and the contiguous host arrays it points to."""
    arr = (AlignSet * max(len(sets), 1))()
    keep = []
    for i, st in enumerate(sets):
        e = arr[i]
        for name, count, cols, dt in (("cloud", "n_points", 4, np.float32), ("src_kp", "n_src", 4, np.float32),
                                      ("tgt_kp", "n_tgt", 4, np.float32), ("corr", "n_corr", 2, np.int32)):
            a = st.get(name)
            if kind == MEM_HOST:
                a = np.ascontiguousarray(np.zeros((0, cols)) if a is None else a, dt).reshape(-1, cols)
                keep.append(a)
                setattr(e, name, a.ctypes.data if len(a) else None)
                setattr(e, count, len(a))
            else:
                ptr, n = (None, 0) if a is None else a
                setattr(e, name, ptr)
                setattr(e, count, int(n))
        T = np.asarray(st["T"], np.float64).reshape(4, 4)
        for k, v in enumerate(T.T.ravel()):
            e.T[k] = float(v)
    return arr, keep


def _slot_array(slot_pairs) -> np.ndarray:
    """(n, 2) int32 array of (source slot, target slot) pairs, laid out as qb200_slot_pair[n]."""
    return np.ascontiguousarray(np.asarray(slot_pairs, np.int32).reshape(-1, 2))


def _scan_arrays(scans: Sequence, kind: int):
    """(void* * n) scan pointers and (int32 * n) point counts of `scans`: (n,4) float32 arrays (MEM_HOST) or (device_ptr, n) tuples
    (MEM_DEVICE); and the contiguous scans they point to."""
    keep = [_f32(sc, 4) for sc in scans] if kind == MEM_HOST else []
    ptrs = [a.ctypes.data for a in keep] if kind == MEM_HOST else [sc[0] for sc in scans]
    sizes = [len(a) for a in keep] if kind == MEM_HOST else [int(sc[1]) for sc in scans]
    n = max(len(scans), 1)
    return (C.c_void_p * n)(*ptrs), (C.c_int32 * n)(*sizes), keep


def load_library(build: bool = True) -> C.CDLL:
    """Load libquatro_b200.so (building it with nvcc if stale).  Raises if it cannot be built/loaded."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = _build.build_cuda() if build else _build.CUDA_LIB
    lib = C.CDLL(str(path))
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError = header/library mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args
    _LIB = lib
    return lib


def default_params() -> Params:
    """config/params.yaml defaults.  Pure-Python mirror of qb200_default_params (so CPU-only tests can
    build a Params without loading the CUDA library); test_capi checks the two agree."""
    p = Params()
    p.voxel_size, p.normal_radius, p.fpfh_radius, p.grid_cell = 0.3, 0.5, 0.75, 0.0
    p.tuple_scale, p.use_crosscheck, p.use_tuple_test, p.tuple_trials_per_corr = 0.95, 1, 1, 100
    p.skip_flagged, p.seed = 1, 0x5EED
    p.noise_bound, p.cbar2, p.rot_noise_bound, p.cote_noise_bound = 0.3, 1.0, 0.0, 0.3
    p.rotation_gnc_factor, p.rotation_cost_threshold, p.kcore_heuristic_threshold = 1.4, 0.00011, 0.5
    p.rotation_max_iterations, p.inlier_selection_mode, p.cote_mode = 50, PMC_HEU, COTE_MEDIAN
    p.using_rot_inliers_when_estimating_cote, p.use_pre_estimated_RyRx = 0, 0
    for i in range(9):
        p.RyRx[i] = 1.0 if i in (0, 4, 8) else 0.0
    return p


def comm_init_all(handles: Sequence["Handle"]):
    """(A) one process, several devices: ncclCommInitAll over the handles' devices."""
    arr = (C.c_void_p * len(handles))(*[h.h for h in handles])
    st = load_library().qb200_comm_init_all(arr, len(handles))
    if st != 0:
        raise QuatroB200Error(st, "qb200_comm_init_all")


def register_batch_sharded(handles: Sequence["Handle"], pairs: Sequence, params: "Params", kind: int = 0) -> np.ndarray:
    """pairs: (src, tgt) numpy arrays (MEM_HOST) or (src_ptr, n_src, tgt_ptr, n_tgt) device tuples whose pair g lives on the device
    of handles[g % len(handles)].  Returns the records in the order of `pairs`."""
    n = len(pairs)
    arr, keep = _pair_array(pairs, kind)
    out = np.zeros(n, RESULT_DTYPE)
    hs = (C.c_void_p * len(handles))(*[h.h for h in handles])
    st = load_library().qb200_register_batch_sharded(hs, len(handles), arr, n, C.byref(params), kind, _ptr(out))
    if st != 0:
        raise QuatroB200Error(st, "qb200_register_batch_sharded " + handles[0].last_error())
    return out


def default_patchwork_params() -> PatchworkParams:
    p = PatchworkParams()
    load_library().qb200_default_patchwork_params(C.byref(p))
    return p


def default_segment_params() -> SegmentParams:
    p = SegmentParams()
    load_library().qb200_default_segment_params(C.byref(p))
    return p


# The reference's lidar models, as ImageProjection's constructor sets them (include/imageProjection.hpp:85-124): n_scan, horizon_scan,
# ang_res_x, ang_res_y, ang_bottom (computed in double like the reference, stored as float)
LIDAR_MODELS = {
    "Velodyne-64-HDE": (64, 1800, 360.0 / 1800, 26.9 / 63, 25.0),
    "VLP-16": (16, 1800, 0.2, 2.0, 15.0 + 0.1),
    "HDL-32E": (32, 1800, 360.0 / 1800, 41.33 / 31, 30.67),
    "Ouster-OS1-16": (16, 1024, 360.0 / 1024, 33.2 / 15, 16.6 + 0.1),
    "Ouster-OS1-64": (64, 1024, 360.0 / 1024, 33.2 / 63, 16.6 + 0.1),
}


def lidar_segment_params(model: str) -> SegmentParams:
    """The default segment parameters with the image of one of LIDAR_MODELS."""
    p = default_segment_params()
    p.n_scan, p.horizon_scan, p.ang_res_x, p.ang_res_y, p.ang_bottom = LIDAR_MODELS[model]
    return p


def default_config() -> Config:
    c = Config()
    c.device, c.max_batch_slots, c.max_raw_points, c.max_voxel_points, c.max_corr = 0, 64, 131072, 16384, 4096
    return c


class Handle:
    """RAII wrapper of qb200_handle.  Raises QuatroB200Error(ERR_NO_DEVICE) when no GPU is usable."""

    def __init__(self, config: Optional[Config] = None, **kw):
        self.lib = load_library()
        cfg = config or default_config()
        for k, v in kw.items():
            setattr(cfg, k, v)
        self.cfg = cfg
        h = C.c_void_p()
        st = self.lib.qb200_create(C.byref(cfg), C.byref(h))
        if st != 0:
            raise QuatroB200Error(st, "qb200_create")
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.lib.qb200_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _check(self, st: int, where: str):
        if st < 0:
            msg = self.lib.qb200_last_error(self.h)
            raise QuatroB200Error(st, where, (msg or b"").decode())
        return st

    def set_stream(self, stream_ptr: int):
        self._check(self.lib.qb200_set_stream(self.h, C.c_void_p(stream_ptr)), "qb200_set_stream")

    def launch_count(self) -> int:
        return int(self.lib.qb200_launch_count(self.h))

    # ---- stages -------------------------------------------------------------------------------
    def voxelize(self, pts4, leaf: float, skip_flagged: int = 1, cap: Optional[int] = None):
        pts4 = _f32(pts4, 4)
        cap = cap or max(1, len(pts4))
        out = np.zeros((cap, 4), np.float32)
        n = C.c_int32(0)
        st = self.lib.qb200_voxelize(self.h, _ptr(pts4), len(pts4), leaf, skip_flagged, _ptr(out), cap, C.byref(n))
        if st != -5:  # ERR_VOXEL_OVERFLOW = PCL's "leaf too small" pass-through: output is the unfiltered input
            self._check(st, "qb200_voxelize")
        return out[: min(n.value, cap)].copy(), st

    def compute_fpfh(self, pts4, normal_radius: float, fpfh_radius: float, grid_cell: float):
        pts4 = _f32(pts4, 4)
        n = len(pts4)
        normals = np.zeros((n, 4), np.float32)
        desc = np.zeros((n, 33), np.float32)
        self._check(self.lib.qb200_compute_fpfh(self.h, _ptr(pts4), n, normal_radius, fpfh_radius, grid_cell, _ptr(normals), _ptr(desc)),
                    "qb200_compute_fpfh")
        return normals, desc

    def match(self, src4, sdesc, tgt4, tdesc, params: Params, cap: Optional[int] = None):
        src4, tgt4, sdesc, tdesc = _f32(src4, 4), _f32(tgt4, 4), _f32(sdesc, 33), _f32(tdesc, 33)
        cap = cap or max(1, min(len(src4), len(tgt4)))
        corr = np.zeros((cap, 2), np.int32)
        n, nm = C.c_int32(0), C.c_int32(0)
        st = self._check(self.lib.qb200_match(self.h, _ptr(src4), len(src4), _ptr(sdesc), _ptr(tgt4), len(tgt4), _ptr(tdesc),
                                              C.byref(params), _ptr(corr), cap, C.byref(n), C.byref(nm)), "qb200_match")
        return corr[: min(n.value, cap)].copy(), nm.value, st

    def build_graph(self, a4, b4, noise_bound: float, cbar2: float, words_per_row: Optional[int] = None):
        a4, b4 = _f32(a4, 4), _f32(b4, 4)
        L = len(a4)
        wpr = words_per_row or (L + 31) // 32
        adj = np.zeros((L, wpr), np.uint32)
        deg = np.zeros(L, np.int32)
        ne = C.c_int64(0)
        self._check(self.lib.qb200_build_graph(self.h, _ptr(a4), _ptr(b4), L, noise_bound, cbar2, _ptr(adj), wpr, _ptr(deg), C.byref(ne)),
                    "qb200_build_graph")
        return adj, deg, ne.value

    def patchwork(self, pts, pp: "PatchworkParams"):
        """qb200_patchwork: (ground (g,4), nonground (m,4), status)."""
        pts = _f32(pts, 4)
        n = len(pts)
        g, ng = np.zeros((max(n, 1), 4), np.float32), np.zeros((max(n, 1), 4), np.float32)
        a, b = C.c_int32(0), C.c_int32(0)
        st = self._check(self.lib.qb200_patchwork(self.h, _ptr(pts), n, C.byref(pp), _ptr(g), C.byref(a), _ptr(ng), C.byref(b)), "qb200_patchwork")
        return g[: a.value].copy(), ng[: b.value].copy(), st

    def segment_cloud(self, pts, sp: "SegmentParams"):
        """qb200_segment_cloud: (valid segments (v,4), outliers (o,4))."""
        pts = _f32(pts, 4)
        npix = sp.n_scan * sp.horizon_scan
        v, o = np.zeros((npix, 4), np.float32), np.zeros((npix, 4), np.float32)
        a, b = C.c_int32(0), C.c_int32(0)
        self._check(self.lib.qb200_segment_cloud(self.h, _ptr(pts), len(pts), C.byref(sp), _ptr(v), C.byref(a), _ptr(o), C.byref(b)),
                    "qb200_segment_cloud")
        return v[: a.value].copy(), o[: b.value].copy()

    def preprocess_batch(self, scans: Sequence, pp: "PatchworkParams", sp: Optional["SegmentParams"] = None, cap: Optional[int] = None,
                         kind: int = MEM_HOST, dest: int = MEM_HOST, arrays: Optional[dict] = None):
        """qb200_preprocess_batch.  scans: (n,4) float32 arrays (MEM_HOST) or (device_ptr, n) tuples (MEM_DEVICE).  cap: points per
        scan and array (default: room for the largest output).  arrays: the caller's own output arrays by name (PREPROCESS_ARRAYS),
        numpy (dest MEM_HOST) or CUDA tensors (dest MEM_DEVICE) of shape (n_scans, cap, 4); a name left out is passed as NULL.
        Returns (per scan a tuple (ground, nonground, valid, outlier) trimmed to min(count, cap), None for a NULL array;
        counts (n,4) int32; status (n,) int32)."""
        return self._preprocess("qb200_preprocess_batch", scans, C.byref(pp), None if sp is None else C.byref(sp),
                                [] if sp is None else [sp], cap, kind, dest, arrays)

    def preprocess_batch_each(self, scans: Sequence, pps: Sequence["PatchworkParams"], sps: Optional[Sequence["SegmentParams"]] = None,
                              cap: Optional[int] = None, kind: int = MEM_HOST, dest: int = MEM_HOST, arrays: Optional[dict] = None):
        """qb200_preprocess_batch_each: preprocess_batch with pps[i] (and sps[i]) for scan i; sps None: ground removal only.  Returns
        what preprocess_batch returns."""
        n = len(scans)
        pa = (PatchworkParams * n)(*pps) if n else None
        sa = None if sps is None else ((SegmentParams * n)(*sps) if n else None)
        return self._preprocess("qb200_preprocess_batch_each", scans, pa, sa, [] if sps is None else list(sps), cap, kind, dest, arrays)

    def _preprocess(self, fn: str, scans, pp_arg, sp_arg, sps, cap, kind, dest, arrays):
        """The two batch pre-processing calls: sps = the segment parameters in use (the default cap makes room for every image)."""
        n = len(scans)
        ptrs, cnts, keep = _scan_arrays(scans, kind)
        if cap is None:
            cap = max([1, *cnts[:n]] + [s.n_scan * s.horizon_scan for s in sps])
        if arrays is None:
            names = PREPROCESS_ARRAYS if sp_arg is not None else PREPROCESS_ARRAYS[:2]
            if dest == MEM_HOST:
                arrays = {k: np.zeros((max(n, 1), cap, 4), np.float32) for k in names}
            else:
                import torch
                arrays = {k: torch.zeros((max(n, 1), cap, 4), dtype=torch.float32, device=f"cuda:{self.cfg.device}") for k in names}
        counts = np.zeros((max(n, 1), 4), np.int32)
        status = np.zeros(max(n, 1), np.int32)
        out = PreprocessOut(cap, dest)
        for k, a in arrays.items():
            setattr(out, k, a.ctypes.data if dest == MEM_HOST else a.data_ptr())
        out.counts, out.status = counts.ctypes.data, status.ctypes.data
        self._check(getattr(self.lib, fn)(self.h, ptrs, cnts, n, kind, pp_arg, sp_arg, C.byref(out)), fn)
        per_scan = []
        for i in range(n):
            row = []
            for j, k in enumerate(PREPROCESS_ARRAYS):
                a = arrays.get(k)
                m = min(int(counts[i, j]), cap)
                row.append(None if a is None else (a[i, :m].copy() if dest == MEM_HOST else a[i, :m].cpu().numpy()))
            per_scan.append(tuple(row))
        return per_scan, counts[:n], status[:n]

    def max_clique(self, adj, mode: int = PMC_HEU, kcore_thr: float = 0.5):
        adj = np.ascontiguousarray(adj, np.uint32)
        L, wpr = adj.shape
        clique = np.zeros(max(L, 1), np.int32)
        kcore = np.zeros(max(L, 1), np.int32)
        order = np.zeros(max(L, 1), np.int32)
        n, mc = C.c_int32(0), C.c_int32(0)
        self._check(self.lib.qb200_max_clique(self.h, _ptr(adj), L, wpr, mode, kcore_thr, _ptr(clique), C.byref(n), _ptr(kcore),
                                              _ptr(order), C.byref(mc)), "qb200_max_clique")
        return clique[: n.value].copy(), kcore[:L].copy(), order[:L].copy(), mc.value

    def max_clique_ex(self, adj, mode: int = PMC_EXACT, kcore_thr: float = 0.5, node_limit: int = 0):
        """qb200_max_clique_ex: clique, kcore, order, max_core, flags (FLAG_CLIQUE_TRUNCATED when the node limit stopped the search)."""
        adj = np.ascontiguousarray(adj, np.uint32)
        L, wpr = adj.shape
        clique, kcore, order = (np.zeros(max(L, 1), np.int32) for _ in range(3))
        n, mc, fl = C.c_int32(0), C.c_int32(0), C.c_int32(0)
        self._check(self.lib.qb200_max_clique_ex(self.h, _ptr(adj), L, wpr, mode, kcore_thr, node_limit, _ptr(clique), C.byref(n),
                                                 _ptr(kcore), _ptr(order), C.byref(mc), C.byref(fl)), "qb200_max_clique_ex")
        return clique[: n.value].copy(), kcore[:L].copy(), order[:L].copy(), mc.value, fl.value

    def solve_pose(self, a4, b4, clique, params: Params):
        a4, b4 = _f32(a4, 4), _f32(b4, 4)
        clique = np.ascontiguousarray(clique, np.int32)
        res = Result()
        rm = np.zeros(max(len(clique), 1), np.uint8)
        tm = np.zeros(max(len(clique), 1), np.uint8)
        st = self._check(self.lib.qb200_solve_pose(self.h, _ptr(a4), _ptr(b4), len(a4), _ptr(clique), len(clique), C.byref(params),
                                                   C.byref(res), _ptr(rm), _ptr(tm)), "qb200_solve_pose")
        return res, rm[: len(clique)], tm[: len(clique)], st

    def solve_correspondences(self, a4, b4, params: Params):
        a4, b4 = _f32(a4, 4), _f32(b4, 4)
        res = Result()
        st = self._check(self.lib.qb200_solve_correspondences(self.h, _ptr(a4), _ptr(b4), len(a4), C.byref(params), C.byref(res)),
                         "qb200_solve_correspondences")
        return res, st

    def match_and_pack(self, src4, tgt4, params: Params, cap: Optional[int] = None):
        src4, tgt4 = _f32(src4, 4), _f32(tgt4, 4)
        cap = cap or max(1, min(len(src4), len(tgt4)))
        corr = np.zeros((cap, 2), np.int32)
        sm = np.zeros((cap, 4), np.float32)
        tm = np.zeros((cap, 4), np.float32)
        n = C.c_int32(0)
        st = self._check(self.lib.qb200_match_and_pack(self.h, _ptr(src4), len(src4), _ptr(tgt4), len(tgt4), C.byref(params), _ptr(corr),
                                                       _ptr(sm), _ptr(tm), cap, C.byref(n)), "qb200_match_and_pack")
        m = min(n.value, cap)
        return corr[:m].copy(), sm[:m].copy(), tm[:m].copy(), st

    def register_pair(self, src4, tgt4, params: Params):
        src4, tgt4 = _f32(src4, 4), _f32(tgt4, 4)
        res = Result()
        st = self._check(self.lib.qb200_register_pair(self.h, _ptr(src4), len(src4), _ptr(tgt4), len(tgt4), C.byref(params), C.byref(res)),
                         "qb200_register_pair")
        return res, st

    pair_array = staticmethod(_pair_array)
    _set_array = staticmethod(_set_array)
    feature_array = staticmethod(_feature_array)

    def register_batch(self, pairs: Sequence, params: Params, kind: int = MEM_HOST) -> np.ndarray:
        """pairs: sequence of (src, tgt).  MEM_HOST: numpy (n,4) float32 arrays; MEM_DEVICE:
        (src_ptr, n_src, tgt_ptr, n_tgt) tuples of raw device addresses.  Returns a RESULT_DTYPE array."""
        arr, keep = self.pair_array(pairs, kind)
        out = np.zeros(len(pairs), RESULT_DTYPE)
        self._check(self.lib.qb200_register_batch(self.h, arr, len(pairs), C.byref(params), kind, _ptr(out)), "qb200_register_batch")
        return out

    def solve_batch(self, sets: Sequence, params: Params, kind: int = MEM_HOST) -> np.ndarray:
        """sets: sequence of (a4, b4) matched point arrays (MEM_HOST: numpy (L,4) float32; MEM_DEVICE: (a_ptr, b_ptr, L)).
        Graph -> clique -> pose for every set; returns a RESULT_DTYPE array."""
        arr, keep = self._set_array(sets, kind)
        out = np.zeros(len(sets), RESULT_DTYPE)
        self._check(self.lib.qb200_solve_batch(self.h, arr, len(sets), C.byref(params), kind, _ptr(out)), "qb200_solve_batch")
        return out

    # ---- per-pair lists of the batch entry points (qb200_pair_lists) ----
    # Each returns (records, lists): lists[i] is a dict of pair i's lists cut to their counts (ListBuffers.trimmed).  dest picks
    # where the call writes them (MEM_HOST: numpy, MEM_DEVICE: CUDA tensors of the handle's device); `buffers` hands in
    # caller-made ListBuffers instead (cap_per_pair / dest are then theirs).
    def _lists_for(self, n: int, cap_per_pair: Optional[int], dest: int, buffers: Optional[ListBuffers], names) -> ListBuffers:
        return buffers or ListBuffers(n, cap_per_pair or self.cfg.max_corr, dest, names, self.cfg.device)

    def _batch_lists(self, name: str, n: int, args: tuple, buffers: Optional[ListBuffers]):
        """name(h, *args, records, lists) for n pairs -> (records, lists as ListBuffers.trimmed, or None without buffers)."""
        out = np.zeros(n, RESULT_DTYPE)
        self._check(getattr(self.lib, name)(self.h, *args, _ptr(out), self._lists_arg(buffers)), name)
        return out, (None if buffers is None else buffers.trimmed(out))

    def register_batch_lists(self, pairs: Sequence, params: Params, kind: int = MEM_HOST, cap_per_pair: Optional[int] = None,
                             dest: int = MEM_HOST, buffers: Optional[ListBuffers] = None):
        """qb200_register_batch_ex: register_batch + every pair's correspondences, matched points, clique, final inliers and masks."""
        arr, keep = self.pair_array(pairs, kind)
        lb = self._lists_for(len(pairs), cap_per_pair, dest, buffers, tuple(LIST_LAYOUT))
        return self._batch_lists("qb200_register_batch_ex", len(pairs), (arr, len(pairs), C.byref(params), kind), lb)

    def register_batch_enqueue_lists_raw(self, pair_array, n: int, params: Params, kind: int, out: np.ndarray, buffers: ListBuffers):
        """qb200_register_batch_enqueue_ex: pair_array, its scans, `out` and the buffers must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_register_batch_enqueue_ex(self.h, pair_array, n, C.byref(params), kind, _ptr(out),
                                                                    self._lists_arg(buffers)), "qb200_register_batch_enqueue_ex")

    def register_cached_lists(self, slot_pairs, params: Params, cap_per_pair: Optional[int] = None, dest: int = MEM_HOST,
                              buffers: Optional[ListBuffers] = None):
        """qb200_register_cached_ex: corr indexes the voxel points cache_read returns."""
        sp = _slot_array(slot_pairs)
        lb = self._lists_for(len(sp), cap_per_pair, dest, buffers, tuple(LIST_LAYOUT))
        return self._batch_lists("qb200_register_cached_ex", len(sp), (_ptr(sp), len(sp), C.byref(params)), lb)

    def solve_batch_lists(self, sets: Sequence, params: Params, kind: int = MEM_HOST, cap_per_pair: Optional[int] = None,
                          dest: int = MEM_HOST, buffers: Optional[ListBuffers] = None):
        """qb200_solve_batch_ex: solve_batch + every set's clique, final inliers and masks (the caller has the correspondences)."""
        arr, keep = self._set_array(sets, kind)
        lb = self._lists_for(len(sets), cap_per_pair, dest, buffers, SET_LISTS)
        return self._batch_lists("qb200_solve_batch_ex", len(sets), (arr, len(sets), C.byref(params), kind), lb)

    # ---- one Params per pair (the _each entry points) ----
    # params: one Params per pair (or set), in the order of the inputs.  buffers: the ListBuffers to fill, or None for records only.
    # Each returns (records, lists): lists as ListBuffers.trimmed, None without buffers.
    @staticmethod
    def params_array(params: Sequence[Params]):
        """(Params * n) array of `params` (at least one element, so that n = 0 still passes a valid pointer)."""
        return (Params * max(len(params), 1))(*params)

    @staticmethod
    def _lists_arg(buffers: Optional[ListBuffers]):
        return None if buffers is None else C.byref(buffers.descriptor())

    def register_batch_each(self, pairs: Sequence, params: Sequence[Params], kind: int = MEM_HOST, buffers: Optional[ListBuffers] = None):
        """qb200_register_batch_each: pair i is registered with params[i] (front-end fields equal in every entry)."""
        assert len(params) == len(pairs)
        arr, keep = self.pair_array(pairs, kind)
        return self._batch_lists("qb200_register_batch_each", len(pairs), (arr, len(pairs), self.params_array(params), kind), buffers)

    def register_batch_enqueue_each_raw(self, pair_array, n: int, params_array, kind: int, out: np.ndarray,
                                        buffers: Optional[ListBuffers] = None):
        """qb200_register_batch_enqueue_each: params_array (params_array()) is copied by the call; pair_array, its scans, `out` and the
        buffers must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_register_batch_enqueue_each(self.h, pair_array, n, params_array, kind, _ptr(out),
                                                                      self._lists_arg(buffers)), "qb200_register_batch_enqueue_each")

    def register_cached_each(self, slot_pairs, params: Sequence[Params], buffers: Optional[ListBuffers] = None):
        """qb200_register_cached_each: slot pair i is registered with params[i] (front-end fields: the ones the slots were cached with)."""
        sp = _slot_array(slot_pairs)
        assert len(params) == len(sp)
        return self._batch_lists("qb200_register_cached_each", len(sp), (_ptr(sp), len(sp), self.params_array(params)), buffers)

    def solve_batch_each(self, sets: Sequence, params: Sequence[Params], kind: int = MEM_HOST, buffers: Optional[ListBuffers] = None):
        """qb200_solve_batch_each: set i is solved with params[i] (front-end fields ignored)."""
        assert len(params) == len(sets)
        arr, keep = self._set_array(sets, kind)
        return self._batch_lists("qb200_solve_batch_each", len(sets), (arr, len(sets), self.params_array(params), kind), buffers)

    # ---- one Params per pair, front end included (the _mixed entry points) ----
    def register_batch_mixed(self, pairs: Sequence, params: Sequence[Params], kind: int = MEM_HOST, buffers: Optional[ListBuffers] = None):
        """qb200_register_batch_mixed: pair i is voxelized, described, matched and solved with params[i] (every field may differ)."""
        assert len(params) == len(pairs)
        arr, keep = self.pair_array(pairs, kind)
        return self._batch_lists("qb200_register_batch_mixed", len(pairs), (arr, len(pairs), self.params_array(params), kind), buffers)

    def register_batch_enqueue_mixed_raw(self, pair_array, n: int, params_array, kind: int, out: np.ndarray,
                                         buffers: Optional[ListBuffers] = None):
        """qb200_register_batch_enqueue_mixed: params_array (params_array()) is copied by the call; pair_array, its scans, `out` and the
        buffers must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_register_batch_enqueue_mixed(self.h, pair_array, n, params_array, kind, _ptr(out),
                                                                       self._lists_arg(buffers)), "qb200_register_batch_enqueue_mixed")

    def register_cached_mixed(self, slot_pairs, params: Sequence[Params], buffers: Optional[ListBuffers] = None):
        """qb200_register_cached_mixed: slot pair i is registered with params[i], whose front-end fields must be the ones both of its
        slots were cached with."""
        sp = _slot_array(slot_pairs)
        assert len(params) == len(sp)
        return self._batch_lists("qb200_register_cached_mixed", len(sp), (_ptr(sp), len(sp), self.params_array(params)), buffers)

    def register_cached_enqueue_mixed_raw(self, slot_array, n: int, params_array, out: np.ndarray, buffers: Optional[ListBuffers] = None):
        """qb200_register_cached_enqueue_mixed: params_array (params_array()) is copied by the call; slot_array (_slot_array()), `out`
        and the buffers must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_register_cached_enqueue_mixed(self.h, _ptr(slot_array), n, params_array, _ptr(out),
                                                                        self._lists_arg(buffers)), "qb200_register_cached_enqueue_mixed")

    def solve_batch_enqueue_each_raw(self, set_array, n: int, params_array, kind: int, out: np.ndarray,
                                     buffers: Optional[ListBuffers] = None):
        """qb200_solve_batch_enqueue_each: params_array (params_array()) is copied by the call; set_array (_set_array()), its points
        (host kind), `out` and the buffers must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_solve_batch_enqueue_each(self.h, set_array, n, params_array, kind, _ptr(out),
                                                                   self._lists_arg(buffers)), "qb200_solve_batch_enqueue_each")

    # ---- caller keypoints and FPFH-33 descriptors (the matcher boundary) ----
    def register_features_each(self, pairs: Sequence, params: Sequence[Params], kind: int = MEM_HOST, buffers: Optional[ListBuffers] = None):
        """qb200_register_features_each: pair i's keypoints and descriptors (feature_array()) are matched and solved with params[i];
        corr indexes the caller's keypoints."""
        assert len(params) == len(pairs)
        arr, keep = self.feature_array(pairs, kind)
        return self._batch_lists("qb200_register_features_each", len(pairs), (arr, len(pairs), self.params_array(params), kind), buffers)

    def register_features_enqueue_each_raw(self, feature_array, n: int, params_array, kind: int, out: np.ndarray,
                                           buffers: Optional[ListBuffers] = None):
        """qb200_register_features_enqueue_each: params_array (params_array()) is copied by the call; feature_array (feature_array()),
        its host arrays, `out` and the buffers must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_register_features_enqueue_each(self.h, feature_array, n, params_array, kind, _ptr(out),
                                                                         self._lists_arg(buffers)), "qb200_register_features_enqueue_each")

    # ---- raw, cached or caller-feature pairs -> correspondences and matched points, not solved (the qb200_match_* calls) ----
    # buffers: a ListBuffers of MATCH_LISTS only, or None for records only.  Each returns (records, lists) like the register forms.
    @staticmethod
    def _match_lists(buffers: Optional[ListBuffers]) -> Optional[ListBuffers]:
        assert buffers is None or set(buffers.arrays) <= set(MATCH_LISTS), "a match call returns corr and the matched points only"
        return buffers

    def match_batch_mixed(self, pairs: Sequence, params: Sequence[Params], kind: int = MEM_HOST, buffers: Optional[ListBuffers] = None):
        """qb200_match_batch_mixed: pair i is voxelized, described and matched with params[i] (solver fields ignored)."""
        assert len(params) == len(pairs)
        arr, keep = self.pair_array(pairs, kind)
        return self._batch_lists("qb200_match_batch_mixed", len(pairs), (arr, len(pairs), self.params_array(params), kind),
                                 self._match_lists(buffers))

    def match_batch_enqueue_mixed_raw(self, pair_array, n: int, params_array, kind: int, out: np.ndarray,
                                      buffers: Optional[ListBuffers] = None):
        """qb200_match_batch_enqueue_mixed: params_array (params_array()) is copied by the call; pair_array, its scans, `out` and the
        buffers must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_match_batch_enqueue_mixed(self.h, pair_array, n, params_array, kind, _ptr(out),
                                                                    self._lists_arg(self._match_lists(buffers))),
                           "qb200_match_batch_enqueue_mixed")

    def match_cached_mixed(self, slot_pairs, params: Sequence[Params], buffers: Optional[ListBuffers] = None):
        """qb200_match_cached_mixed: slot pair i is matched with params[i], whose front-end fields must be the ones both of its slots
        were cached with."""
        sp = _slot_array(slot_pairs)
        assert len(params) == len(sp)
        return self._batch_lists("qb200_match_cached_mixed", len(sp), (_ptr(sp), len(sp), self.params_array(params)), self._match_lists(buffers))

    def match_cached_enqueue_mixed_raw(self, slot_array, n: int, params_array, out: np.ndarray, buffers: Optional[ListBuffers] = None):
        """qb200_match_cached_enqueue_mixed: params_array (params_array()) is copied by the call; slot_array (_slot_array()), `out` and
        the buffers must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_match_cached_enqueue_mixed(self.h, _ptr(slot_array), n, params_array, _ptr(out),
                                                                     self._lists_arg(self._match_lists(buffers))),
                           "qb200_match_cached_enqueue_mixed")

    def match_features_each(self, pairs: Sequence, params: Sequence[Params], kind: int = MEM_HOST, buffers: Optional[ListBuffers] = None):
        """qb200_match_features_each: pair i's keypoints and descriptors (feature_array()) are matched with params[i]; corr indexes the
        caller's keypoints."""
        assert len(params) == len(pairs)
        arr, keep = self.feature_array(pairs, kind)
        return self._batch_lists("qb200_match_features_each", len(pairs), (arr, len(pairs), self.params_array(params), kind),
                                 self._match_lists(buffers))

    def match_features_enqueue_each_raw(self, feature_array, n: int, params_array, kind: int, out: np.ndarray,
                                        buffers: Optional[ListBuffers] = None):
        """qb200_match_features_enqueue_each: params_array (params_array()) is copied by the call; feature_array (feature_array()), its
        host arrays, `out` and the buffers must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_match_features_enqueue_each(self.h, feature_array, n, params_array, kind, _ptr(out),
                                                                      self._lists_arg(self._match_lists(buffers))),
                           "qb200_match_features_enqueue_each")

    # ---- caller keypoints and descriptors of any length (qb200_match_descriptors_each, qb200_register_descriptors_each) ----
    descriptor_array = staticmethod(_descriptor_array)

    def match_descriptors_each(self, pairs: Sequence, params: Sequence[Params], kind: int = MEM_HOST,
                               buffers: Optional[ListBuffers] = None):
        """qb200_match_descriptors_each: pair i's keypoints and descriptors (descriptor_array()) are matched with params[i]; corr
        indexes the caller's keypoints."""
        assert len(params) == len(pairs)
        arr, keep = self.descriptor_array(pairs, kind)
        return self._batch_lists("qb200_match_descriptors_each", len(pairs), (arr, len(pairs), self.params_array(params), kind),
                                 self._match_lists(buffers))

    def match_descriptors_enqueue_each_raw(self, descriptor_array, n: int, params_array, kind: int, out: np.ndarray,
                                           buffers: Optional[ListBuffers] = None):
        """qb200_match_descriptors_enqueue_each: params_array (params_array()) is copied by the call; descriptor_array
        (descriptor_array()), its host arrays, `out` and the buffers must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_match_descriptors_enqueue_each(self.h, descriptor_array, n, params_array, kind, _ptr(out),
                                                                         self._lists_arg(self._match_lists(buffers))),
                           "qb200_match_descriptors_enqueue_each")

    def register_descriptors_each(self, pairs: Sequence, params: Sequence[Params], kind: int = MEM_HOST,
                                  buffers: Optional[ListBuffers] = None):
        """qb200_register_descriptors_each: pair i's keypoints and descriptors (descriptor_array()) are matched and solved with
        params[i]; corr indexes the caller's keypoints."""
        assert len(params) == len(pairs)
        arr, keep = self.descriptor_array(pairs, kind)
        return self._batch_lists("qb200_register_descriptors_each", len(pairs), (arr, len(pairs), self.params_array(params), kind),
                                 buffers)

    def register_descriptors_enqueue_each_raw(self, descriptor_array, n: int, params_array, kind: int, out: np.ndarray,
                                              buffers: Optional[ListBuffers] = None):
        """qb200_register_descriptors_enqueue_each: params_array (params_array()) is copied by the call; descriptor_array
        (descriptor_array()), its host arrays, `out` and the buffers must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_register_descriptors_enqueue_each(self.h, descriptor_array, n, params_array, kind,
                                                                            _ptr(out), self._lists_arg(buffers)),
                           "qb200_register_descriptors_enqueue_each")

    # ---- caller graphs -> maximum cliques (qb200_max_clique_batch_each) ----
    graph_array = staticmethod(_graph_array)

    @staticmethod
    def _graph_lists(buffers: Optional[ListBuffers]) -> Optional[ListBuffers]:
        assert buffers is None or set(buffers.arrays) <= set(GRAPH_LISTS), "a graph batch returns the clique only"
        return buffers

    def max_clique_batch_each(self, graphs: Sequence, params: Sequence[Params], kind: int = MEM_HOST, buffers: Optional[ListBuffers] = None):
        """qb200_max_clique_batch_each: graph i (see graph_array()) is solved with the inlier_selection_mode, kcore_heuristic_threshold
        and max_clique_node_limit of params[i]; buffers: a ListBuffers of GRAPH_LISTS, or None for records only."""
        assert len(params) == len(graphs)
        arr, keep = self.graph_array(graphs)
        return self._batch_lists("qb200_max_clique_batch_each", len(graphs), (arr, len(graphs), self.params_array(params), kind),
                                 self._graph_lists(buffers))

    def max_clique_batch_enqueue_each_raw(self, graph_array, n: int, params_array, kind: int, out: np.ndarray,
                                          buffers: Optional[ListBuffers] = None):
        """qb200_max_clique_batch_enqueue_each: graph_array (graph_array()) and params_array (params_array()) are read by the call; the
        host arrays behind graph_array, `out` and the buffers must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_max_clique_batch_enqueue_each(self.h, graph_array, n, params_array, kind, _ptr(out),
                                                                        self._lists_arg(self._graph_lists(buffers))),
                           "qb200_max_clique_batch_enqueue_each")

    # ---- correspondence sets -> TIM graphs (qb200_build_graph_batch_each) ----
    def build_graph_batch_each(self, sets: Sequence, params: Sequence[Params], kind: int = MEM_HOST,
                               buffers: Optional[GraphBuffers] = None) -> np.ndarray:
        """qb200_build_graph_batch_each: set i (as solve_batch takes it) is built with the noise_bound and cbar2 of params[i]; its
        adjacency rows, degrees and edge list go to `buffers` (None: records only).  Returns the records."""
        assert len(params) == len(sets)
        arr, keep = self._set_array(sets, kind)
        out = np.zeros(len(sets), RESULT_DTYPE)
        d = GraphOut() if buffers is None else buffers.descriptor()
        self._check(self.lib.qb200_build_graph_batch_each(self.h, arr, len(sets), self.params_array(params), kind, _ptr(out), C.byref(d)),
                    "qb200_build_graph_batch_each")
        return out

    def build_graph_batch_enqueue_each_raw(self, set_array, n: int, params_array, kind: int, out: np.ndarray, buffers: GraphBuffers):
        """qb200_build_graph_batch_enqueue_each: params_array (params_array()) and the descriptor are copied by the call; set_array
        (_set_array()), its points (host kind), `out` and the buffers must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_build_graph_batch_enqueue_each(self.h, set_array, n, params_array, kind, _ptr(out),
                                                                         C.byref(buffers.descriptor())),
                           "qb200_build_graph_batch_enqueue_each")

    # ---- registered pairs -> aligned clouds and good matches (qb200_align_batch_each) ----
    align_array = staticmethod(_align_array)

    def align_buffers(self, n: int, cap_points: int, cap_corr: int, dest: int = MEM_HOST, arrays=tuple(ALIGN_ARRAYS)) -> dict:
        """Zeroed output arrays of an align call by name: numpy (dest MEM_HOST) or CUDA tensors of the handle's device (MEM_DEVICE), of
        shape (n, cap_points, 4) for aligned4 and (n, cap_corr, ...) for the others."""
        def shape(k):
            return (max(n, 1), cap_points if k == "aligned4" else cap_corr, *ALIGN_ARRAYS[k][1])
        if dest == MEM_HOST:
            return {k: np.zeros(shape(k), ALIGN_ARRAYS[k][0]) for k in arrays}
        import torch
        dt = {np.float32: torch.float32, np.int32: torch.int32}
        return {k: torch.zeros(shape(k), dtype=dt[ALIGN_ARRAYS[k][0]], device=f"cuda:{self.cfg.device}") for k in arrays}

    @staticmethod
    def align_out(cap_points: int, cap_corr: int, dest: int, arrays: dict, counts: Optional[np.ndarray],
                  status: Optional[np.ndarray]) -> AlignOut:
        """The qb200_align_out of `arrays` (align_buffers()) and the host int32 arrays counts ((n, 3)) / status; a name left out, or a
        None, is NULL."""
        out = AlignOut(cap_points, cap_corr, dest)
        for k, a in arrays.items():
            setattr(out, k, a.ctypes.data if dest == MEM_HOST else a.data_ptr())
        out.counts = None if counts is None else counts.ctypes.data
        out.status = None if status is None else status.ctypes.data
        return out

    def align_batch_each(self, sets: Sequence, params: Sequence[Params], kind: int = MEM_HOST, dest: int = MEM_HOST,
                         cap_points: Optional[int] = None, cap_corr: Optional[int] = None, arrays: Optional[dict] = None):
        """qb200_align_batch_each: set i (see align_array()) is aligned with the threshold 3 * params[i].voxel_size.  cap_points /
        cap_corr: entries reserved per set (default max_raw_points / max_corr).  arrays: the caller's own outputs by name
        (ALIGN_ARRAYS), numpy for dest MEM_HOST or CUDA tensors for MEM_DEVICE; a name left out is NULL.  Returns (per set a dict of
        its arrays trimmed to min(count, cap): numpy copies, tensor views on the device; counts (n, 3) int32; status (n,) int32)."""
        n = len(sets)
        assert len(params) == n
        cp = self.cfg.max_raw_points if cap_points is None else cap_points
        cc = self.cfg.max_corr if cap_corr is None else cap_corr
        arrays = self.align_buffers(n, cp, cc, dest) if arrays is None else arrays
        counts, status = np.zeros((max(n, 1), 3), np.int32), np.zeros(max(n, 1), np.int32)
        arr, keep = self.align_array(sets, kind)
        out = self.align_out(cp, cc, dest, arrays, counts, status)
        self._check(self.lib.qb200_align_batch_each(self.h, arr, n, self.params_array(params), kind, C.byref(out)),
                    "qb200_align_batch_each")
        per_set = []
        for i in range(n):
            m = {"aligned4": min(int(counts[i, 0]), cp), "matched4": min(int(counts[i, 1]), cc), "good_ids": min(int(counts[i, 2]), cc),
                 "good4": min(int(counts[i, 2]), cc)}
            per_set.append({k: (a[i, :m[k]].copy() if dest == MEM_HOST else a[i, :m[k]]) for k, a in arrays.items()})
        return per_set, counts[:n], status[:n]

    def align_batch_enqueue_each_raw(self, align_array, n: int, params_array, kind: int, out: AlignOut):
        """qb200_align_batch_enqueue_each: align_array (align_array()), params_array (params_array()) and the descriptor `out`
        (align_out()) are read by the call; host-kind inputs and every array `out` names must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_align_batch_enqueue_each(self.h, align_array, n, params_array, kind, C.byref(out)),
                           "qb200_align_batch_enqueue_each")

    # ---- caller inlier sets -> poses (qb200_solve_pose_batch_each) ----
    inlier_array = staticmethod(_inlier_array)

    def solve_pose_batch_each(self, sets: Sequence, inliers: Sequence, params: Sequence[Params], kind: int = MEM_HOST,
                              buffers: Optional[ListBuffers] = None):
        """qb200_solve_pose_batch_each: set i (as solve_batch takes it) is solved from the ids inliers[i] (see inlier_array(); chain
        order, not sorted) with params[i]; buffers: a ListBuffers of SET_LISTS, or None for records only."""
        assert len(params) == len(sets)
        arr, keep = self.inlier_array(sets, inliers, kind)
        return self._batch_lists("qb200_solve_pose_batch_each", len(sets), (arr, len(sets), self.params_array(params), kind), buffers)

    def solve_pose_batch_enqueue_each_raw(self, inlier_array, n: int, params_array, kind: int, out: np.ndarray,
                                          buffers: Optional[ListBuffers] = None):
        """qb200_solve_pose_batch_enqueue_each: inlier_array (inlier_array()) and params_array (params_array()) are read by the call;
        the host arrays behind inlier_array, `out` and the buffers must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_solve_pose_batch_enqueue_each(self.h, inlier_array, n, params_array, kind, _ptr(out),
                                                                        self._lists_arg(buffers)), "qb200_solve_pose_batch_enqueue_each")

    def cache_scans_enqueue_each_raw(self, scan_ptrs, counts, slot_ids, n: int, params_array, kind: int):
        """qb200_cache_scans_enqueue_each: scan_ptrs / counts (_scan_arrays()), slot_ids (c_int32 * n) and params_array
        (params_array()) are read by the call; host-kind scans must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_cache_scans_enqueue_each(self.h, scan_ptrs, counts, slot_ids, n, params_array, kind),
                           "qb200_cache_scans_enqueue_each")

    # ---- raw scans -> voxel keypoints, normals and FPFH-33 (the front end in batches) ----
    def feature_buffers(self, n: int, cap: int, dest: int = MEM_HOST, arrays=tuple(FEATURE_ARRAYS)) -> dict:
        """Zeroed output arrays of a describe call by name: numpy (dest MEM_HOST) or CUDA tensors of the handle's device (MEM_DEVICE),
        each of shape (n, cap, floats per keypoint)."""
        shape = lambda k: (max(n, 1), cap, FEATURE_ARRAYS[k])
        if dest == MEM_HOST:
            return {k: np.zeros(shape(k), np.float32) for k in arrays}
        import torch
        return {k: torch.zeros(shape(k), dtype=torch.float32, device=f"cuda:{self.cfg.device}") for k in arrays}

    @staticmethod
    def feature_out(cap: int, dest: int, arrays: dict, counts: np.ndarray, status: np.ndarray) -> FeatureOut:
        """The qb200_feature_out of `arrays` (feature_buffers()) and the host int32 arrays counts / status; a name left out is NULL."""
        out = FeatureOut(cap, dest)
        for k, a in arrays.items():
            setattr(out, k, a.ctypes.data if dest == MEM_HOST else a.data_ptr())
        out.counts, out.status = counts.ctypes.data, status.ctypes.data
        return out

    def describe_batch_each(self, scans: Sequence, params: Sequence[Params], kind: int = MEM_HOST, dest: int = MEM_HOST,
                            cap_per_scan: Optional[int] = None, arrays: Optional[dict] = None):
        """qb200_describe_batch_each: scan i (an (n,4) float32 array for MEM_HOST, a (device_ptr, n) tuple for MEM_DEVICE) is voxelized
        and described with the front-end fields of params[i].  cap_per_scan: keypoints reserved per scan (default max_voxel_points).
        arrays: the caller's own outputs by name (FEATURE_ARRAYS), numpy for dest MEM_HOST or CUDA tensors for MEM_DEVICE, each of
        shape (n, cap, 4 or 33); a name left out is NULL.  Returns (per scan a tuple (vox4, normals4, desc33) trimmed to
        min(count, cap): numpy copies, tensor views on the device, None for a NULL array; counts (n,) int32; status (n,) int32)."""
        return self._describe("qb200_describe_batch_each", tuple(FEATURE_ARRAYS), scans, params, kind, dest, cap_per_scan, arrays)

    def describe_batch_enqueue_each_raw(self, scan_ptrs, counts, n: int, params_array, kind: int, out: FeatureOut):
        """qb200_describe_batch_enqueue_each: scan_ptrs / counts (_scan_arrays()), params_array (params_array()) and the descriptor `out`
        (feature_out()) are read by the call; host-kind scans and every array `out` names must stay alive until register_batch_flush."""
        return self._check(self.lib.qb200_describe_batch_enqueue_each(self.h, scan_ptrs, counts, n, params_array, kind, C.byref(out)),
                           "qb200_describe_batch_enqueue_each")

    # ---- raw scans -> voxel centroids (the voxel filter in batches) ----
    def voxelize_batch_each(self, scans: Sequence, params: Sequence[Params], kind: int = MEM_HOST, dest: int = MEM_HOST,
                            cap_per_scan: Optional[int] = None, arrays: Optional[dict] = None):
        """qb200_voxelize_batch_each: scan i (an (n,4) float32 array for MEM_HOST, a (device_ptr, n) tuple for MEM_DEVICE) is filtered
        with params[i].voxel_size and skip_flagged, as voxelize() filters it.  cap_per_scan: entries reserved per scan (default
        max_voxel_points).  arrays: the caller's own vox4 output ({"vox4": ...}, numpy for dest MEM_HOST or a CUDA tensor for MEM_DEVICE,
        shape (n, cap, 4)), or {} for counts and status only.  Returns (per scan its vox4 trimmed to min(count, cap): a numpy copy, a
        tensor view on the device, None without vox4; counts (n,) int32; status (n,) int32)."""
        per_scan, counts, status = self._describe("qb200_voxelize_batch_each", VOXEL_ARRAYS, scans, params, kind, dest, cap_per_scan,
                                                  arrays)
        return [v[0] for v in per_scan], counts, status

    def voxelize_batch_enqueue_each_raw(self, scan_ptrs, counts, n: int, params_array, kind: int, out: FeatureOut):
        """qb200_voxelize_batch_enqueue_each: scan_ptrs / counts (_scan_arrays()), params_array (params_array()) and the descriptor `out`
        (feature_out(), vox4 only or nothing) are read by the call; host-kind scans and every array `out` names must stay alive until
        register_batch_flush."""
        return self._check(self.lib.qb200_voxelize_batch_enqueue_each(self.h, scan_ptrs, counts, n, params_array, kind, C.byref(out)),
                           "qb200_voxelize_batch_enqueue_each")

    # ---- caller keypoint clouds -> normals and FPFH-33 (FPFH without the voxel filter, in batches) ----
    def describe_points_each(self, clouds: Sequence, params: Sequence[Params], kind: int = MEM_HOST, dest: int = MEM_HOST,
                             cap_per_scan: Optional[int] = None, arrays: Optional[dict] = None):
        """qb200_describe_points_each: cloud i (an (n,4) float32 array for MEM_HOST, a (device_ptr, n) tuple for MEM_DEVICE) is described
        as it is with the lattice fields of params[i].  cap_per_scan: keypoints reserved per cloud (default max_voxel_points).  arrays:
        the caller's own normals4 / desc33 outputs by name, numpy for dest MEM_HOST or CUDA tensors for MEM_DEVICE, each of shape
        (n, cap, 4 or 33); a name left out is NULL.  Returns (per cloud a tuple (normals4, desc33) trimmed to min(count, cap): numpy
        copies, tensor views on the device, None for a NULL array; counts (n,) int32; status (n,) int32)."""
        return self._describe("qb200_describe_points_each", POINT_ARRAYS, clouds, params, kind, dest, cap_per_scan, arrays)

    def _describe(self, fn: str, names, clouds, params, kind, dest, cap_per_scan, arrays):
        """The blocking describe and voxelize calls: `names` = the output arrays the call can fill, in the order of the returned
        tuples."""
        n = len(clouds)
        assert len(params) == n
        cap = cap_per_scan or self.cfg.max_voxel_points
        arrays = self.feature_buffers(n, cap, dest, names) if arrays is None else arrays
        counts, status = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.int32)
        ptrs, cnts, keep = _scan_arrays(clouds, kind)
        out = self.feature_out(cap, dest, arrays, counts, status)
        self._check(getattr(self.lib, fn)(self.h, ptrs, cnts, n, self.params_array(params), kind, C.byref(out)), fn)
        per_cloud = []
        for i in range(n):
            m = min(int(counts[i]), cap)
            per_cloud.append(tuple(None if k not in arrays else (arrays[k][i, :m].copy() if dest == MEM_HOST else arrays[k][i, :m])
                                   for k in names))
        return per_cloud, counts[:n], status[:n]

    def describe_points_enqueue_each_raw(self, cloud_ptrs, counts, n: int, params_array, kind: int, out: FeatureOut):
        """qb200_describe_points_enqueue_each: cloud_ptrs / counts (_scan_arrays()), params_array (params_array()) and the descriptor
        `out` (feature_out(), without vox4) are read by the call; host-kind clouds and every array `out` names must stay alive until
        register_batch_flush."""
        return self._check(self.lib.qb200_describe_points_enqueue_each(self.h, cloud_ptrs, counts, n, params_array, kind, C.byref(out)),
                           "qb200_describe_points_enqueue_each")

    def last_features(self, which: int, cap: Optional[int] = None):
        """(normals (n,4), descriptors (n,33)) of the source (0) / target (1) cloud of the last match_and_pack."""
        cap = cap or self.cfg.max_voxel_points
        nrm, desc = np.zeros((cap, 4), np.float32), np.zeros((cap, 33), np.float32)
        n = C.c_int32(0)
        self._check(self.lib.qb200_get_last_features(self.h, which, _ptr(nrm), _ptr(desc), cap, C.byref(n)), "qb200_get_last_features")
        m = min(n.value, cap)
        return nrm[:m].copy(), desc[:m].copy()

    # ---- scan cache ----
    def cache_reserve(self, n_slots: int):
        self._check(self.lib.qb200_cache_reserve(self.h, n_slots), "qb200_cache_reserve")

    def cache_scans(self, scans: Sequence, slot_ids: Sequence[int], params: Params, kind: int = MEM_HOST):
        """scans: (n,4) float32 arrays (MEM_HOST) or (device_ptr, n) tuples (MEM_DEVICE)."""
        n = len(scans)
        ptrs, cnts, keep = _scan_arrays(scans, kind)
        ids = (C.c_int32 * max(n, 1))(*[int(x) for x in slot_ids])
        self._check(self.lib.qb200_cache_scans(self.h, ptrs, cnts, ids, n, C.byref(params), kind), "qb200_cache_scans")

    def cache_scans_each(self, scans: Sequence, slot_ids: Sequence[int], params: Sequence[Params], kind: int = MEM_HOST):
        """qb200_cache_scans_each: scan i goes to slot_ids[i], voxelized and described with params[i]."""
        n = len(scans)
        assert len(params) == n
        ptrs, cnts, keep = _scan_arrays(scans, kind)
        ids = (C.c_int32 * max(n, 1))(*[int(x) for x in slot_ids])
        self._check(self.lib.qb200_cache_scans_each(self.h, ptrs, cnts, ids, n, self.params_array(params), kind), "qb200_cache_scans_each")

    def register_cached(self, slot_pairs, params: Params) -> np.ndarray:
        sp = _slot_array(slot_pairs)
        out = np.zeros(len(sp), RESULT_DTYPE)
        self._check(self.lib.qb200_register_cached(self.h, _ptr(sp), len(sp), C.byref(params), _ptr(out)), "qb200_register_cached")
        return out

    def cache_copy(self, from_slot: int, to_slot: int):
        self._check(self.lib.qb200_cache_copy(self.h, from_slot, to_slot), "qb200_cache_copy")

    def cache_read(self, slot: int, cap: Optional[int] = None):
        """-> (voxel points (n,4), normals (n,4), descriptors (n,33)) of a cached scan."""
        cap = cap or self.cfg.max_voxel_points
        vox, nrm, desc = np.zeros((cap, 4), np.float32), np.zeros((cap, 4), np.float32), np.zeros((cap, 33), np.float32)
        n = C.c_int32(0)
        self._check(self.lib.qb200_cache_read(self.h, slot, _ptr(vox), _ptr(nrm), _ptr(desc), cap, C.byref(n)), "qb200_cache_read")
        m = min(n.value, cap)
        return vox[:m].copy(), nrm[:m].copy(), desc[:m].copy()

    # ---- multi-GPU (comm.cu) ----
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        st = load_library().qb200_comm_unique_id(buf)
        if st != 0:
            raise QuatroB200Error(st, "qb200_comm_unique_id")
        return buf.raw

    def comm_init_rank(self, world: int, rank: int, unique_id: bytes):
        buf = C.create_string_buffer(unique_id, 128)
        self._check(self.lib.qb200_comm_init_rank(self.h, world, rank, buf), "qb200_comm_init_rank")
        self.world, self.rank = world, rank

    def register_batch_rank_raw(self, pair_array, n_local: int, params: Params, kind: int, out_all: np.ndarray, defer: bool = False):
        """out_all: RESULT_DTYPE array of world * n_local records, filled in round-robin global order (index i * world + r)."""
        return self._check(self.lib.qb200_register_batch_rank(self.h, pair_array, n_local, C.byref(params), kind, _ptr(out_all), int(defer)),
                           "qb200_register_batch_rank")

    def bind_numa(self) -> int:
        return int(self.lib.qb200_bind_numa(self.h))

    def comm_wait(self):
        return self._check(self.lib.qb200_comm_wait(self.h), "qb200_comm_wait")

    def register_batch_raw(self, pair_array, n: int, params: Params, kind: int, out: np.ndarray):
        """Zero-overhead variant for bench.py: pre-built (Pair * n) array and RESULT_DTYPE output."""
        return self._check(self.lib.qb200_register_batch(self.h, pair_array, n, C.byref(params), kind, _ptr(out)), "qb200_register_batch")

    def register_batch_enqueue_raw(self, pair_array, n: int, params: Params, kind: int, out: np.ndarray):
        """Pipelined form: queue the batch (pair_array, its scans and `out` must stay alive until register_batch_flush)."""
        return self._check(self.lib.qb200_register_batch_enqueue(self.h, pair_array, n, C.byref(params), kind, _ptr(out)), "qb200_register_batch_enqueue")

    def register_batch_flush(self):
        return self._check(self.lib.qb200_register_batch_flush(self.h), "qb200_register_batch_flush")

    def last_clique(self, cap: int = 1 << 16):
        idx = np.zeros(cap, np.int32)
        n = C.c_int32(0)
        self._check(self.lib.qb200_get_last_clique(self.h, _ptr(idx), cap, C.byref(n)), "qb200_get_last_clique")
        return idx[: n.value].copy()

    def last_final_inliers(self, cap: int = 1 << 16):
        idx = np.zeros(cap, np.int32)
        n = C.c_int32(0)
        self._check(self.lib.qb200_get_last_final_inliers(self.h, _ptr(idx), cap, C.byref(n)), "qb200_get_last_final_inliers")
        return idx[: n.value].copy()

    def last_correspondences(self, cap: int = 1 << 16):
        corr = np.zeros((cap, 2), np.int32)
        sm = np.zeros((cap, 4), np.float32)
        tm = np.zeros((cap, 4), np.float32)
        n = C.c_int32(0)
        self._check(self.lib.qb200_get_last_correspondences(self.h, _ptr(corr), _ptr(sm), _ptr(tm), cap, C.byref(n)),
                    "qb200_get_last_correspondences")
        return corr[: n.value].copy(), sm[: n.value].copy(), tm[: n.value].copy()

    def debug_match_stats(self, reset: bool = True) -> dict:
        out = np.zeros(4, np.uint64)
        self._check(self.lib.qb200_debug_match_stats(self.h, _ptr(out), int(reset)), "qb200_debug_match_stats")
        return {"exact_evals": int(out[0]), "tiles": int(out[1]), "aborted_stripes": int(out[3])}

    def debug_nn_tables(self, n_src: int, n_tgt: int):
        """(best target of every source point, best source of every target point) of the last match, packed uint64
        (distance bits << 32 | index), ~0 = none."""
        rb, cb = np.full(n_src, ~np.uint64(0)), np.full(n_tgt, ~np.uint64(0))
        self._check(self.lib.qb200_debug_nn_tables(self.h, _ptr(rb), n_src, _ptr(cb), n_tgt), "qb200_debug_nn_tables")
        return rb, cb

    def debug_tc_profile(self, reset: bool = True) -> np.ndarray:
        out = np.zeros(24, np.uint64)
        self._check(self.lib.qb200_debug_tc_profile(self.h, _ptr(out), int(reset)), "qb200_debug_tc_profile")
        return out

    def debug_tc_footprint(self) -> dict:
        """Threads, shared memory, registers and resident CTAs per SM of the tensor-core nearest-neighbour kernel."""
        out = np.zeros(5, np.int32)
        self._check(self.lib.qb200_debug_tc_footprint(self.h, _ptr(out)), "qb200_debug_tc_footprint")
        return {"threads": int(out[0]), "dyn_smem": int(out[1]), "static_smem": int(out[2]), "regs": int(out[3]),
                "ctas_per_sm": int(out[4])}

    def debug_match_verify(self, reset: bool = True) -> dict:
        out = np.zeros(2, np.uint64)
        self._check(self.lib.qb200_debug_match_verify(self.h, _ptr(out), int(reset)), "qb200_debug_match_verify")
        return {"compared": int(out[0]), "mismatches": int(out[1])}

    def debug_tc_distances(self, a33, b33) -> np.ndarray:
        a33, b33 = _f32(a33, 33), _f32(b33, 33)
        out = np.zeros((128, 128), np.float32)
        self._check(self.lib.qb200_debug_tc_distances(self.h, _ptr(a33), len(a33), _ptr(b33), len(b33), _ptr(out)), "qb200_debug_tc_distances")
        return out[: len(a33), : len(b33)].copy()

    def kernel_ms(self):
        """(ms, launches) of the two roofline kernels during the last register_batch:
        index 0 = match_stripe_kernel (K6), 1 = tim_graph_kernel (K8)."""
        ms = np.zeros(2, np.float32)
        calls = np.zeros(2, np.int32)
        self.lib.qb200_get_kernel_ms(self.h, _ptr(ms), _ptr(calls), 2)
        return ms, calls

    def stage_ms(self) -> np.ndarray:
        ms = np.zeros(8, np.float32)
        self.lib.qb200_get_stage_ms(self.h, _ptr(ms), 8)
        return ms
