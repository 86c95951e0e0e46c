"""Synthetic scan pairs (host side, deterministic per seed) -- input generator for tests and bench.

outdoor_pair() wraps quatro_b200/synth/synth.cpp (64-ring HDL-64E geometry, SURVEY.md 8d config 2).
matched_pairs() makes correspondence sets (inliers under a known yaw/translation + outliers) for
the back-end stages.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _build

_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        lib = C.CDLL(str(_build.build_synth()))
        lib.qb200_synth_outdoor_pair.restype = C.c_int
        lib.qb200_synth_outdoor_pair.argtypes = [C.c_uint64, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int), C.c_void_p,
                                                 C.POINTER(C.c_int), C.c_int, C.c_void_p]
        lib.qb200_synth_outdoor_pair_ex.restype = C.c_int
        lib.qb200_synth_outdoor_pair_ex.argtypes = [C.c_uint64, C.c_int, C.c_int, C.POINTER(Scene), C.c_void_p, C.POINTER(C.c_int),
                                                    C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_void_p]
        lib.qb200_synth_indoor_pair.restype = C.c_int
        lib.qb200_synth_indoor_pair.argtypes = [C.c_uint64, C.c_int, C.c_double, C.c_int, C.c_void_p, C.POINTER(C.c_int), C.c_void_p,
                                                C.POINTER(C.c_int), C.c_int, C.c_void_p]
        _LIB = lib
    return _LIB


class Scene(C.Structure):
    """struct qb200_synth_scene of synth.cpp."""
    _fields_ = [("n_build", C.c_int), ("n_pole", C.c_int), ("n_car", C.c_int), ("extent", C.c_double), ("max_dist", C.c_double),
                ("sigma", C.c_double), ("n_clutter", C.c_int)]


STREET = (30, 50, 15, 70.0, 10.0, 0.02, 0)       # BASELINE configs[1..3]: the street scene (mean L ~ 300 after the tuple test)


def outdoor_pair(seed: int, rings: int = 64, azimuths: int = 1800, scene=STREET):
    """Returns (src (n,4) float32, tgt (m,4) float32, T_gt 4x4 float64) with p_tgt = T_gt @ p_src.
    w = -1 marks ground returns.  scene = (n_build, n_pole, n_car, extent, max_dist, sigma, n_clutter)."""
    cap = rings * azimuths
    src = np.zeros((cap, 4), np.float32)
    tgt = np.zeros((cap, 4), np.float32)
    ns, nt = C.c_int(0), C.c_int(0)
    T = np.zeros(16, np.float64)
    sc = Scene(*scene)
    _lib().qb200_synth_outdoor_pair_ex(seed, rings, azimuths, C.byref(sc), src.ctypes.data, C.byref(ns), tgt.ctypes.data, C.byref(nt), cap,
                                       T.ctypes.data)
    return src[: ns.value].copy(), tgt[: nt.value].copy(), T.reshape(4, 4).T.copy()


def indoor_pair(seed: int, n_rays: int = 500000, extent: float = 3.0, n_furniture: int = 40):
    """Dense indoor pair (BASELINE configs[4]): a furnished room of 2*extent x 2*extent x 3 m scanned with n_rays uniformly distributed
    rays from two poses, 5 mm range noise, nothing flagged (the floor stays in).  The default 6 x 6 m room gives 34-53 k voxel points
    per cloud at a 0.05 m voxel; a 18 x 18 m hall (extent 9) gives 43-152 k (max_voxel_points up to 262144 holds either).  Returns (src (n,4), tgt (m,4), T_gt 4x4) with p_tgt = T_gt @ p_src."""
    src = np.zeros((n_rays, 4), np.float32)
    tgt = np.zeros((n_rays, 4), np.float32)
    ns, nt = C.c_int(0), C.c_int(0)
    T = np.zeros(16, np.float64)
    _lib().qb200_synth_indoor_pair(seed, n_rays, extent, n_furniture, src.ctypes.data, C.byref(ns), tgt.ctypes.data, C.byref(nt), n_rays,
                                   T.ctypes.data)
    return src[: ns.value].copy(), tgt[: nt.value].copy(), T.reshape(4, 4).T.copy()


def matched_pairs(seed: int, L: int, inlier_ratio: float = 0.3, noise: float = 0.05, extent: float = 50.0,
                  yaw_deg: float | None = None, trans=None):
    """L matched point pairs (a_i, b_i): inliers b = Rz(yaw) a + t + noise, outliers random.
    Returns a4 (L,4) f32, b4 (L,4) f32, T_gt 4x4, inlier mask."""
    rng = np.random.default_rng(seed)
    yaw = np.deg2rad(rng.uniform(-180, 180) if yaw_deg is None else yaw_deg)
    t = rng.uniform(-5, 5, 3) * np.array([1, 1, 0.05]) if trans is None else np.asarray(trans, float)
    R = np.array([[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]])
    a = rng.uniform(-extent, extent, (L, 3)) * np.array([1, 1, 0.1])
    inl = rng.uniform(size=L) < inlier_ratio
    b = a @ R.T + t + rng.normal(0, noise, (L, 3))
    b[~inl] = rng.uniform(-extent, extent, ((~inl).sum(), 3)) * np.array([1, 1, 0.1])
    a4 = np.ones((L, 4), np.float32)
    b4 = np.ones((L, 4), np.float32)
    a4[:, :3] = a
    b4[:, :3] = b
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = t
    return a4, b4, T, inl


def pose_error(T_est: np.ndarray, T_ref: np.ndarray):
    """(rotation error in degrees, translation error in metres)."""
    dR = T_est[:3, :3] @ T_ref[:3, :3].T
    c = np.clip((np.trace(dR) - 1) / 2, -1, 1)
    return float(np.degrees(np.arccos(c))), float(np.linalg.norm(T_est[:3, 3] - T_ref[:3, 3]))
