"""ctypes wrapper of oracle/build/libquatro_oracle.so (TEST INFRASTRUCTURE)."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path
from typing import Optional

import numpy as np

from quatro_b200.capi import Params, Result, _f32, _ptr

HERE = Path(__file__).resolve().parent
LIB = HERE / "build" / "libquatro_oracle.so"


class Oracle:
    def __init__(self, build: bool = True):
        srcs = [HERE / "quatro_oracle.cpp", HERE / "preprocess_oracle.inc", HERE / "qo_math.h", HERE.parent / "include" / "quatro_b200.h"]
        stale = (not LIB.exists()) or any(s.stat().st_mtime > LIB.stat().st_mtime for s in srcs)
        if stale and build:
            r = subprocess.run(["make", "-C", str(HERE)], capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError("oracle build failed:\n" + r.stdout + r.stderr)
        self.lib = C.CDLL(str(LIB))
        L = self.lib
        L.qo_test_atan2f.restype = C.c_float
        L.qo_test_atan2f.argtypes = [C.c_float, C.c_float]
        L.qo_test_acosf.restype = C.c_float
        L.qo_test_acosf.argtypes = [C.c_float]
        L.qo_test_cote.restype = C.c_double
        L.qo_test_cote.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_int, C.c_void_p]
        L.qo_test_gnc.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(Params), C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
        L.qo_voxelize.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        L.qo_compute_fpfh.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
        L.qo_neighbors.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_int]
        L.qo_match.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.POINTER(Params), C.c_void_p, C.c_int,
                               C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p]
        L.qo_nn_tables.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.qo_build_graph.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_void_p, C.c_int, C.c_void_p,
                                     C.POINTER(C.c_int64)]
        L.qo_max_clique.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_void_p, C.POINTER(C.c_int), C.c_void_p,
                                    C.c_void_p, C.POINTER(C.c_int)]
        L.qo_max_clique_ex.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int64, C.c_void_p, C.POINTER(C.c_int),
                                       C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.qo_solve_pose.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(Params), C.POINTER(Result),
                                    C.c_void_p, C.c_void_p, C.c_void_p]
        L.qo_solve_correspondences.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(Params), C.POINTER(Result), C.c_void_p,
                                               C.POINTER(C.c_int), C.c_void_p, C.POINTER(C.c_int)]
        L.qo_match_and_pack.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(Params), C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.qo_register_pair.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(Params), C.POINTER(Result), C.c_void_p]
        L.qo_test_philox.argtypes = [C.c_uint64, C.c_uint64, C.c_void_p]
        L.qo_test_kcore.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]

    def set_literal(self, on: bool) -> bool:
        """Literal mode: libstdc++ std::sort on tied keys and distance-ordered neighbour accumulation instead of the determinism
        fixes D3 / D8 (measurement only; the CUDA library is compared with the canonical mode).  Returns the previous mode."""
        return bool(self.lib.qo_set_literal(1 if on else 0))

    def set_num_threads(self, n: int) -> int:
        return self.lib.qo_set_num_threads(n)

    # ---- math ---------------------------------------------------------------------------------
    def atan2f(self, y, x):
        return np.array([self.lib.qo_test_atan2f(float(a), float(b)) for a, b in zip(np.ravel(y), np.ravel(x))], np.float32)

    def acosf(self, x):
        return np.array([self.lib.qo_test_acosf(float(a)) for a in np.ravel(x)], np.float32)

    def sincosf(self, x):
        s, c = C.c_float(), C.c_float()
        out = []
        for a in np.ravel(x):
            self.lib.qo_test_sincosf(C.c_float(float(a)), C.byref(s), C.byref(c))
            out.append((s.value, c.value))
        return np.array(out, np.float32)

    def philox(self, seed: int, ctr: int):
        o = np.zeros(4, np.uint32)
        self.lib.qo_test_philox(seed, ctr, _ptr(o))
        return o

    def svd2x2(self, H):
        H = np.ascontiguousarray(H, np.float64).reshape(4)
        U, S, V = np.zeros(4), np.zeros(2), np.zeros(4)
        self.lib.qo_test_svd2x2(_ptr(H), _ptr(U), _ptr(S), _ptr(V))
        return U.reshape(2, 2), S, V.reshape(2, 2)

    def svd_rot2d(self, X, Y, W):
        X, Y, W = (np.ascontiguousarray(a, np.float64) for a in (X, Y, W))
        R = np.zeros(4)
        self.lib.qo_test_svd_rot2d(_ptr(X), _ptr(Y), _ptr(W), X.shape[1], _ptr(R))
        return R.reshape(2, 2)

    def pair_features(self, p1, n1, p2, n2):
        a = [np.ascontiguousarray(list(v) + [0.0] * (4 - len(v)), np.float32) for v in (p1, n1, p2, n2)]
        f = np.zeros(3, np.float32)
        ok = self.lib.qo_test_pair_features(_ptr(a[0]), _ptr(a[1]), _ptr(a[2]), _ptr(a[3]), _ptr(f))
        return bool(ok), f

    def cote(self, X, rng: float, median: bool = True):
        X = np.ascontiguousarray(X, np.float64)
        inl = np.zeros(len(X), np.uint8)
        e = self.lib.qo_test_cote(_ptr(X), len(X), rng, int(median), _ptr(inl))
        return e, inl.astype(bool)

    def gnc(self, src2, dst2, params: Params, rot_nb: float):
        src2, dst2 = np.ascontiguousarray(src2, np.float64), np.ascontiguousarray(dst2, np.float64)
        c = src2.shape[1]
        R, inl, cost = np.zeros(4), np.zeros(c, np.uint8), np.zeros(1)
        it = self.lib.qo_test_gnc(_ptr(src2), _ptr(dst2), c, C.byref(params), rot_nb, _ptr(R), _ptr(inl), _ptr(cost))
        return R.reshape(2, 2), inl.astype(bool), float(cost[0]), it

    def kcore(self, adj):
        adj = np.ascontiguousarray(adj, np.uint32)
        L, wpr = adj.shape
        k, o = np.zeros(L, np.int32), np.zeros(L, np.int32)
        mc = self.lib.qo_test_kcore(_ptr(adj), L, wpr, _ptr(k), _ptr(o))
        return k, o, mc

    # ---- stages (same signatures as quatro_b200.capi.Handle) --------------------------------------
    def voxelize(self, pts4, leaf: float, skip_flagged: int = 1, cap: Optional[int] = None):
        pts4 = _f32(pts4, 4)
        cap = cap or max(1, len(pts4))
        out = np.zeros((cap, 4), np.float32)
        n = C.c_int(0)
        st = self.lib.qo_voxelize(_ptr(pts4), len(pts4), leaf, skip_flagged, _ptr(out), cap, C.byref(n))
        return out[: min(n.value, cap)].copy(), st

    def compute_fpfh(self, pts4, normal_radius: float, fpfh_radius: float, grid_cell: float, want_spfh: bool = False):
        pts4 = _f32(pts4, 4)
        n = len(pts4)
        normals, desc = np.zeros((n, 4), np.float32), np.zeros((n, 33), np.float32)
        spfh = np.zeros((n, 33), np.float32) if want_spfh else None
        st = self.lib.qo_compute_fpfh(_ptr(pts4), n, normal_radius, fpfh_radius, grid_cell, _ptr(normals), _ptr(desc), _ptr(spfh))
        assert st == 0, st
        return (normals, desc, spfh) if want_spfh else (normals, desc)

    def neighbors(self, pts4, grid_cell: float, q: int, radius: float, cap: int = 4096):
        pts4 = _f32(pts4, 4)
        idx, d2 = np.zeros(cap, np.int32), np.zeros(cap, np.float32)
        k = self.lib.qo_neighbors(_ptr(pts4), len(pts4), grid_cell, q, radius, _ptr(idx), _ptr(d2), cap)
        return idx[:k].copy(), d2[:k].copy()

    def match(self, src4, sdesc, tgt4, tdesc, params: Params, cap: Optional[int] = None, want_mutual: bool = False):
        src4, tgt4, sdesc, tdesc = _f32(src4, 4), _f32(tgt4, 4), _f32(sdesc, 33), _f32(tdesc, 33)
        cap = cap or max(1, min(len(src4), len(tgt4)))
        corr = np.zeros((cap, 2), np.int32)
        mutual = np.zeros((max(1, min(len(src4), len(tgt4))), 2), np.int32)
        n, nm = C.c_int(0), C.c_int(0)
        st = self.lib.qo_match(_ptr(src4), len(src4), _ptr(sdesc), _ptr(tgt4), len(tgt4), _ptr(tdesc), C.byref(params), _ptr(corr), cap,
                               C.byref(n), C.byref(nm), _ptr(mutual))
        assert st >= 0, st
        if want_mutual:
            return corr[: min(n.value, cap)].copy(), nm.value, st, mutual[: nm.value].copy()
        return corr[: min(n.value, cap)].copy(), nm.value, st

    def nn_tables(self, adesc, bdesc):
        """Both nearest-neighbour tables of match() for adesc (rows) against bdesc (columns), without the larger-cloud swap:
        (best B of every A row, best A of every B column) as packed uint64 (distance bits << 32 | index), ~0 = none."""
        adesc, bdesc = _f32(adesc, 33), _f32(bdesc, 33)
        ba, bb = np.zeros(len(adesc), np.uint64), np.zeros(len(bdesc), np.uint64)
        st = self.lib.qo_nn_tables(_ptr(adesc), len(adesc), _ptr(bdesc), len(bdesc), _ptr(ba), _ptr(bb))
        assert st == 0, st
        return ba, bb

    def build_graph(self, a4, b4, noise_bound: float, cbar2: float, words_per_row: Optional[int] = None):
        a4, b4 = _f32(a4, 4), _f32(b4, 4)
        L = len(a4)
        wpr = words_per_row or (L + 31) // 32
        adj, deg, ne = np.zeros((L, wpr), np.uint32), np.zeros(L, np.int32), C.c_int64(0)
        st = self.lib.qo_build_graph(_ptr(a4), _ptr(b4), L, noise_bound, cbar2, _ptr(adj), wpr, _ptr(deg), C.byref(ne))
        assert st == 0
        return adj, deg, ne.value

    def patchwork(self, pts, pp):
        pts = _f32(pts, 4)
        n = len(pts)
        g, ng = np.zeros((max(n, 1), 4), np.float32), np.zeros((max(n, 1), 4), np.float32)
        a, b = C.c_int(0), C.c_int(0)
        self.lib.qo_patchwork.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_void_p, C.POINTER(C.c_int)]
        st = self.lib.qo_patchwork(_ptr(pts), n, C.byref(pp), _ptr(g), C.byref(a), _ptr(ng), C.byref(b))
        assert st >= 0, st
        return g[: a.value].copy(), ng[: b.value].copy(), st

    def segment_cloud(self, pts, sp):
        pts = _f32(pts, 4)
        npix = sp.n_scan * sp.horizon_scan
        v, o = np.zeros((npix, 4), np.float32), np.zeros((npix, 4), np.float32)
        a, b = C.c_int(0), C.c_int(0)
        self.lib.qo_segment_cloud.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_void_p, C.POINTER(C.c_int)]
        st = self.lib.qo_segment_cloud(_ptr(pts), len(pts), C.byref(sp), _ptr(v), C.byref(a), _ptr(o), C.byref(b))
        assert st >= 0, st
        return v[: a.value].copy(), o[: b.value].copy()

    def max_clique(self, adj, mode: int = 1, kcore_thr: float = 0.5):
        adj = np.ascontiguousarray(adj, np.uint32)
        L, wpr = adj.shape
        clique, kcore, order = (np.zeros(max(L, 1), np.int32) for _ in range(3))
        n, mc = C.c_int(0), C.c_int(0)
        st = self.lib.qo_max_clique(_ptr(adj), L, wpr, mode, kcore_thr, _ptr(clique), C.byref(n), _ptr(kcore), _ptr(order), C.byref(mc))
        assert st >= 0, st
        return clique[: n.value].copy(), kcore[:L].copy(), order[:L].copy(), mc.value

    def max_clique_ex(self, adj, mode: int = 0, kcore_thr: float = 0.5, node_limit: int = 0):
        adj = np.ascontiguousarray(adj, np.uint32)
        L, wpr = adj.shape
        clique, kcore, order = (np.zeros(max(L, 1), np.int32) for _ in range(3))
        n, mc, fl = C.c_int(0), C.c_int(0), C.c_int(0)
        st = self.lib.qo_max_clique_ex(_ptr(adj), L, wpr, mode, kcore_thr, node_limit, _ptr(clique), C.byref(n), _ptr(kcore), _ptr(order),
                                       C.byref(mc), C.byref(fl))
        assert st >= 0, st
        return clique[: n.value].copy(), kcore[:L].copy(), order[:L].copy(), mc.value, fl.value

    def solve_pose(self, a4, b4, clique, params: Params, want_final: bool = False):
        """want_final: also return the final inlier list (correspondence ids, getFinalInliersIndices) as a fifth element."""
        a4, b4 = _f32(a4, 4), _f32(b4, 4)
        clique = np.ascontiguousarray(clique, np.int32)
        res = Result()
        rm, tm = np.zeros(max(len(clique), 1), np.uint8), np.zeros(max(len(clique), 1), np.uint8)
        fi = np.zeros(max(len(clique), 1), np.int32)
        st = self.lib.qo_solve_pose(_ptr(a4), _ptr(b4), len(a4), _ptr(clique), len(clique), C.byref(params), C.byref(res), _ptr(rm), _ptr(tm),
                                    _ptr(fi))
        out = (res, rm[: len(clique)], tm[: len(clique)], st)
        return out + (fi[: res.n_final_inliers].copy(),) if want_final else out

    def solve_correspondences(self, a4, b4, params: Params, want_sets: bool = False):
        a4, b4 = _f32(a4, 4), _f32(b4, 4)
        L = len(a4)
        res = Result()
        clique, fin = np.zeros(max(L, 1), np.int32), np.zeros(max(L, 1), np.int32)
        nc, nf = C.c_int(0), C.c_int(0)
        st = self.lib.qo_solve_correspondences(_ptr(a4), _ptr(b4), L, C.byref(params), C.byref(res), _ptr(clique), C.byref(nc), _ptr(fin),
                                               C.byref(nf))
        if want_sets:
            return res, st, clique[: nc.value].copy(), fin[: nf.value].copy()
        return res, st

    def match_and_pack(self, src4, tgt4, params: Params, cap: Optional[int] = None):
        src4, tgt4 = _f32(src4, 4), _f32(tgt4, 4)
        cap = cap or max(1, min(len(src4), len(tgt4)))
        corr, sm, tm = np.zeros((cap, 2), np.int32), np.zeros((cap, 4), np.float32), np.zeros((cap, 4), np.float32)
        n, nm = C.c_int(0), C.c_int(0)
        st = self.lib.qo_match_and_pack(_ptr(src4), len(src4), _ptr(tgt4), len(tgt4), C.byref(params), _ptr(corr), _ptr(sm), _ptr(tm), cap,
                                        C.byref(n), C.byref(nm))
        m = min(n.value, cap)
        return corr[:m].copy(), sm[:m].copy(), tm[:m].copy(), st

    def register_pair(self, src4, tgt4, params: Params, want_times: bool = False):
        src4, tgt4 = _f32(src4, 4), _f32(tgt4, 4)
        res = Result()
        ts = np.zeros(8, np.float64)
        st = self.lib.qo_register_pair(_ptr(src4), len(src4), _ptr(tgt4), len(tgt4), C.byref(params), C.byref(res), _ptr(ts))
        return (res, st, ts) if want_times else (res, st)
