"""Batches of caller keypoints and descriptors of any length: qb200_match_descriptors_each / _enqueue_each and
qb200_register_descriptors_each / _enqueue_each.

The reference for other lengths is the matcher restated with a descriptor length and a row stride: both exact nearest-neighbour
searches in C++ (tests/fixtures/nn_dim_ref.cpp, fmaf chains over d = 0 .. dim - 1), the mutual check, and the tuple test of
tests/independent_ref.py.  On the CPU: the POD from a C compiler, a C++ program using the calls builds against the library, and the
restatement equals the oracle's qo_match / qo_nn_tables at 33 floats (whatever the stride, and with zero bins appended).  On the GPU,
against the restatement bit for bit (the full nearest-neighbour tables through qb200_debug_nn_tables, then the correspondences and
records): every length class of
nn_dim_kernel with stride = dim and stride > dim, the stripe and chunk edges, and adversarial descriptors.  FPFH-33 rows padded with
zero bins to 34 and 40 floats (run by nn_dim_kernel) and 33-float rows at a wider stride (run by the tensor-core matcher) give the
records and lists of the _features_ calls, on street pairs and on the tuple test's adversarial scenes.  A batch that mixes lengths,
strides and memory kinds over several waves and lanes equals its pairs alone; queued forms interleaved with other inputs equal the
blocking calls; register lists solve again to the same records; a lane soiled by a 512-float wave at capacity gives a fresh handle's
output; and every rejection happens before anything runs."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from independent_ref import tuple_match
from quatro_b200 import capi, synth
from quatro_b200.capi import (MATCH_LISTS, MEM_DEVICE, MEM_HOST, RESULT_DTYPE, DescriptorPair, ListBuffers, default_params)
from support import P4, ROOT, build_against_lib, device_copies, host_lists, make_handle, make_params, sentinel, sentinel_lists

NEW = ("qb200_match_descriptors_each", "qb200_match_descriptors_enqueue_each", "qb200_register_descriptors_each",
       "qb200_register_descriptors_enqueue_each")
DIMS = (1, 2, 7, 8, 31, 32, 34, 63, 64, 65, 125, 352, 512)


# ---- builders ----------------------------------------------------------------------------------------------------------------------
def _rows(desc, stride, fill=np.nan):
    """n x dim descriptors in rows of `stride` floats, the bins past dim set to `fill` (never read)"""
    desc = np.asarray(desc, np.float32)
    out = np.full((len(desc), stride), fill, np.float32)
    out[:, :desc.shape[1]] = desc
    return out


def _scene(rng, ns, nt, dim):
    """ns source keypoints and descriptors; the target holds the first min(ns, nt) of them moved, with descriptors perturbed, then
    random ones.  Descriptors are non-negative like histograms."""
    src, desc = P4(rng.uniform(-20, 20, (ns, 3))), rng.gamma(0.5, 1.0, (ns, dim)).astype(np.float32)
    m = min(ns, nt)
    c, s_ = np.cos(0.3), np.sin(0.3)
    R = np.array([[c, -s_, 0], [s_, c, 0], [0, 0, 1]])
    tgt_xyz = np.concatenate([src[:m, :3] @ R.T + [1.0, -2.0, 0.5] + rng.normal(0, 0.02, (m, 3)), rng.uniform(-20, 20, (nt - m, 3))])
    tdesc = np.concatenate([desc[:m] + rng.normal(0, 0.05, (m, dim)), rng.gamma(0.5, 1.0, (nt - m, dim))]).astype(np.float32)
    return src, desc, P4(tgt_xyz, w=0.5), tdesc


def _pair(scene, stride=None, fill=np.nan):
    """a host descriptor pair of register/match_descriptors_each: (src4, src_rows, tgt4, tgt_rows, dim)"""
    s, sd, t, td = scene
    dim = sd.shape[1]
    stride = stride or dim
    return s, _rows(sd, stride, fill), t, _rows(td, stride, fill), dim


def _device_pairs(pairs):
    """host descriptor pairs -> the MEM_DEVICE tuples, and the tensors behind them"""
    out, keep = [], []
    for s, sd, t, td, dim in pairs:
        _, ts = device_copies([s, sd, t, td])
        keep.append(ts)
        out.append((ts[0].data_ptr(), ts[1].data_ptr(), len(s), ts[2].data_ptr(), ts[3].data_ptr(), len(t), dim, sd.shape[1]))
    return out, keep


def _flat(recs, lb):
    return recs.tobytes(), [{k: v.tobytes() for k, v in d.items()} for d in host_lists(lb.trimmed(recs))]


# ---- the reference for any length ---------------------------------------------------------------------------------------------------
class DimRef:
    """The matcher on descriptor rows of any length: nn_dim_ref.cpp's two searches, the mutual check, independent_ref.tuple_match."""

    def __init__(self, path):
        self.lib = C.CDLL(str(path))
        self.lib.nn_tables_dim.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]

    def nn_tables(self, adesc, bdesc, dim):
        """(best B of every A row, best A of every B row) as packed uint64 (distance bits << 32 | index), ~0 = none; the stride is
        the rows' width"""
        a, b = np.ascontiguousarray(adesc, np.float32), np.ascontiguousarray(bdesc, np.float32)
        assert a.ndim == b.ndim == 2 and a.shape[1] == b.shape[1]
        ba, bb = np.zeros(len(a), np.uint64), np.zeros(len(b), np.uint64)
        assert self.lib.nn_tables_dim(a.ctypes.data, len(a), b.ctypes.data, len(b), dim, a.shape[1], ba.ctypes.data, bb.ctypes.data) == 0
        return ba, bb

    def match(self, s, sd, t, td, dim, p):
        """(correspondences as (source, target) rows, mutual count) of a pair with params p"""
        if len(s) == 0 or len(t) == 0:
            return np.zeros((0, 2), np.int32), 0
        ba, bb = self.nn_tables(sd, td, dim)
        none = np.uint64(0xFFFFFFFFFFFFFFFF)
        i = np.flatnonzero(ba != none)
        j = (ba[i] & np.uint64(0xFFFFFFFF)).astype(np.int64)
        back = bb[j]
        keep = (back != none) & ((back & np.uint64(0xFFFFFFFF)).astype(np.int64) == i)
        mutual = np.stack([i[keep], j[keep]], 1)
        r = tuple_match(s, t, mutual, p.use_tuple_test, p.tuple_scale, p.tuple_trials_per_corr, p.seed)
        return r["corr"], len(mutual)


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    out = tmp_path_factory.mktemp("nn_dim_ref") / "libnn_dim_ref.so"
    r = subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-ffp-contract=off", "-mfma", "-fno-fast-math", "-fPIC",
                        "-shared", str(ROOT / "tests" / "fixtures" / "nn_dim_ref.cpp"), "-o", str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return DimRef(out)


# ---- CPU ---------------------------------------------------------------------------------------------------------------------------
def test_descriptor_pair_mirror_matches_the_c_layout(tmp_path):
    """sizeof and every offsetof of qb200_descriptor_pair from a C compiler (the header compiles as C11), against the ctypes mirror."""
    body = '  printf("size %zu\\n", sizeof(qb200_descriptor_pair));\n  printf("max %d\\n", QB200_MAX_DESC_DIM);\n' + "".join(
        f'  printf("{f} %zu\\n", offsetof(qb200_descriptor_pair, {f}));\n' for f, _ in DescriptorPair._fields_)
    (tmp_path / "pod.c").write_text('#include <stddef.h>\n#include <stdio.h>\n#include "quatro_b200.h"\nint main(void) {\n' + body +
                                    "  return 0;\n}\n")
    r = subprocess.run(["/usr/bin/gcc", "-std=c11", "-Wall", "-Werror", "-pedantic", f"-I{ROOT / 'include'}", str(tmp_path / "pod.c"), "-o",
                        str(tmp_path / "pod")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    probe = dict(ln.split() for ln in subprocess.run([str(tmp_path / "pod")], capture_output=True, text=True, check=True).stdout.splitlines())
    assert C.sizeof(DescriptorPair) == int(probe["size"]) == 48
    assert int(probe["max"]) == capi.DESC_DIM_MAX == 512
    for f, _ in DescriptorPair._fields_:
        assert getattr(DescriptorPair, f).offset == int(probe[f]), f


def test_library_exports_the_descriptor_calls(tmp_path):
    lib = capi.load_library()
    for n in NEW:
        assert n in capi.EXPORTED_SYMBOLS and hasattr(lib, n)
        assert getattr(lib, n).argtypes == lib.qb200_match_features_each.argtypes
        assert getattr(lib, n)(None, None, 0, None, MEM_HOST, None, None) == -1
    build_against_lib(tmp_path, "tests/fixtures/descriptor_batch_shim.cpp")


def test_reference_at_33_floats_equals_the_oracle(oracle, ref):
    """the restatement at dim 33 equals qo_match / qo_nn_tables whatever the stride; zero bins appended add nothing"""
    rng = np.random.default_rng(3)
    s, sd, t, td = _scene(rng, 500, 420, 33)
    sd[::7] = 0.0
    sd[5, 3], td[9, :], td[11, 2], sd[20, :] = np.nan, np.inf, -np.inf, 3e38
    p = make_params(seed=7)
    corr, nm, st = oracle.match(s, sd, t, td, p, cap=4096)
    ta = oracle.nn_tables(sd, td)
    assert len(corr) > 50
    for stride in (33, 40):
        c2, nm2 = ref.match(s, _rows(sd, stride), t, _rows(td, stride), 33, p)
        assert st == 0 and nm2 == nm and np.array_equal(c2, corr), stride
        tb = ref.nn_tables(_rows(sd, stride), _rows(td, stride), 33)
        assert all(np.array_equal(a, b) for a, b in zip(ta, tb)), stride
    for dim in (34, 40):
        c2, nm2 = ref.match(s, _rows(sd, dim, 0.0), t, _rows(td, dim, 0.0), dim, p)
        assert nm2 == nm and np.array_equal(c2, corr), dim


# ---- GPU: against the reference -------------------------------------------------------------------------------------------------------
V_SMALL = 1024


@pytest.fixture(scope="module")
def h1():
    h = make_handle(1, max_batch_slots=4, max_voxel_points=V_SMALL, max_corr=1024)
    yield h
    h.close()


def _against_ref(h, ref, pair, p, label):
    """one pair through a one-pair match_descriptors_each: its nearest-neighbour tables, correspondences and record against the
    restatement"""
    s, sd, t, td, dim = pair
    lb = ListBuffers(1, h.cfg.max_corr, MEM_HOST, MATCH_LISTS)
    recs, lists = h.match_descriptors_each([pair], [p], buffers=lb)
    rec = recs[0]
    if len(s) and len(t):
        rb, cb = h.debug_nn_tables(len(s), len(t))
        ra, ca = ref.nn_tables(sd, td, dim)
        assert np.array_equal(rb, ra), f"{label}: row table differs at {np.flatnonzero(rb != ra)[:5]}"
        assert np.array_equal(cb, ca), f"{label}: column table differs at {np.flatnonzero(cb != ca)[:5]}"
    corr, nm = ref.match(s, sd, t, td, dim, p)
    assert np.array_equal(lists[0]["corr"], corr), f"{label}: correspondences differ"
    assert lists[0]["src_matched4"].tobytes() == s[corr[:, 0]].tobytes() and lists[0]["tgt_matched4"].tobytes() == t[corr[:, 1]].tobytes()
    assert (rec["n_mutual"], rec["n_corr"], rec["n_src_vox"], rec["n_tgt_vox"]) == (nm, len(corr), len(s), len(t)), label
    assert rec["status"] == (0 if len(s) and len(t) else 2), label
    return rec


@pytest.mark.gpu
@pytest.mark.parametrize("dim", DIMS)
def test_every_length_equals_the_reference(h1, ref, dim):
    rng = np.random.default_rng(dim)
    scene = _scene(rng, 300, 260, dim)
    for stride in (dim, dim + 5):
        for use_tuple in (1, 0):
            rec = _against_ref(h1, ref, _pair(scene, stride), make_params(use_tuple_test=use_tuple, seed=dim), f"{dim}/{stride}")
            assert rec["n_mutual"] > (20 if dim > 2 else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", (7, 64, 65))
def test_stripe_and_chunk_edges_equal_the_reference(h1, ref, dim):
    rng = np.random.default_rng(100 + dim)
    for ns, nt in ((1, 1), (1, 129), (127, 128), (128, 127), (129, 129), (V_SMALL, 127), (129, V_SMALL), (V_SMALL, V_SMALL)):
        _against_ref(h1, ref, _pair(_scene(rng, ns, nt, dim), dim + 3), make_params(seed=ns), f"{dim}: {ns} x {nt}")


def _adversarial(rng, dim):
    """(label, source rows, target rows): the matcher's hard cases at `dim` floats"""
    A, B = rng.gamma(0.5, 1.0, (400, dim)).astype(np.float32), rng.gamma(0.5, 1.0, (300, dim)).astype(np.float32)
    same = np.repeat(A[:1], 600, axis=0)
    ties_a = rng.integers(0, 2, (400, dim)).astype(np.float32)     # small integer distances: many candidates at equal distance
    ties_b = rng.integers(0, 2, (300, dim)).astype(np.float32)
    zeros_a, zeros_b = A.copy(), B.copy()
    zeros_a[::3] = 0.0
    zeros_b[::4] = 0.0
    bad_a, bad_b = A.copy(), B.copy()
    bad_a[5, dim // 2], bad_a[9, :] = np.nan, np.inf
    bad_a[11, dim - 1], bad_b[2, 0], bad_b[17, dim // 3] = -np.inf, np.nan, np.inf
    bad_b[30, :], bad_a[40, 0] = 3e38, 3e38
    return [("duplicate rows", np.concatenate([same, A[:50]]), np.concatenate([same[:400], B[:50]])),
            ("equal distances", ties_a, ties_b), ("all-zero rows", zeros_a, zeros_b), ("NaN, inf and 3e38", bad_a, bad_b),
            ("empty target", A, B[:0]), ("empty source", A[:0], B)]


@pytest.mark.gpu
@pytest.mark.parametrize("dim", (8, 125))
def test_adversarial_descriptors_equal_the_reference(h1, ref, dim):
    rng = np.random.default_rng(7 * dim)
    for label, A, B in _adversarial(rng, dim):
        a4, b4 = P4(rng.uniform(-30, 30, (len(A), 3))), P4(rng.uniform(-30, 30, (len(B), 3)))
        _against_ref(h1, ref, (a4, _rows(A, dim + 1), b4, _rows(B, dim + 1), dim), make_params(use_tuple_test=0), label)


# ---- GPU: zero-padded FPFH-33 through nn_dim_kernel, and 33 floats at another stride, equal the _features_ calls ---------------------
N_STREET = 10


@pytest.fixture(scope="module")
def street_feats():
    """keypoints and FPFH-33 of street pairs, read back from a scan cache"""
    pairs = [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(950, 950 + N_STREET)]
    with make_handle(1, max_batch_slots=4) as h:
        h.cache_reserve(2 * N_STREET)
        h.cache_scans([s for pr in pairs for s in pr], list(range(2 * N_STREET)), default_params())
        out = []
        for i in range(N_STREET):
            (sv, _, sd), (tv, _, td) = h.cache_read(2 * i), h.cache_read(2 * i + 1)
            out.append((sv, sd, tv, td))
    return out


def _padded(feats, dim, stride):
    """FPFH-33 pairs as descriptor pairs of `dim` floats (zero bins appended) in rows of `stride` floats"""
    return [(s, _rows(_rows(sd, dim, 0.0), stride), t, _rows(_rows(td, dim, 0.0), stride), dim) for s, sd, t, td in feats]


@pytest.mark.gpu
def test_padded_fpfh_equals_the_feature_calls_on_street_pairs(street_feats):
    params = [make_params(seed=3 + i, use_tuple_test=int(i % 3 != 1)) for i in range(N_STREET)]
    with make_handle(4, max_batch_slots=4) as h:
        for reg in (False, True):
            fn = "register" if reg else "match"
            lists = None if reg else MATCH_LISTS
            lb = ListBuffers(N_STREET, h.cfg.max_corr, MEM_HOST, *(() if reg else (lists,)))
            want = _flat(getattr(h, f"{fn}_features_each")(street_feats, params, buffers=lb)[0], lb)
            recs = np.frombuffer(want[0], RESULT_DTYPE)
            assert (recs["n_corr"] > 30).all() and (not reg or (recs["valid"] == 1).sum() >= N_STREET - 2)
            for dim, stride in ((33, 40), (34, 34), (34, 40), (40, 40)):
                pairs = _padded(street_feats, dim, stride)
                for kind in (MEM_HOST, MEM_DEVICE):
                    ps, keep = _device_pairs(pairs) if kind == MEM_DEVICE else (pairs, None)
                    lb = ListBuffers(N_STREET, h.cfg.max_corr, MEM_HOST, *(() if reg else (lists,)))
                    got = _flat(getattr(h, f"{fn}_descriptors_each")(ps, params, kind, buffers=lb)[0], lb)
                    assert got == want, (fn, dim, stride, kind)


@pytest.mark.gpu
def test_padded_fpfh_equals_the_feature_calls_on_tuple_scenes():
    from test_tuple_adversarial import CORR_MAX, scenes
    names = [n for n, sc in scenes().items() if max(len(sc.src), len(sc.tgt)) <= 4097]
    cap = min(CORR_MAX, 8192)
    with make_handle(4, max_batch_slots=8, max_voxel_points=8192, max_corr=cap) as h:
        feats = [(scenes()[n].src, scenes()[n].sdesc, scenes()[n].tgt, scenes()[n].tdesc) for n in names]
        params = [scenes()[n].params() for n in names]
        lb = ListBuffers(len(names), cap, MEM_HOST, MATCH_LISTS)
        want = _flat(h.match_features_each(feats, params, buffers=lb)[0], lb)
        for dim, stride in ((34, 40), (40, 40), (33, 36)):
            lb = ListBuffers(len(names), cap, MEM_HOST, MATCH_LISTS)
            got = _flat(h.match_descriptors_each(_padded(feats, dim, stride), params, buffers=lb)[0], lb)
            for k, n in enumerate(names):
                sz = RESULT_DTYPE.itemsize
                assert got[0][k * sz:(k + 1) * sz] == want[0][k * sz:(k + 1) * sz] and got[1][k] == want[1][k], (n, dim, stride)


# ---- GPU: batches ------------------------------------------------------------------------------------------------------------------
MIX = [(33, 33), (7, 7), (125, 128), (33, 40), (512, 512), (32, 32), (1, 4), (34, 40), (352, 361), (64, 64), (33, 33), (65, 70),
       (8, 8), (2, 2)]
MIX_SIZES = [(300, 280), (0, 40), (129, 128), (256, 300), (200, 150), (1, 1), (500, 450), (128, 129), (150, 140), (40, 0), (600, 600),
             (127, 255), (1024, 1000), (60, 61)]


def _mix(rng):
    pairs = [_pair(_scene(rng, ns, nt, dim), stride) for (dim, stride), (ns, nt) in zip(MIX, MIX_SIZES)]
    params = [make_params(seed=50 + i, use_tuple_test=i % 2, tuple_scale=(0.95, 0.9)[i % 2], inlier_selection_mode=(0, 1, 2, 3)[i % 4])
              for i in range(len(pairs))]
    return pairs, params


@pytest.mark.gpu
def test_a_mixed_batch_equals_each_pair_alone(h1):
    pairs, params = _mix(np.random.default_rng(9))
    with make_handle(4, max_batch_slots=4, max_voxel_points=V_SMALL, max_corr=1024) as h4:
        dev, keep = _device_pairs(pairs)
        for reg in (False, True):
            fn = "register_descriptors_each" if reg else "match_descriptors_each"
            kinds = (() if reg else (MATCH_LISTS,))
            single = []
            for pr, p in zip(pairs, params):
                lb = ListBuffers(1, 1024, MEM_HOST, *kinds)
                single.append(_flat(getattr(h1, fn)([pr], [p], buffers=lb)[0], lb))
            recs = np.frombuffer(b"".join(s[0] for s in single), RESULT_DTYPE)
            assert (recs["status"][[1, 9]] == 2).all() and (recs["n_corr"] > 20).sum() >= 8
            for h in (h1, h4):
                for kind, ps in ((MEM_HOST, pairs), (MEM_DEVICE, dev)):
                    lb = ListBuffers(len(pairs), 1024, MEM_DEVICE if kind == MEM_HOST else MEM_HOST, *kinds, device=h.cfg.device)
                    got = _flat(getattr(h, fn)(ps, params, kind, buffers=lb)[0], lb)
                    sz = RESULT_DTYPE.itemsize
                    for i in range(len(pairs)):
                        assert got[0][i * sz:(i + 1) * sz] == single[i][0], (fn, kind, MIX[i], MIX_SIZES[i])
                        assert got[1][i] == single[i][1][0], (fn, kind, MIX[i], MIX_SIZES[i])


@pytest.mark.gpu
def test_queued_forms_interleaved_with_other_inputs_equal_the_blocking_calls():
    pairs, params = _mix(np.random.default_rng(10))
    street = [synth.outdoor_pair(s, rings=16, azimuths=600)[:2] for s in range(960, 966)]
    rng = np.random.default_rng(11)
    feats = [_scene(rng, 300, 280, 33) for _ in range(6)]
    sp = [make_params(seed=i) for i in range(len(street))]
    with make_handle(4, max_batch_slots=4, max_voxel_points=4096, max_corr=1024) as h:
        h.cache_reserve(4)
        h.cache_scans([street[0][0], street[0][1], street[1][0], street[1][1]], [0, 1, 2, 3], default_params())
        dev, keep = _device_pairs(pairs)
        d_host, k1 = h.descriptor_array(pairs)
        d_dev, k2 = h.descriptor_array(dev, MEM_DEVICE)
        f_arr, k3 = h.feature_array(feats)
        p_arr, k4 = h.pair_array(street)
        s_arr = capi._slot_array([(0, 1), (2, 3)])
        pa = [h.params_array(x) for x in (params, sp, params[:6], sp[:2], params)]
        outs = [np.zeros(n, RESULT_DTYPE) for n in (len(pairs), len(street), 6, 2, len(pairs))]
        bufs = [ListBuffers(len(pairs), 1024, MEM_HOST, MATCH_LISTS), ListBuffers(len(street), 1024, MEM_HOST),
                ListBuffers(6, 1024, MEM_HOST), ListBuffers(2, 1024, MEM_HOST),
                ListBuffers(len(pairs), 1024, MEM_DEVICE, device=h.cfg.device)]
        h.match_descriptors_enqueue_each_raw(d_host, len(pairs), pa[0], MEM_HOST, outs[0], bufs[0])
        h.register_batch_enqueue_mixed_raw(p_arr, len(street), pa[1], MEM_HOST, outs[1], bufs[1])
        h.register_features_enqueue_each_raw(f_arr, 6, pa[2], MEM_HOST, outs[2], bufs[2])
        h.register_cached_enqueue_mixed_raw(s_arr, 2, pa[3], outs[3], bufs[3])
        h.register_descriptors_enqueue_each_raw(d_dev, len(pairs), pa[4], MEM_DEVICE, outs[4], bufs[4])
        h.register_batch_flush()
        got = [_flat(o, b) for o, b in zip(outs, bufs)]
        want = []
        for k, fn in enumerate((lambda lb: h.match_descriptors_each(pairs, params, buffers=lb),
                                lambda lb: h.register_batch_mixed(street, sp, buffers=lb),
                                lambda lb: h.register_features_each(feats, params[:6], buffers=lb),
                                lambda lb: h.register_cached_mixed([(0, 1), (2, 3)], sp[:2], buffers=lb),
                                lambda lb: h.register_descriptors_each(pairs, params, buffers=lb))):
            lb = ListBuffers(len(outs[k]), 1024, MEM_HOST, *((MATCH_LISTS,) if k == 0 else ()))
            want.append(_flat(fn(lb)[0], lb))
        for k in range(5):
            assert got[k] == want[k], k


@pytest.mark.gpu
def test_register_lists_solve_again_to_the_same_records():
    pairs, params = _mix(np.random.default_rng(12))
    with make_handle(4, max_batch_slots=4, max_voxel_points=V_SMALL, max_corr=1024) as h:
        dev, keep = _device_pairs(pairs)
        lb = ListBuffers(len(pairs), 1024, MEM_DEVICE, device=h.cfg.device)
        recs, lists = h.register_descriptors_each(dev, params, MEM_DEVICE, buffers=lb)
        sm, tm = lb.arrays["src_matched4"], lb.arrays["tgt_matched4"]
        sets = [(sm[i].data_ptr(), tm[i].data_ptr(), int(recs[i]["n_corr"])) for i in range(len(pairs))]
        again, _ = h.solve_batch_each(sets, params, MEM_DEVICE)
        for i in range(len(pairs)):
            if recs[i]["status"] == 2:
                continue
            for k in ("valid", "status", "n_corr", "n_edges", "max_core", "clique_size", "gnc_iters", "n_rot_inliers", "n_final_inliers"):
                assert again[i][k] == recs[i][k], (i, k, again[i][k], recs[i][k])
            assert np.asarray(again[i]["T"]).tobytes() == np.asarray(recs[i]["T"]).tobytes(), i


@pytest.mark.gpu
def test_a_lane_soiled_by_a_512_float_wave_gives_a_fresh_handles_output():
    rng = np.random.default_rng(13)
    big = [_pair(_scene(rng, V_SMALL, V_SMALL, 512)) for _ in range(4)]
    small = [_pair(_scene(rng, ns, nt, dim), stride) for (dim, stride), (ns, nt) in
             (((7, 7), (100, 90)), ((33, 40), (300, 280)), ((65, 65), (129, 64)), ((2, 3), (50, 60)))]
    params = [make_params(seed=i) for i in range(4)]
    cap = 1024

    def run(h):
        lb = sentinel_lists(ListBuffers(4, cap, MEM_HOST, MATCH_LISTS))
        recs, _ = h.match_descriptors_each(small, params, buffers=lb)
        return recs, lb

    with make_handle(1, max_batch_slots=4, max_voxel_points=V_SMALL, max_corr=cap) as fresh:
        want, wlb = run(fresh)
    with make_handle(1, max_batch_slots=4, max_voxel_points=V_SMALL, max_corr=cap) as h:
        h.register_descriptors_each(big, params)
        got, glb = run(h)
    assert got.tobytes() == want.tobytes()
    for name in MATCH_LISTS:
        assert glb.arrays[name].tobytes() == wlb.arrays[name].tobytes(), name
        for i in range(4):   # every entry past a pair's live count keeps its sentinel
            assert (glb.arrays[name][i][got[i]["n_corr"]:].view(np.uint8) == 0xA5).all(), (name, i)


@pytest.mark.gpu
def test_a_rejected_call_writes_and_queues_nothing(h1):
    lib = h1.lib
    rng = np.random.default_rng(14)
    pairs, params = _mix(rng)
    good, keep_good = h1.descriptor_array(pairs)
    good_params = h1.params_array(params)
    want, _ = h1.match_descriptors_each(pairs, params)
    s, sd, t, td, dim = _pair(_scene(rng, 100, 90, 16), 20)
    _, dv = device_copies([s, sd, t, td])
    ok = DescriptorPair(s.ctypes.data, sd.ctypes.data, t.ctypes.data, td.ctypes.data, len(s), len(t), 16, 20)
    okd = DescriptorPair(dv[0].data_ptr(), dv[1].data_ptr(), dv[2].data_ptr(), dv[3].data_ptr(), len(s), len(t), 16, 20)

    def edit(base, **kw):
        d = DescriptorPair.from_buffer_copy(base)
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    def call(entries, kind=MEM_HOST, ps=None):
        arr = (DescriptorPair * len(entries))(*entries)
        out, lb = sentinel(len(entries), RESULT_DTYPE), sentinel_lists(ListBuffers(len(entries), 64, MEM_HOST, MATCH_LISTS))
        st = lib.qb200_match_descriptors_enqueue_each(h1.h, arr, len(entries), h1.params_array(ps or [params[0]] * len(entries)), kind,
                                                      capi._ptr(out), C.byref(lb.descriptor()))
        return st, out, lb

    cases = {
        "dim 0": (lambda: call([ok, edit(ok, dim=0), ok]), -1, "descriptor pair 1"),
        "dim 513": (lambda: call([ok, ok, edit(ok, dim=513, stride=513)]), -1, "descriptor pair 2"),
        "stride < dim": (lambda: call([edit(ok, stride=15), ok, ok]), -1, "descriptor pair 0"),
        "null descriptors": (lambda: call([ok, edit(ok, tgt_desc=None), ok]), -1, "descriptor pair 1"),
        "null keypoints": (lambda: call([ok, ok, edit(ok, src=None)]), -1, "descriptor pair 2"),
        "misaligned device descriptors": (lambda: call([okd, edit(okd, src_desc=dv[1].data_ptr() + 2), okd], MEM_DEVICE), -1,
                                          "descriptor pair 1"),
        "host memory as device kind": (lambda: call([okd, ok, okd], MEM_DEVICE), -1, "descriptor pair 1"),
        "crosscheck off": (lambda: call([ok] * 3, ps=[params[0], params[1], make_params(use_crosscheck=0)]), -4, "entry 2"),
    }
    for name, (fn, code, names) in cases.items():
        out1 = np.zeros(len(pairs), RESULT_DTYPE)
        assert lib.qb200_match_descriptors_enqueue_each(h1.h, good, len(pairs), good_params, MEM_HOST, capi._ptr(out1), None) == 0
        st, out, lb = fn()
        err = lib.qb200_last_error(h1.h).decode()
        assert st == code, (name, st, err)
        assert names in err, (name, err)
        h1.register_batch_flush()
        assert (out.view(np.uint8) == 0xA5).all() and all((a.view(np.uint8) == 0xA5).all() for a in lb.arrays.values()), name
        assert out1.tobytes() == want.tobytes(), name
