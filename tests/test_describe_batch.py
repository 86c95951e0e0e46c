"""The front end in batches: qb200_describe_batch_each and qb200_describe_batch_enqueue_each.
Every scan's keypoints, normals and FPFH-33 rows are byte-identical to a cache write of that scan alone read back with
qb200_cache_read, and to qb200_voxelize + qb200_compute_fpfh, for host and device scans and outputs on one lane and on four; the
described features of street pairs register like the raw pairs; refused, empty and clipped scans write exactly what the header says;
a rejected call writes and queues nothing; and describe calls share one stream with every other batch kind."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import (FEATURE_ARRAYS, LIST_LAYOUT, MEM_DEVICE, MEM_HOST, RESULT_DTYPE, SET_LISTS, FeatureOut, ListBuffers)
from support import P4, ROOT, _host, device_copies, host_lists, make_handle, make_params, sentinel

NEW = ("qb200_describe_batch_each", "qb200_describe_batch_enqueue_each")
OK, CAPACITY, OVERFLOW = 0, 3, -5


# ---- CPU: the POD, the header, the symbols -----------------------------------------------------------------------------------------
def test_feature_out_mirror_matches_the_c_layout(tmp_path):
    """sizeof and every offsetof of qb200_feature_out from a C compiler (the header compiles as C11), against the ctypes mirror."""
    body = '  printf("size %zu\\n", sizeof(qb200_feature_out));\n' + "".join(
        f'  printf("{f} %zu\\n", offsetof(qb200_feature_out, {f}));\n' for f, _ in FeatureOut._fields_)
    (tmp_path / "pod.c").write_text('#include <stddef.h>\n#include <stdio.h>\n#include "quatro_b200.h"\nint main(void) {\n' + body +
                                    "  return 0;\n}\n")
    r = subprocess.run(["/usr/bin/gcc", "-std=c11", "-Wall", "-Werror", "-pedantic", f"-I{ROOT / 'include'}", str(tmp_path / "pod.c"), "-o",
                        str(tmp_path / "pod")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    probe = dict(ln.split() for ln in subprocess.run([str(tmp_path / "pod")], capture_output=True, text=True, check=True).stdout.splitlines())
    assert C.sizeof(FeatureOut) == int(probe["size"]) == 48
    for f, _ in FeatureOut._fields_:
        assert getattr(FeatureOut, f).offset == int(probe[f]), f


def test_library_exports_the_describe_calls():
    lib = capi.load_library()
    want = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int32), C.c_int32, C.POINTER(capi.Params), C.c_int32, C.POINTER(FeatureOut)]
    for n in NEW:
        assert n in capi.EXPORTED_SYMBOLS and hasattr(lib, n)
        assert getattr(lib, n).argtypes == want and getattr(lib, n).restype == C.c_int32
    assert lib.qb200_describe_batch_each(None, None, None, 0, None, MEM_HOST, None) == -1
    assert lib.qb200_describe_batch_enqueue_each(None, None, None, 0, None, MEM_HOST, None) == -1


# ---- configurations ----------------------------------------------------------------------------------------------------------------
SLOTS, RAW_CAP = 2, 65536        # a describe wave holds 2 * SLOTS = 4 scans
CFG = dict(max_batch_slots=SLOTS, max_raw_points=RAW_CAP)
STREET = make_params()
DENSE = make_params(voxel_size=0.22, use_tuple_test=0)
COARSE = make_params(voxel_size=0.4, grid_cell=0.4, skip_flagged=0, seed=14)
WIDE = make_params(voxel_size=0.25, normal_radius=0.6, fpfh_radius=0.9, grid_cell=1.0)
INDOOR = make_params(voxel_size=0.08, normal_radius=0.16, fpfh_radius=0.24, noise_bound=0.05, cote_noise_bound=0.05)


def _bytes(per_scan):
    """per scan the bytes of (vox4, normals4, desc33), device tensors read back"""
    out = []
    for row in per_scan:
        out.append(tuple(None if a is None else (a.tobytes() if isinstance(a, np.ndarray) else a.cpu().numpy().tobytes()) for a in row))
    return out


def _cache_ref(h, scans, params):
    """per scan: (vox, normals, desc) bytes of a cache write of that scan alone read back, and its count"""
    h.cache_reserve(len(scans))
    out = []
    for i, (s, p) in enumerate(zip(scans, params)):
        h.cache_scans_each([s], [i], [p])
        v, n, d = h.cache_read(i)
        out.append(((v.tobytes(), n.tobytes(), d.tobytes()), len(v)))
    return out


def _stage_ref(h, scan, p):
    """qb200_voxelize + qb200_compute_fpfh with the entry's voxel and lattice fields"""
    vox, st = h.voxelize(scan, p.voxel_size, p.skip_flagged, cap=h.cfg.max_voxel_points)
    assert st == 0
    cell = p.grid_cell if p.grid_cell > 0 else np.float32(p.fpfh_radius) * np.float32(1.001953125)
    nrm, desc = h.compute_fpfh(vox, p.normal_radius, p.fpfh_radius, float(cell))
    return vox.tobytes(), nrm.tobytes(), desc.tobytes()


# ---- GPU fixtures ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mixed():
    """street, dense, coarse, wide and indoor scans with their entries: 11 scans, three waves"""
    street = [c for s in range(40, 45) for c in synth.outdoor_pair(s, rings=32, azimuths=900)[:2]]
    indoor = list(synth.indoor_pair(3, n_rays=60000)[:2])
    scans = street[:8] + indoor + street[8:9]
    params = [STREET, DENSE, COARSE, WIDE, STREET, DENSE, COARSE, WIDE, INDOOR, INDOOR, DENSE]
    return scans, params


@pytest.fixture(scope="module")
def h1():
    h = make_handle(1, **CFG)
    yield h
    h.close()


@pytest.fixture(scope="module")
def h4():
    h = make_handle(4, **CFG)
    yield h
    h.close()


@pytest.fixture(scope="module")
def ref(mixed):
    with make_handle(4, **CFG) as h:
        yield _cache_ref(h, *mixed)


# ---- GPU 1: every scan equals its cache write alone and the stage calls ---------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 4])
def test_describe_equals_the_cache_and_the_stage_calls(h1, h4, mixed, ref, lanes):
    h = h1 if lanes == 1 else h4
    scans, params = mixed
    counts_ref = [n for _, n in ref]
    assert min(counts_ref) > 1000 and len(set(counts_ref)) > 5
    for i in (0, 3, 8, 10):
        assert _stage_ref(h, scans[i], params[i]) == ref[i][0], i
    dev, keep = device_copies(scans)
    for kind, ss in ((MEM_HOST, scans), (MEM_DEVICE, dev)):
        for dest in (MEM_HOST, MEM_DEVICE):
            per_scan, counts, status = h.describe_batch_each(ss, params, kind, dest)
            assert (status == OK).all() and list(counts) == counts_ref, (kind, dest)
            assert _bytes(per_scan) == [r for r, _ in ref], (kind, dest)
            assert not h.stage_ms().any() and not h.kernel_ms()[0].any()   # a call that registers nothing reports zeros


# ---- GPU 2: described features register like the raw pairs ----------------------------------------------------------------------------
@pytest.mark.gpu
def test_described_features_register_like_the_raw_pairs(h1, h4):
    pairs = [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(60, 66)]
    pp = [make_params(voxel_size=(0.3, 0.25, 0.35)[i % 3], grid_cell=0.8 if i % 2 else 0.0, seed=5 + i, use_tuple_test=int(i != 4),
                      noise_bound=0.35 if i == 2 else 0.3) for i in range(len(pairs))]
    scans = [c for pr in pairs for c in pr]
    per_scan, counts, status = h4.describe_batch_each(scans, [p for p in pp for _ in (0, 1)])
    assert (status == OK).all()
    feats = [(per_scan[2 * i][0], per_scan[2 * i][2], per_scan[2 * i + 1][0], per_scan[2 * i + 1][2]) for i in range(len(pairs))]
    lb_f, lb_r = ListBuffers(len(pairs), h1.cfg.max_corr), ListBuffers(len(pairs), h1.cfg.max_corr)
    got, _ = h1.register_features_each(feats, pp, buffers=lb_f)
    want, _ = h1.register_batch_mixed(pairs, pp, buffers=lb_r)
    assert (want["status"] == OK).sum() >= len(pairs) - 1 and (want["clique_size"] > 3).all()
    assert got.tobytes() == want.tobytes()
    assert _lists(lb_f, got) == _lists(lb_r, want)


# ---- GPU 3: empty, flagged, refused and clipped scans; one more scan than a rotation ---------------------------------------------------
def _edge_batch():
    """(label, scan, entry, expected status): refused scans in the middle of the batch, between ordinary neighbours"""
    rng = np.random.default_rng(3)
    street = [c for s in range(80, 84) for c in synth.outdoor_pair(s, rings=32, azimuths=900)[:2]]
    flagged = P4(rng.uniform(-10, 10, (5000, 3)), w=-1.0)
    many = P4(rng.uniform(-40, 40, (60000, 3)))                   # ~60 k occupied voxels of 0.3 m: above max_voxel_points
    overflow = P4([[0.5, 0.5, 0.5], [65535.5, 32767.5, 0.5], [7.5, 7.5, 0.5]])   # PCL's int voxel index would overflow at leaf 1
    return [("street 0", street[0], STREET, OK), ("empty", np.zeros((0, 4), np.float32), STREET, OK), ("street 1", street[1], DENSE, OK),
            ("all flagged", flagged, STREET, OK), ("street 2", street[2], COARSE, OK), ("capacity", many, STREET, CAPACITY),
            ("street 3", street[3], STREET, OK), ("overflow", overflow, make_params(voxel_size=1.0, normal_radius=1.0, fpfh_radius=1.5), OVERFLOW),
            ("street 4", street[4], WIDE, OK), ("flagged kept", flagged, COARSE, OK)] + \
        [(f"street {5 + k}", street[5 + k % 3], (STREET, DENSE, WIDE)[k % 3], OK) for k in range(7)]


def _lists(buffers, records):
    return [{k: v.tobytes() for k, v in d.items()} for d in host_lists(buffers.trimmed(records))]


@pytest.mark.gpu
@pytest.mark.parametrize("cap", [16384, 3000])
def test_edge_scans_write_exactly_their_entries(h4, cap):
    batch = _edge_batch()
    n = len(batch)
    assert n == 2 * SLOTS * 4 + 1                                  # one more scan than a full rotation of waves over the lanes
    scans, params = [b[1] for b in batch], [b[2] for b in batch]
    with make_handle(4, **CFG) as r:
        ref = _cache_ref(r, scans, params)
    dev, keep = device_copies(scans)
    for kind, ss in ((MEM_HOST, scans), (MEM_DEVICE, dev)):
        for dest in (MEM_HOST, MEM_DEVICE):
            arrays = {k: sentinel((n + 1, cap, w), kind=dest) for k, w in FEATURE_ARRAYS.items()}
            counts, status = np.full(n, -7, np.int32), np.full(n, -7, np.int32)
            out = h4.feature_out(cap, dest, arrays, counts, status)
            ptrs, cnts, keep_h = capi._scan_arrays(ss, kind)
            assert h4.lib.qb200_describe_batch_each(h4.h, ptrs, cnts, n, h4.params_array(params), kind, C.byref(out)) == 0
            got = {k: _host(a) for k, a in arrays.items()}
            for k, a in got.items():
                assert (a[n].view(np.uint8) == 0xA5).all(), (kind, dest, k)          # nothing past the last scan's cap
            for i, (label, _, _, st) in enumerate(batch):
                assert status[i] == st, (label, status[i])
                (rv, rn, rd), rc = ref[i]
                want_n = rc if st == OK else 0
                assert counts[i] == want_n, (label, counts[i], want_n)
                if label in ("empty", "all flagged"):
                    assert want_n == 0
                m = min(want_n, cap)
                for k, rb, w in (("vox4", rv, 4), ("normals4", rn, 4), ("desc33", rd, 33)):
                    assert got[k][i, :m].tobytes() == rb[:m * w * 4], (label, k, kind, dest)
                    assert (got[k][i, m:].view(np.uint8) == 0xA5).all(), (label, k, kind, dest)
            if cap == 3000:
                assert (counts > cap).sum() >= 8                      # the full count of a clipped scan is reported


# ---- GPU 4: refusals -------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_rejected_call_writes_and_queues_nothing(h4, mixed, ref):
    lib = h4.lib
    scans, params = mixed
    n, cap = len(scans), 16384
    ptrs, cnts, keep = capi._scan_arrays(scans, MEM_HOST)
    pa = h4.params_array(params)

    def call(dest=MEM_HOST, cap_=cap, arrays=None, counts=True, ps=None, shift=None, kind_as=None):
        arrays = arrays if arrays is not None else {k: sentinel((n + 1, max(cap_, 1), w), kind=dest) for k, w in FEATURE_ARRAYS.items()}
        c, s = np.full(n, -7, np.int32), np.full(n, -7, np.int32)
        out = h4.feature_out(cap_, dest, arrays, c, s)
        if kind_as is not None:
            out.kind = kind_as
        if not counts:
            out.counts = None
        for k, d in (shift or {}).items():
            setattr(out, k, getattr(out, k) + d)
        st = lib.qb200_describe_batch_enqueue_each(h4.h, ptrs, cnts, n, ps if ps is not None else pa, MEM_HOST, C.byref(out))
        return st, arrays, c, s

    dev = {k: sentinel((n + 1, cap, w), kind=MEM_DEVICE) for k, w in FEATURE_ARRAYS.items()}
    bad_ps = [capi.Params.from_buffer_copy(p) for p in params]
    bad_ps[4].fpfh_radius = 0.2                                    # below its normal radius
    cases = {
        "misaligned device vox4": (lambda: call(MEM_DEVICE, arrays=dev, shift={"vox4": 4}), "vox4"),
        "misaligned device normals4": (lambda: call(MEM_DEVICE, arrays=dev, shift={"normals4": 8}), "normals4"),
        "misaligned device desc33": (lambda: call(MEM_DEVICE, arrays=dev, shift={"desc33": 2}), "desc33"),
        "host memory as device kind": (lambda: call(MEM_HOST, kind_as=MEM_DEVICE), "vox4"),
        "null counts": (lambda: call(counts=False), "counts"),
        "cap_per_scan 0": (lambda: call(cap_=0), "cap_per_scan"),
        "bad params entry": (lambda: call(ps=h4.params_array(bad_ps)), "entry 4"),
    }
    for name, (fn, culprit) in cases.items():
        # a batch queued before the refused call completes on the flush
        arrays0 = {k: sentinel((n + 1, cap, w), kind=MEM_HOST) for k, w in FEATURE_ARRAYS.items()}
        c0, s0 = np.zeros(n, np.int32), np.zeros(n, np.int32)
        out0 = h4.feature_out(cap, MEM_HOST, arrays0, c0, s0)
        assert lib.qb200_describe_batch_enqueue_each(h4.h, ptrs, cnts, n, pa, MEM_HOST, C.byref(out0)) == 0
        st, arrays, c, s = fn()
        err = lib.qb200_last_error(h4.h).decode()
        assert st == -1, (name, st, err)
        assert culprit in err, (name, err)
        h4.register_batch_flush()
        assert (c == -7).all() and (s == -7).all(), name
        for k, a in arrays.items():
            assert (_host(a).view(np.uint8) == 0xA5).all(), (name, k)
        assert list(c0) == [r[1] for r in ref] and (s0 == OK).all(), name
        assert [tuple(arrays0[k][i, :c0[i]].tobytes() for k in FEATURE_ARRAYS) for i in range(n)] == [r[0] for r in ref], name


# ---- GPU 5: one stream of describe, raw, cached, feature and set batches and a cache write --------------------------------------------
@pytest.mark.gpu
def test_one_stream_of_describe_and_every_other_batch(mixed, ref):
    scans, params = mixed
    n = len(scans)
    pairs = [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(90, 95)]
    pp = [make_params(seed=3 + i, voxel_size=(0.3, 0.25)[i % 2]) for i in range(len(pairs))]
    sets = [tuple(a[:L] for a in synth.matched_pairs(700 + i, L, inlier_ratio=0.35, noise=0.03)[:2]) for i, L in enumerate([40, 300, 1200])]
    sp = [make_params()] * len(sets)
    slot_pairs = [(0, 1), (2, 3), (4, 5)]
    cache_scans = [c for pr in pairs[:3] for c in pr]
    cache_pp = [p for p in pp[:3] for _ in (0, 1)]
    with make_handle(4, **CFG) as h:
        h.cache_reserve(6)
        # the features of the first two street pairs, described beforehand
        d, _, _ = h.describe_batch_each([c for pr in pairs[:2] for c in pr], [p for p in pp[:2] for _ in (0, 1)])
        feats = [(d[0][0], d[0][2], d[1][0], d[1][2]), (d[2][0], d[2][2], d[3][0], d[3][2])]
        dev, keep = device_copies(scans)
        cap = h.cfg.max_voxel_points

        def run(queued):
            outs = {}
            a_host, a_dev = h.feature_buffers(n, cap, MEM_HOST), h.feature_buffers(n, cap, MEM_DEVICE)
            cnt = [np.zeros(n, np.int32) for _ in range(4)]
            o_host, o_dev = h.feature_out(cap, MEM_HOST, a_host, cnt[0], cnt[1]), h.feature_out(cap, MEM_DEVICE, a_dev, cnt[2], cnt[3])
            recs = [np.zeros(k, RESULT_DTYPE) for k in (len(pairs), len(slot_pairs), len(feats), len(sets))]
            bufs = [ListBuffers(len(r), h.cfg.max_corr, MEM_HOST, SET_LISTS if k == 3 else tuple(LIST_LAYOUT)) for k, r in enumerate(recs)]
            sh, ch, kh = capi._scan_arrays(scans, MEM_HOST)
            sd, cd, _ = capi._scan_arrays(dev, MEM_DEVICE)
            wp, wc, wk = capi._scan_arrays(cache_scans, MEM_HOST)
            ids = (C.c_int32 * 6)(*range(6))
            pair_arr, kp = h.pair_array(pairs)
            feat_arr, kf = h.feature_array(feats)
            set_arr, ks = h._set_array(sets, MEM_HOST)
            slot_arr = capi._slot_array(slot_pairs)
            pa = [h.params_array(x) for x in (params, pp, cache_pp, pp[:3], pp[:2], sp)]
            steps = [
                lambda: h.describe_batch_enqueue_each_raw(sh, ch, n, pa[0], MEM_HOST, o_host),
                lambda: h.register_batch_enqueue_mixed_raw(pair_arr, len(pairs), pa[1], MEM_HOST, recs[0], bufs[0]),
                lambda: h.cache_scans_enqueue_each_raw(wp, wc, ids, 6, pa[2], MEM_HOST),
                lambda: h.register_cached_enqueue_mixed_raw(slot_arr, len(slot_pairs), pa[3], recs[1], bufs[1]),
                lambda: h.register_features_enqueue_each_raw(feat_arr, len(feats), pa[4], MEM_HOST, recs[2], bufs[2]),
                lambda: h.solve_batch_enqueue_each_raw(set_arr, len(sets), pa[5], MEM_HOST, recs[3], bufs[3]),
                lambda: h.describe_batch_enqueue_each_raw(sd, cd, n, pa[0], MEM_DEVICE, o_dev),
            ]
            for step in steps:
                step()
                if not queued:
                    h.register_batch_flush()
            h.register_batch_flush()
            outs["records"] = [r.tobytes() for r in recs]
            outs["lists"] = [_lists(b, r) for b, r in zip(bufs, recs)]
            outs["counts"] = [c.tobytes() for c in cnt]
            outs["described"] = []
            for j, arr in enumerate((a_host, a_dev)):
                arr = {k: _host(a) for k, a in arr.items()}
                outs["described"].append([tuple(arr[k][i, :cnt[2 * j][i]].tobytes() for k in FEATURE_ARRAYS) for i in range(n)])
            return outs

        got, want = run(True), run(False)
        assert got == want
        assert got["described"][0] == got["described"][1] == [r for r, _ in ref]
        recs = np.frombuffer(got["records"][0], RESULT_DTYPE)
        assert (recs["status"] == OK).sum() >= len(pairs) - 1
