"""The voxel filter in batches: qb200_voxelize_batch_each and qb200_voxelize_batch_enqueue_each.
Every scan's count, status and centroids are byte-identical to qb200_voxelize of that scan alone, for host and device scans and outputs
on one lane and on four: QB200_CAPACITY_EXCEEDED scans give their first max_voxel_points centroids and QB200_ERR_VOXEL_OVERFLOW scans
PCL's pass-through of their kept points; clipped, empty and skipped scans write exactly what the header says; the centroids feed
describe-points as the describe call's own do; a voxelize wave runs no FPFH; a rejected call writes and queues nothing; and voxelize
calls share one stream with every other batch kind."""
import ctypes as C

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import (MEM_DEVICE, MEM_HOST, PREPROCESS_ARRAYS, RESULT_DTYPE, Handle, ListBuffers, default_patchwork_params,
                              default_segment_params)
import support
from support import P4, _host, device_copies, make_handle, sentinel

NEW = ("qb200_voxelize_batch_each", "qb200_voxelize_batch_enqueue_each")
OK, CAPACITY, OVERFLOW = 0, 3, -5
KINDS = [(k, d) for k in (MEM_HOST, MEM_DEVICE) for d in (MEM_HOST, MEM_DEVICE)]


# ---- CPU: the symbols --------------------------------------------------------------------------------------------------------------
def test_library_exports_the_voxelize_calls():
    lib = capi.load_library()
    want = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int32), C.c_int32, C.POINTER(capi.Params), C.c_int32, C.POINTER(capi.FeatureOut)]
    for n in NEW:
        assert n in capi.EXPORTED_SYMBOLS and hasattr(lib, n)
        assert getattr(lib, n).argtypes == want and getattr(lib, n).restype == C.c_int32
    assert lib.qb200_voxelize_batch_each(None, None, None, 0, None, MEM_HOST, None) == -1
    assert lib.qb200_voxelize_batch_enqueue_each(None, None, None, 0, None, MEM_HOST, None) == -1


# ---- configurations ----------------------------------------------------------------------------------------------------------------
def make_params(**kw):
    """support.make_params keeping default_params()'s rot_noise_bound of 0, the latch: the register calls here run with it"""
    return support.make_params(rot_noise_bound=0.0, **kw)


SLOTS, RAW_CAP = 2, 65536        # a voxelize wave holds 2 * SLOTS = 4 scans
CFG = dict(max_batch_slots=SLOTS, max_raw_points=RAW_CAP)
STREET = make_params()
DENSE = make_params(voxel_size=0.22)
COARSE = make_params(voxel_size=0.4, skip_flagged=0)
INDOOR = make_params(voxel_size=0.08)
FINE_KEEP = make_params(voxel_size=0.25, skip_flagged=0)


def _ref(h, scans, params):
    """per scan: (centroid bytes, count, status) of qb200_voxelize of that scan alone with unlimited room"""
    out = []
    for s, p in zip(scans, params):
        v, st = h.voxelize(s, p.voxel_size, p.skip_flagged, cap=max(1, len(s)))
        out.append((v.tobytes(), len(v), st))
    return out


# ---- GPU fixtures ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mixed():
    """street, dense, coarse and indoor scans with varied leaves and both skip_flagged values: 11 scans, three waves"""
    street = [c for s in range(40, 45) for c in synth.outdoor_pair(s, rings=32, azimuths=900)[:2]]
    indoor = list(synth.indoor_pair(3, n_rays=60000)[:2])
    scans = street[:8] + indoor + street[8:9]
    params = [STREET, DENSE, COARSE, FINE_KEEP, STREET, DENSE, COARSE, FINE_KEEP, INDOOR, make_params(voxel_size=0.1, skip_flagged=0),
              DENSE]
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
    with make_handle(1, **CFG) as h:
        yield _ref(h, *mixed)


# ---- GPU 1: every scan equals qb200_voxelize, the oracle and the describe call's centroids ------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 4])
def test_voxelize_equals_the_stage_call_and_the_oracle(h1, h4, mixed, ref, oracle, lanes):
    h = h1 if lanes == 1 else h4
    scans, params = mixed
    assert all(st == OK for _, _, st in ref) and min(n for _, n, _ in ref) > 1000 and len({n for _, n, _ in ref}) > 5
    if lanes == 1:
        for i, (s, p) in enumerate(zip(scans, params)):
            v, st = oracle.voxelize(s, p.voxel_size, p.skip_flagged, cap=max(1, len(s)))
            assert st == OK and v.tobytes() == ref[i][0], i
    described, dcounts, dstatus = h.describe_batch_each(scans, params)
    assert (dstatus == OK).all()
    assert [d[0].tobytes() for d in described] == [r[0] for r in ref]
    dev, keep = device_copies(scans)
    for kind, dest in KINDS:
        per_scan, counts, status = h.voxelize_batch_each(dev if kind == MEM_DEVICE else scans, params, kind, dest)
        assert list(counts) == [n for _, n, _ in ref] and list(status) == [st for _, _, st in ref], (kind, dest)
        assert [_host(v).tobytes() for v in per_scan] == [r[0] for r in ref], (kind, dest)
        assert not h.stage_ms().any() and not h.kernel_ms()[0].any()   # a call that registers nothing reports zeros


# ---- GPU 2: empty, skipped, non-finite, capacity and pass-through scans; one more scan than a rotation -------------------------------
def _pass_through(rng, n, skip_flagged):
    """n points in a 10 m cube plus two far corners (PCL's int voxel index overflows at leaf 1), with NaN, inf and w < 0 records
    interleaved"""
    xyz = rng.uniform(0, 10, (n, 3))
    xyz[n // 3] = (65535.5, 32767.5, 0.5)
    xyz[2 * n // 3] = (0.5, 0.5, 0.5)
    pts = P4(xyz)
    pts[::7, 0] = np.nan
    pts[3::11, 1] = np.inf
    pts[5::13, 2] = -np.inf
    pts[2::5, 3] = -1.0
    pts[4::9, 3] = rng.uniform(0, 2, len(pts[4::9]))               # verbatim w values
    pts[n // 3, :3], pts[2 * n // 3, :3] = (65535.5, 32767.5, 0.5), (0.5, 0.5, 0.5)
    pts[n // 3, 3] = pts[2 * n // 3, 3] = 1.0
    return pts, make_params(voxel_size=1.0, skip_flagged=skip_flagged)


def _edge_batch():
    """(label, scan, entry): scans refused by the filter in the middle of the batch, between ordinary neighbours"""
    rng = np.random.default_rng(5)
    street = [c for s in range(80, 83) for c in synth.outdoor_pair(s, rings=32, azimuths=900)[:2]]
    flagged = P4(rng.uniform(-10, 10, (5000, 3)), w=-1.0)
    many = P4(rng.uniform(-40, 40, (60000, 3)))                   # ~60 k occupied voxels of 0.3 m: above max_voxel_points
    nonfinite = P4(rng.uniform(-20, 20, (8000, 3)))
    nonfinite[::3, 0] = np.nan
    nonfinite[1::5, 2] = np.inf
    big_pass, p_big = _pass_through(rng, 34000, 1)                 # about 20 k kept points: above max_voxel_points and 3000
    small_pass, p_small = _pass_through(rng, 2500, 0)
    return [("street 0", street[0], STREET), ("empty", np.zeros((0, 4), np.float32), STREET), ("street 1", street[1], DENSE),
            ("all flagged, skipped", flagged, STREET), ("all flagged, kept", flagged, COARSE), ("non-finite", nonfinite, DENSE),
            ("capacity", many, STREET), ("street 2", street[2], COARSE), ("pass-through, skip 1", big_pass, p_big),
            ("street 3", street[3], FINE_KEEP), ("pass-through, skip 0", small_pass, p_small), ("street 4", street[4], STREET)] + \
        [(f"street {5 + k}", street[(5 + k) % 6], (STREET, DENSE, COARSE)[k % 3]) for k in range(5)]


@pytest.fixture(scope="module")
def edge():
    batch = _edge_batch()
    scans, params = [b[1] for b in batch], [b[2] for b in batch]
    with make_handle(1, **CFG) as r:
        want = _ref(r, scans, params)
        V = r.cfg.max_voxel_points
    st = {b[0]: w[2] for b, w in zip(batch, want)}
    n_of = {b[0]: w[1] for b, w in zip(batch, want)}
    assert st["capacity"] == CAPACITY and n_of["capacity"] == V
    assert st["pass-through, skip 1"] == st["pass-through, skip 0"] == OVERFLOW
    assert n_of["pass-through, skip 1"] > V and 0 < n_of["pass-through, skip 0"] < 3000
    assert n_of["empty"] == n_of["all flagged, skipped"] == 0 and n_of["all flagged, kept"] > 0 and n_of["non-finite"] > 0
    assert sum(s == OK for s in st.values()) == len(batch) - 3
    return batch, scans, params, want


@pytest.mark.gpu
@pytest.mark.parametrize("cap", ["max_voxel_points", 3000, "above"])
def test_edge_scans_write_exactly_their_entries(h4, edge, cap):
    batch, scans, params, want = edge
    n = len(batch)
    assert n == 2 * SLOTS * 4 + 1                                  # one more scan than a full rotation of waves over the lanes
    V = h4.cfg.max_voxel_points
    cap = {"max_voxel_points": V, "above": V + 8192}.get(cap, cap)
    dev, keep = device_copies(scans)
    for kind, dest in KINDS:
        arrays = {"vox4": sentinel((n + 1, cap, 4), kind=dest)}
        counts, status = np.full(n, -7, np.int32), np.full(n, -7, np.int32)
        out = h4.feature_out(cap, dest, arrays, counts, status)
        ptrs, cnts, keep_h = capi._scan_arrays(dev if kind == MEM_DEVICE else scans, kind)
        assert h4.lib.qb200_voxelize_batch_each(h4.h, ptrs, cnts, n, h4.params_array(params), kind, C.byref(out)) == 0
        got = _host(arrays["vox4"])
        assert (got[n].view(np.uint8) == 0xA5).all(), (kind, dest)          # nothing past the last scan's cap
        for i, (label, _, _) in enumerate(batch):
            rb, rc, rs = want[i]
            assert (counts[i], status[i]) == (rc, rs), (label, counts[i], status[i], rc, rs)
            m = min(rc, cap)
            assert got[i, :m].tobytes() == rb[:m * 16], (label, kind, dest, cap)
            assert (got[i, m:].view(np.uint8) == 0xA5).all(), (label, kind, dest, cap)
        if cap == 3000:
            assert (counts > cap).sum() >= 8                          # the full count of a clipped scan is reported


# ---- GPU 3: counts and status alone ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_counts_only_call(h4, edge):
    batch, scans, params, want = edge
    dev, keep = device_copies(scans)
    for kind, dest in KINDS:
        per_scan, counts, status = h4.voxelize_batch_each(dev if kind == MEM_DEVICE else scans, params, kind, dest, arrays={})
        assert all(v is None for v in per_scan)
        assert list(counts) == [w[1] for w in want] and list(status) == [w[2] for w in want], (kind, dest)


# ---- GPU 4: the device chains --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_voxelize_then_describe_points_equals_describe(h4, mixed):
    scans, params = mixed
    wide = [make_params(voxel_size=p.voxel_size, skip_flagged=p.skip_flagged, normal_radius=2.5 * p.voxel_size,
                        fpfh_radius=(4.0 if i % 2 else 3.0) * p.voxel_size, grid_cell=0.0 if i % 3 else 4.5 * p.voxel_size)
            for i, p in enumerate(params)]
    dev, keep = device_copies(scans)
    vox, counts, status = h4.voxelize_batch_each(dev, wide, MEM_DEVICE, MEM_DEVICE)
    assert (status == OK).all()
    clouds = [(v.data_ptr(), int(c)) for v, c in zip(vox, counts)]
    pts, pc, ps = h4.describe_points_each(clouds, wide, MEM_DEVICE, MEM_HOST)
    want, wc, ws = h4.describe_batch_each(dev, wide, MEM_DEVICE, MEM_HOST)
    assert list(pc) == list(wc) == list(counts) and (ps == OK).all() and (ws == OK).all()
    for i in range(len(scans)):
        assert _host(vox[i]).tobytes() == want[i][0].tobytes(), i
        assert pts[i][0].tobytes() == want[i][1].tobytes() and pts[i][1].tobytes() == want[i][2].tobytes(), i


@pytest.mark.gpu
def test_preprocess_then_voxelize_on_the_device():
    scans = [c for s in range(20, 23) for c in synth.outdoor_pair(s)[:2]]   # 64-ring scans, as the segmentation's range image expects
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("QB200_LANES", "4")
        h = Handle(max_batch_slots=SLOTS)
    with h:
        import torch
        sp = default_segment_params()
        cap = max([len(s) for s in scans] + [sp.n_scan * sp.horizon_scan])
        arrays = {k: torch.zeros((len(scans), cap, 4), dtype=torch.float32, device="cuda") for k in PREPROCESS_ARRAYS}
        _, pcounts, pstatus = h.preprocess_batch(scans, default_patchwork_params(), sp, cap=cap, dest=MEM_DEVICE, arrays=arrays)
        assert (pstatus == OK).all() and pcounts[:, 2].sum() > 0
        valid = [arrays["valid4"][i, :pcounts[i, 2]] for i in range(len(scans))]   # left on the device
        params = [make_params(voxel_size=(0.3, 0.2, 0.5)[i % 3], skip_flagged=i % 2) for i in range(len(scans))]
        vox, counts, status = h.voxelize_batch_each([(v.data_ptr(), len(v)) for v in valid], params, MEM_DEVICE, MEM_HOST)
        want = _ref(h, [_host(v) for v in valid], params)
        assert list(counts) == [w[1] for w in want] and list(status) == [w[2] for w in want]
        assert [v.tobytes() for v in vox] == [w[0] for w in want]


# ---- GPU 5: no normals or FPFH in a voxelize wave ----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_voxelize_call_launches_less_than_a_describe_call(h4, mixed):
    scans, params = mixed
    h4.voxelize_batch_each(scans, params)                          # both warmed up, lanes allocated
    h4.describe_batch_each(scans, params)
    c0 = h4.launch_count()
    h4.voxelize_batch_each(scans, params)
    c1 = h4.launch_count()
    h4.describe_batch_each(scans, params)
    c2 = h4.launch_count()
    assert 0 < c1 - c0 < c2 - c1, (c1 - c0, c2 - c1)


# ---- GPU 6: refusals -------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_rejected_call_writes_and_queues_nothing(h4, mixed, ref):
    lib = h4.lib
    scans, params = mixed
    n, cap = len(scans), h4.cfg.max_voxel_points
    ptrs, cnts, keep = capi._scan_arrays(scans, MEM_HOST)
    dev, keep_d = device_copies(scans)
    pa = h4.params_array(params)

    def bad_entry(k, v):
        ps = [capi.Params.from_buffer_copy(p) for p in params]
        ps[k].voxel_size = v
        return h4.params_array(ps)

    def call(dest=MEM_HOST, cap_=cap, arrays=None, drop=None, ps=None, kind_as=None, extra=None, scan_ptrs=None, scan_n=None,
             kind=MEM_HOST):
        arrays = arrays if arrays is not None else {"vox4": sentinel((n + 1, max(cap_, 1), 4), kind=dest)}
        c, s = np.full(n, -7, np.int32), np.full(n, -7, np.int32)
        out = h4.feature_out(cap_, dest, arrays, c, s)
        if kind_as is not None:
            out.kind = kind_as
        if drop:
            setattr(out, drop, None)
        for k, v in (extra or {}).items():
            setattr(out, k, v)
        st = lib.qb200_voxelize_batch_enqueue_each(h4.h, scan_ptrs or ptrs, scan_n or cnts, n, ps if ps is not None else pa, kind,
                                                   C.byref(out))
        return st, arrays, c, s

    dev_out = {"vox4": sentinel((n + 1, cap, 4), kind=MEM_DEVICE)}
    spare = np.zeros((n, cap, 33), np.float32)
    too_many = (C.c_int32 * n)(*[len(s) for s in scans])
    too_many[6] = RAW_CAP + 1
    host_as_dev = capi._scan_arrays(scans, MEM_HOST)
    cases = {
        "voxel_size 0": (lambda: call(ps=bad_entry(3, 0.0)), "entry 3"),
        "voxel_size -1": (lambda: call(ps=bad_entry(5, -1.0)), "entry 5"),
        "voxel_size NaN": (lambda: call(ps=bad_entry(9, float("nan"))), "entry 9"),
        "normals4": (lambda: call(extra={"normals4": spare.ctypes.data}), "normals4"),
        "desc33": (lambda: call(extra={"desc33": spare.ctypes.data}), "desc33"),
        "cap_per_scan 0": (lambda: call(cap_=0), "cap_per_scan"),
        "null counts": (lambda: call(drop="counts"), "counts"),
        "null status": (lambda: call(drop="status"), "status"),
        "misaligned device vox4": (lambda: call(MEM_DEVICE, arrays=dev_out, extra={"vox4": dev_out["vox4"].data_ptr() + 4}), "vox4"),
        "host outputs as device kind": (lambda: call(MEM_HOST, kind_as=MEM_DEVICE), "vox4"),
        "host scans as device kind": (lambda: call(scan_ptrs=host_as_dev[0], scan_n=host_as_dev[1], kind=MEM_DEVICE), "scan 0"),
        "n_points above max_raw_points": (lambda: call(scan_n=too_many), "scan 6"),
    }
    for name, (fn, culprit) in cases.items():
        # a batch queued before the refused call completes on the flush
        arrays0 = {"vox4": sentinel((n + 1, cap, 4), kind=MEM_HOST)}
        c0, s0 = np.zeros(n, np.int32), np.zeros(n, np.int32)
        out0 = h4.feature_out(cap, MEM_HOST, arrays0, c0, s0)
        assert lib.qb200_voxelize_batch_enqueue_each(h4.h, ptrs, cnts, n, pa, MEM_HOST, C.byref(out0)) == 0
        st, arrays, c, s = fn()
        err = lib.qb200_last_error(h4.h).decode()
        assert st == -1, (name, st, err)
        assert culprit in err, (name, err)
        h4.register_batch_flush()
        assert (c == -7).all() and (s == -7).all(), name
        assert (_host(arrays["vox4"]).view(np.uint8) == 0xA5).all(), name
        assert (spare == 0).all(), name
        assert list(c0) == [r[1] for r in ref] and (s0 == OK).all(), name
        assert [arrays0["vox4"][i, :c0[i]].tobytes() for i in range(n)] == [r[0] for r in ref], name


# ---- GPU 7: one stream of voxelize, raw-pair, describe and cache-write batches ------------------------------------------------------
@pytest.mark.gpu
def test_one_stream_of_voxelize_and_every_other_batch(mixed, ref, edge):
    scans, params = mixed
    _, escans, eparams, ewant = edge
    n, ne = len(scans), len(escans)
    pairs = [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(90, 94)]
    pp = [make_params(seed=3 + i, voxel_size=(0.3, 0.25)[i % 2]) for i in range(len(pairs))]
    for p in pp:
        p.rot_noise_bound = 2 * p.noise_bound
    cache_scans = [c for pr in pairs[:2] for c in pr]
    cache_pp = [p for p in pp[:2] for _ in (0, 1)]
    with make_handle(4, **CFG) as h:
        h.cache_reserve(4)
        dev, keep = device_copies(escans)
        cap = h.cfg.max_voxel_points

        def run(queued):
            vh, vd = h.feature_buffers(n, cap, MEM_HOST, ("vox4",)), h.feature_buffers(ne, cap, MEM_DEVICE, ("vox4",))
            dh = h.feature_buffers(n, cap, MEM_HOST)
            cnt = [np.zeros(k, np.int32) for k in (n, n, ne, ne, n, n)]
            o_vh, o_vd = h.feature_out(cap, MEM_HOST, vh, cnt[0], cnt[1]), h.feature_out(cap, MEM_DEVICE, vd, cnt[2], cnt[3])
            o_dh = h.feature_out(cap, MEM_HOST, dh, cnt[4], cnt[5])
            rec = np.zeros(len(pairs), RESULT_DTYPE)
            buf = ListBuffers(len(pairs), h.cfg.max_corr, MEM_HOST)
            sh, ch, kh = capi._scan_arrays(scans, MEM_HOST)
            sd, cd, _ = capi._scan_arrays(dev, MEM_DEVICE)
            wp, wc, wk = capi._scan_arrays(cache_scans, MEM_HOST)
            ids = (C.c_int32 * 4)(*range(4))
            pair_arr, kp = h.pair_array(pairs)
            pa = [h.params_array(x) for x in (params, eparams, pp, cache_pp)]
            steps = [
                lambda: h.voxelize_batch_enqueue_each_raw(sh, ch, n, pa[0], MEM_HOST, o_vh),
                lambda: h.register_batch_enqueue_mixed_raw(pair_arr, len(pairs), pa[2], MEM_HOST, rec, buf),
                lambda: h.describe_batch_enqueue_each_raw(sh, ch, n, pa[0], MEM_HOST, o_dh),
                lambda: h.cache_scans_enqueue_each_raw(wp, wc, ids, 4, pa[3], MEM_HOST),
                lambda: h.voxelize_batch_enqueue_each_raw(sd, cd, ne, pa[1], MEM_DEVICE, o_vd),
            ]
            for step in steps:
                step()
                if not queued:
                    h.register_batch_flush()
            h.register_batch_flush()
            vd_h = _host(vd["vox4"])
            return {
                "records": rec.tobytes(),
                "counts": [c.tobytes() for c in cnt],
                "voxelized": [vh["vox4"][i, :cnt[0][i]].tobytes() for i in range(n)],
                "edge": [vd_h[i, :min(cnt[2][i], cap)].tobytes() for i in range(ne)],
                "described": [tuple(dh[k][i, :cnt[4][i]].tobytes() for k in ("vox4", "normals4", "desc33")) for i in range(n)],
                "cached": [tuple(a.tobytes() for a in h.cache_read(i)) for i in range(4)],
            }

        got, want = run(True), run(False)
        assert got == want
        assert got["voxelized"] == [r[0] for r in ref]
        assert [d[0] for d in got["described"]] == [r[0] for r in ref]
        assert got["edge"] == [w[0][:min(w[1], cap) * 16] for w in ewant]
        assert (np.frombuffer(got["records"], RESULT_DTYPE)["status"] == OK).sum() >= len(pairs) - 1
