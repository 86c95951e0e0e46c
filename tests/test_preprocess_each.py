"""qb200_preprocess_batch_each: pre-processing of a batch in which every scan has its own Patchwork and range-image parameters (lidar
model, mounting height, zone layout, neighbour mode, ...).  Every scan's outputs, counts and status must be byte-identical to
qb200_preprocess_batch on that scan alone with its own entry, and to the CPU oracle's patchwork -> segment_cloud chain, whatever the
wave, the scan's neighbours, its position or the memory kinds."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from quatro_b200 import _build, capi, synth
from quatro_b200.capi import (LIDAR_MODELS, MEM_DEVICE, MEM_HOST, PREPROCESS_ARRAYS, default_patchwork_params, default_segment_params,
                              lidar_segment_params)
from support import ROOT, same_bits

MODELS = list(LIDAR_MODELS)
SENTINEL = 0xA5


# ---- CPU ---------------------------------------------------------------------------------------------------------------------
def test_header_declares_preprocess_batch_each():
    text = (ROOT / "include" / "quatro_b200.h").read_text()
    decl = re.search(r"int qb200_preprocess_batch_each\(([^;]*)\);", text)
    assert decl, "qb200_preprocess_batch_each is not declared"
    args = " ".join(decl.group(1).split())
    assert args == ("qb200_handle* h, const float* const* scans4, const int32_t* n_points, int32_t n_scans, qb200_mem_kind kind, "
                    "const qb200_patchwork_params* pp, const qb200_segment_params* sp, const qb200_preprocess_out* out"), args
    assert "qb200_preprocess_batch_each" in capi.EXPORTED_SYMBOLS


def test_preprocess_each_fixture_compiles(tmp_path):
    """The INTEGRATION.md mixed-fleet example (device outputs into qb200_register_batch) builds against the library."""
    lib = _build.build_cuda()
    cuda = Path(_build.nvcc_path()).resolve().parent.parent
    exe = tmp_path / "preprocess_each_shim"
    cmd = ["/usr/bin/g++", "-std=c++17", "-Wall", "-Werror", f"-I{ROOT / 'include'}", f"-I{cuda / 'include'}",
           str(ROOT / "tests/fixtures/preprocess_each_shim.cpp"), f"-L{lib.parent}", "-lquatro_b200", f"-L{cuda / 'lib64'}", "-lcudart",
           f"-Wl,-rpath,{lib.parent}", f"-Wl,-rpath,{cuda / 'lib64'}", "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr


def test_preprocess_batch_each_refuses_a_null_handle():
    lib = capi.load_library()
    counts, status = np.zeros(4, np.int32), np.zeros(1, np.int32)
    out = capi.PreprocessOut(1, MEM_HOST)
    out.counts, out.status = counts.ctypes.data, status.ctypes.data
    assert lib.qb200_preprocess_batch_each(None, None, None, 0, MEM_HOST, None, None, C.byref(out)) == -1


def test_lidar_models_follow_the_reference_table():
    assert {m: LIDAR_MODELS[m][:2] for m in MODELS} == {"Velodyne-64-HDE": (64, 1800), "VLP-16": (16, 1800), "HDL-32E": (32, 1800),
                                                        "Ouster-OS1-16": (16, 1024), "Ouster-OS1-64": (64, 1024)}
    d, v = default_segment_params(), lidar_segment_params("Velodyne-64-HDE")
    assert bytes(d) == bytes(v)


# ---- helpers -----------------------------------------------------------------------------------------------------------------
# zone layouts (sectors, rings): 504 (the default), 1664, 3328 and 4096 (the limit) patches
LAYOUTS = [((16, 32, 54, 32), (2, 4, 4, 4)), ((32, 64, 64, 64), (4, 8, 8, 8)), ((64, 128, 128, 128), (4, 8, 8, 8)),
           ((64, 128, 128, 128), (4, 10, 10, 10))]


def _pp(height=1.723, layout=0, num_iter=3, global_elev=0):
    pp = default_patchwork_params()
    pp.sensor_height, pp.num_iter, pp.using_global_elevation = height, num_iter, global_elev
    sec, rings = LAYOUTS[layout]
    for k in range(4):
        pp.num_sectors_each_zone[k], pp.num_rings_each_zone[k] = sec[k], rings[k]
    return pp


def _sp(model="Velodyne-64-HDE", mode=2, min_pts=30):
    sp = lidar_segment_params(model)
    sp.neighbor_mode, sp.min_pts_for_subclustering = mode, min_pts
    return sp


def _fleet_scan(seed, model, height):
    """A generator scan with the model's rings and columns, seen from a sensor `height` above the ground (the generator's is 1.723)."""
    rings, cols = LIDAR_MODELS[model][:2]
    s = synth.outdoor_pair(seed, rings=rings, azimuths=cols)[seed % 2].copy()
    s[:, 2] += np.float32(1.723 - height)
    return s


def _fleet(n, seed0):
    """n scans of the five lidar models in turn, each with its own height, zone layout, iteration count, global-elevation switch,
    neighbour mode and segment size."""
    scans, pps, sps = [], [], []
    for i in range(n):
        model, h = MODELS[i % 5], 1.60 + 0.025 * ((7 * i) % 11)
        scans.append(_fleet_scan(seed0 + i, model, h))
        pps.append(_pp(h, layout=(i // 2) % 4, num_iter=(3, 5, 1)[i % 3], global_elev=(i // 3) % 2))
        sps.append(_sp(model, mode=(i // 2) % 3, min_pts=(30, 10, 60, 45)[i % 4]))
    return scans, pps, sps


def _alone(h, scan, pp, sp):
    """qb200_preprocess_batch on the scan alone with its entry: (outputs, counts, status)."""
    per, counts, status = h.preprocess_batch([scan], pp, sp)
    return per[0], list(counts[0]), int(status[0])


def _oracle(oracle, scan, pp, sp):
    g, ng, st = oracle.patchwork(scan, pp)
    if sp is None:
        return (g, ng, None, None), [len(g), len(ng), 0, 0], st
    v, o = oracle.segment_cloud(ng, sp)
    return (g, ng, v, o), [len(g), len(ng), len(v), len(o)], st


def _same_scan(got, ref, where):
    (outs, cnt, st), (routs, rcnt, rst) = got, ref
    assert list(cnt) == list(rcnt) and st == rst, (where, list(cnt), list(rcnt), st, rst)
    for k, (a, b) in enumerate(zip(outs, routs)):
        if b is None:
            assert a is None or len(a) == 0, (where, PREPROCESS_ARRAYS[k])
            continue
        assert same_bits(a, b), f"{where}: {PREPROCESS_ARRAYS[k]} differs"


def _check_each(h, scans, pps, sps, refs, **kw):
    """The batch against each scan's references (a list per scan of (outputs, counts, status))."""
    per, counts, status = h.preprocess_batch_each(scans, pps, sps, **kw)
    assert len(per) == len(scans)
    for i in range(len(scans)):
        for r in refs[i]:
            _same_scan((per[i], counts[i], int(status[i])), r, i)
    return per, counts, status


def _capacity_scan():
    """An ordinary scene plus one patch of 17000 points (more than a patch's 16384 in shared memory)."""
    rng = np.random.default_rng(5)
    base = _fleet_scan(990, "VLP-16", 1.723)
    blob = np.stack([rng.uniform(5.0, 5.5, 17000), rng.uniform(0.05, 0.3, 17000), rng.normal(-1.72, 0.01, 17000), np.ones(17000)], 1)
    return np.concatenate([base, blob.astype(np.float32)])


# ---- GPU ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fleet(oracle):
    """11 fleet scans with their entries, and each scan's oracle chain."""
    scans, pps, sps = _fleet(11, 1100)
    return scans, pps, sps, [_oracle(oracle, s, p, q) for s, p, q in zip(scans, pps, sps)]


@pytest.mark.gpu
@pytest.mark.parametrize("slots", [1, 2, 4])
def test_mixed_sensors_across_waves_match_single_scans_and_oracle(fleet, slots):
    """Waves of 2, 4 and 8 scans: the same scans ride in different waves next to different sensors."""
    scans, pps, sps, orc = fleet
    assert {sp.n_scan * sp.horizon_scan for sp in sps} == {64 * 1800, 16 * 1800, 32 * 1800, 16 * 1024, 64 * 1024}
    assert len({(p.num_sectors_each_zone[3], p.num_rings_each_zone[1]) for p in pps}) == 4 and len({p.sensor_height for p in pps}) > 5
    assert {sp.neighbor_mode for sp in sps} == {0, 1, 2} and {p.num_iter for p in pps} == {1, 3, 5}
    with capi.Handle(max_batch_slots=slots) as h:
        refs = [[_alone(h, s, p, q), orc[i]] for i, (s, p, q) in enumerate(zip(scans, pps, sps))]
        _, counts, status = _check_each(h, scans, pps, sps, refs)
        assert (status == 0).all() and (counts[:, 2] > 0).sum() >= len(scans) // 2
        if slots == 2:
            _inputs_outputs_and_cap(h, scans, pps, sps, refs)


def _inputs_outputs_and_cap(h, scans, pps, sps, refs):
    """Host and device inputs and outputs give the references' bytes; a cap that clips some scans keeps their prefixes and writes
    nothing past it."""
    import torch
    dev = [torch.from_numpy(np.ascontiguousarray(s)).cuda() for s in scans]
    dev_in = [(d.data_ptr(), len(s)) for d, s in zip(dev, scans)]
    for kind, inp in ((MEM_HOST, scans), (MEM_DEVICE, dev_in)):
        for dest in (MEM_HOST, MEM_DEVICE):
            _check_each(h, inp, pps, sps, [r[:1] for r in refs], kind=kind, dest=dest)
    counts = np.array([r[0][1] for r in refs])
    cap = 4000
    assert (counts > cap).any() and (counts <= cap).any()      # the cap clips some scans' arrays and not others
    n = len(scans)
    for dest in (MEM_HOST, MEM_DEVICE):
        host = {k: np.full((n, cap, 4), SENTINEL * 0x01010101, np.uint32).view(np.float32) for k in PREPROCESS_ARRAYS}
        arrays = host if dest == MEM_HOST else {k: torch.from_numpy(a.copy()).cuda() for k, a in host.items()}
        per, c2, _ = h.preprocess_batch_each(scans, pps, sps, cap=cap, dest=dest, arrays=arrays)
        assert np.array_equal(c2, counts)
        got = {k: (a if dest == MEM_HOST else a.cpu().numpy()) for k, a in arrays.items()}
        for i in range(n):
            for j, k in enumerate(PREPROCESS_ARRAYS):
                m = min(int(counts[i, j]), cap)
                assert same_bits(got[k][i, :m], refs[i][0][0][j][:m]), (dest, i, k)
                assert (got[k][i, m:].view(np.uint8) == SENTINEL).all(), (dest, i, k, "written past the count or the cap")


@pytest.mark.gpu
def test_identical_entries_equal_the_broadcast_call():
    scans = [_fleet_scan(1200 + i, "Velodyne-64-HDE", 1.723) for i in range(9)]
    pp, sp = _pp(1.70, layout=1, num_iter=4), _sp("Velodyne-64-HDE", mode=1, min_pts=20)
    with capi.Handle(max_batch_slots=2) as h:
        for spp in (sp, None):
            b0 = h.launch_count()
            ref = h.preprocess_batch(scans, pp, spp)
            b1 = h.launch_count()
            got = h.preprocess_batch_each(scans, [pp] * len(scans), None if spp is None else [spp] * len(scans))
            b2 = h.launch_count()
            assert b2 - b1 == b1 - b0, (b1 - b0, b2 - b1)
            assert np.array_equal(got[1], ref[1]) and np.array_equal(got[2], ref[2])
            for i in range(len(scans)):
                assert all((a is None and b is None) or same_bits(a, b) for a, b in zip(got[0][i], ref[0][i])), i
        # an empty batch: nothing launched, nothing written
        b0 = h.launch_count()
        per, counts, status = h.preprocess_batch_each([], [], [])
        assert per == [] and h.launch_count() == b0


@pytest.mark.gpu
def test_shuffled_scans_permute_the_results(fleet):
    scans, pps, sps, _ = fleet
    with capi.Handle(max_batch_slots=2) as h:
        per, counts, status = h.preprocess_batch_each(scans, pps, sps)
        perm = np.random.default_rng(3).permutation(len(scans))
        per2, counts2, status2 = h.preprocess_batch_each([scans[i] for i in perm], [pps[i] for i in perm], [sps[i] for i in perm])
        for j, i in enumerate(perm):
            assert np.array_equal(counts2[j], counts[i]) and status2[j] == status[i]
            assert all(same_bits(a, b) for a, b in zip(per2[j], per[i])), (i, j)


@pytest.mark.gpu
def test_edge_scans_in_mixed_waves(oracle):
    """An empty scan, an all-NaN scan and the capacity scan (status 3) between ordinary scans, each with a configuration of its own."""
    scans, pps, sps = _fleet(4, 1300)
    edge = [np.zeros((0, 4), np.float32), np.full((300, 4), np.nan, np.float32), _capacity_scan()]
    epp = [_pp(1.65, layout=3, num_iter=2), _pp(1.80, layout=1, global_elev=1), _pp(1.723, layout=0, num_iter=4)]
    esp = [_sp("HDL-32E", mode=0), _sp("Ouster-OS1-64", mode=1, min_pts=5), _sp("VLP-16", mode=2, min_pts=50)]
    order = [0, 4, 1, 5, 2, 6, 3]        # ordinary, edge, ordinary, ...
    all_s, all_p, all_q = scans + edge, pps + epp, sps + esp
    scans, pps, sps = [all_s[i] for i in order], [all_p[i] for i in order], [all_q[i] for i in order]
    with capi.Handle(max_batch_slots=2) as h:
        for q in (sps, None):
            refs = [[_alone(h, s, p, None if q is None else q[i]), _oracle(oracle, s, p, None if q is None else q[i])]
                    for i, (s, p) in enumerate(zip(scans, pps))]
            _, counts, status = _check_each(h, scans, pps, q, refs)
            assert list(status) == [0, 0, 0, 0, 0, 3, 0] and counts[5][1] > 0
            assert counts[1].sum() == 0 and counts[3].sum() == 0
            if q is None:
                assert (counts[:, 2:] == 0).all()


def _raw_each(h, scans, pps, sps, n_arrays=None):
    """qb200_preprocess_batch_each through ctypes with 0xA5-filled outputs; pps / sps None = a NULL table.  Returns (rc, counts,
    status, arrays)."""
    lib = capi.load_library()
    n = len(scans)
    ptrs, cnts, keep = capi._scan_arrays(scans, MEM_HOST)
    cap = 64
    arrays = {k: np.full((n, cap, 4), SENTINEL * 0x01010101, np.uint32) for k in PREPROCESS_ARRAYS}
    counts, status = np.full((n, 4), SENTINEL * 0x01010101, np.uint32), np.full(n, SENTINEL * 0x01010101, np.uint32)
    out = capi.PreprocessOut(cap, MEM_HOST)
    for k, a in arrays.items():
        setattr(out, k, a.ctypes.data)
    out.counts, out.status = counts.ctypes.data, status.ctypes.data
    pa = None if pps is None else (capi.PatchworkParams * n)(*pps)
    sa = None if sps is None else (capi.SegmentParams * n)(*sps)
    rc = lib.qb200_preprocess_batch_each(h.h, ptrs, cnts, n, MEM_HOST, pa, sa, C.byref(out))
    return rc, counts, status, arrays


@pytest.mark.gpu
def test_a_bad_entry_rejects_the_whole_call_and_writes_nothing():
    scans, pps, sps = _fleet(5, 1400)

    def bad(field, value, on="sp"):
        p = capi.SegmentParams.from_buffer_copy(sps[0]) if on == "sp" else capi.PatchworkParams.from_buffer_copy(pps[0])
        if field == "patches":          # 4097 patches: one past the limit
            for k in range(4):
                p.num_rings_each_zone[k], p.num_sectors_each_zone[k] = 1, 1024 + (k == 3)
        else:
            setattr(p, field, value)
        return p

    cases = [("sp", bad("n_scan", 65)), ("sp", bad("horizon_scan", 7)), ("pp", bad("num_zones", 3, "pp")),
             ("pp", bad("min_range", 2.5, "pp")), ("pp", bad("patches", None, "pp"))]
    ok = _pp()
    for k in range(4):
        ok.num_rings_each_zone[k], ok.num_sectors_each_zone[k] = 1, 1024
    with capi.Handle(max_batch_slots=1) as h:
        assert _raw_each(h, scans[:1], [ok], sps[:1])[0] == 0     # 4096 patches pass
        for pos in (0, 2, 4):
            for on, entry in cases:
                p2, s2 = list(pps), list(sps)
                (p2 if on == "pp" else s2)[pos] = entry
                rc, counts, status, arrays = _raw_each(h, scans, p2, s2)
                assert rc == -1, (pos, on)
                msg = capi.load_library().qb200_last_error(h.h).decode()
                assert f"scan {pos}" in msg, msg
                assert (counts.view(np.uint8) == SENTINEL).all() and (status.view(np.uint8) == SENTINEL).all()
                assert all((a.view(np.uint8) == SENTINEL).all() for a in arrays.values()), (pos, on)
        rc, counts, status, arrays = _raw_each(h, scans, None, sps)
        assert rc == -1 and (counts.view(np.uint8) == SENTINEL).all() and (status.view(np.uint8) == SENTINEL).all()
        assert _raw_each(h, [], None, None)[0] == 0           # a NULL table is fine for an empty batch
        # the next valid call is unaffected
        refs = [[_alone(h, s, p, q)] for s, p, q in zip(scans, pps, sps)]
        _check_each(h, scans, pps, sps, refs)


def _chain_records(h, scans, pairs, pps, sps, p, via):
    """Valid segments of every scan by one _each call (device outputs) or by per-scan calls (host outputs), then registration."""
    import torch
    if via == "single":
        valid = [h.preprocess_batch([s], pp, sp)[0][0][2] for s, pp, sp in zip(scans, pps, sps)]
        return h.register_batch([(valid[a], valid[b]) for a, b in pairs], p)
    cap = max(sp.n_scan * sp.horizon_scan for sp in sps)
    buf = {"valid4": torch.zeros((len(scans), cap, 4), dtype=torch.float32, device="cuda")}
    _, counts, status = h.preprocess_batch_each(scans, pps, sps, cap=cap, dest=MEM_DEVICE, arrays=buf)
    assert (status == 0).all()
    ptr = lambda i: buf["valid4"][i].data_ptr()
    return h.register_batch([(ptr(a), int(counts[a, 2]), ptr(b), int(counts[b, 2])) for a, b in pairs], p, kind=MEM_DEVICE)


@pytest.mark.gpu
def test_device_outputs_of_a_mixed_fleet_feed_registration_unchanged():
    p = capi.default_params()
    p.skip_flagged = 0
    scans, pps, sps, pairs = [], [], [], []
    for k, model in enumerate(("Velodyne-64-HDE", "HDL-32E", "Ouster-OS1-64")):
        rings, cols = LIDAR_MODELS[model][:2]
        src, tgt, _ = synth.outdoor_pair(1500 + k, rings=rings, azimuths=cols)
        for j, s in enumerate((src, tgt)):
            height = 1.62 + 0.05 * (2 * k + j)
            s = s.copy()
            s[:, 2] += np.float32(1.723 - height)
            scans.append(s)
            pps.append(_pp(height))
            sps.append(_sp(model))
        pairs.append((2 * k, 2 * k + 1))
    pairs.append((1, 2))
    with capi.Handle(max_batch_slots=2) as h:
        ref = _chain_records(h, scans, pairs, pps, sps, p, "single")
        assert (ref["status"] == 0).sum() >= 3
        got = _chain_records(h, scans, pairs, pps, sps, p, "each")
        assert got.tobytes() == ref.tobytes()
