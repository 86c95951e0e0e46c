"""qb200_preprocess_batch: the example's pre-processing (Patchwork ground removal, then range-image sub-cluster removal) for many scans
in one call.  Every scan's four outputs, counts and status must be byte-identical to qb200_patchwork followed by qb200_segment_cloud
on the same handle, and to the CPU oracle's chain, whatever the batch size, the wave, the scan's position, the memory kinds or the
capacity per scan."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import MEM_DEVICE, MEM_HOST, PREPROCESS_ARRAYS, default_patchwork_params, default_segment_params
from support import build_against_lib, same_bits

CANARY = np.uint32(0x7FC0DEAD)   # a NaN no kernel writes


def test_preprocess_batch_fixture_compiles(tmp_path):
    exe = build_against_lib(tmp_path, "tests/fixtures/preprocess_batch_shim.cpp")
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr


def test_preprocess_batch_refuses_a_null_handle():
    lib = capi.load_library()
    counts, status = np.zeros(4, np.int32), np.zeros(1, np.int32)
    out = capi.PreprocessOut(1, MEM_HOST)
    out.counts, out.status = counts.ctypes.data, status.ctypes.data
    assert lib.qb200_preprocess_batch(None, None, None, 0, MEM_HOST, C.byref(default_patchwork_params()), None, C.byref(out)) == -1


# ---- helpers -----------------------------------------------------------------------------------------------------------------
def _scene(seed, n_obj=20):
    """Flat ground seen from the origin + boxes standing on it (w < 0 marks ground), shuffled."""
    rng = np.random.default_rng(seed)
    az, r = rng.uniform(0, 2 * np.pi, 30000), rng.uniform(3.0, 70.0, 30000)
    g = np.stack([r * np.cos(az), r * np.sin(az), -1.723 + rng.normal(0, 0.02, len(r))], 1)
    objs = []
    for _ in range(n_obj):
        c = rng.uniform(-50, 50, 2)
        side = rng.integers(0, 4, 600)
        u, v = rng.uniform(-1, 1, 600), rng.uniform(-1.4, 1.1, 600)
        objs.append(np.stack([np.where(side < 2, np.where(side == 0, -1.0, 1.0), u) + c[0],
                              np.where(side < 2, u, np.where(side == 2, -1.0, 1.0)) + c[1], v], 1))
    pts = np.concatenate([g, *objs]).astype(np.float32)
    out = np.ones((len(pts), 4), np.float32)
    out[:, :3] = pts
    out[:len(g), 3] = -1.0
    return out[rng.permutation(len(out))]


def _single(h, scan, pp, sp):
    """The two single-scan calls: (ground, nonground, valid, outlier), counts, status."""
    g, ng, st = h.patchwork(scan, pp)
    if sp is None:
        return (g, ng, None, None), [len(g), len(ng), 0, 0], st
    v, o = h.segment_cloud(ng, sp)
    return (g, ng, v, o), [len(g), len(ng), len(v), len(o)], st


def _oracle(oracle, scan, pp, sp):
    g, ng, st = oracle.patchwork(scan, pp)
    if sp is None:
        return (g, ng, None, None), [len(g), len(ng), 0, 0], st
    v, o = oracle.segment_cloud(ng, sp)
    return (g, ng, v, o), [len(g), len(ng), len(v), len(o)], st


def _check_batch(h, scans, pp, sp, oracle=None, **kw):
    per, counts, status = h.preprocess_batch(scans, pp, sp, **kw)
    assert len(per) == len(scans)
    for i, sc in enumerate(scans):
        refs = [_single(h, sc, pp, sp)] + ([_oracle(oracle, sc, pp, sp)] if oracle is not None else [])
        for outs, cnt, st in refs:
            assert list(counts[i]) == cnt and status[i] == st, (i, list(counts[i]), cnt, status[i], st)
            for k, (a, b) in enumerate(zip(per[i], outs)):
                if b is None:
                    assert counts[i][k] == 0
                    continue
                assert same_bits(a, b), f"scan {i}: {PREPROCESS_ARRAYS[k]} differs"
    return per, counts, status


def _generator_scans(n, seed0=700, small=False):
    """64 x 1800 generator scans (the default segment parameters' image); small: 32 x 900 (sparse: almost every pixel an outlier)."""
    size = {"rings": 32, "azimuths": 900} if small else {}
    return [synth.outdoor_pair(seed0 + i, **size)[i % 2] for i in range(n)]


# ---- GPU ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("lanes", ["1", None])
def test_batch_of_several_waves_matches_single_calls_and_oracle(oracle, monkeypatch, lanes):
    """2S + 3 generator scans: two full waves and a partial one."""
    if lanes:
        monkeypatch.setenv("QB200_LANES", lanes)
    else:
        monkeypatch.delenv("QB200_LANES", raising=False)
    pp, sp = default_patchwork_params(), default_segment_params()
    with capi.Handle(max_batch_slots=4) as h:
        scans = _generator_scans(2 * 2 * 4 + 3 - 4) + _generator_scans(4, 730, small=True)
        _, counts, _ = _check_batch(h, scans, pp, sp, oracle)
        assert (counts[:-4, 2] > 0).all()


def _capacity_scan():
    """A scan with one patch of 17000 points (more than a patch's 16384 in shared memory) next to an ordinary scene."""
    rng = np.random.default_rng(5)
    base = _scene(8, n_obj=4)
    blob = np.stack([rng.uniform(5.0, 5.5, 17000), rng.uniform(0.05, 0.3, 17000), rng.normal(-1.72, 0.01, 17000), np.ones(17000)], 1)
    return np.concatenate([base, blob.astype(np.float32)])


@pytest.mark.gpu
def test_mixed_waves_with_edge_scans(oracle):
    R = 60000
    pp, sp = default_patchwork_params(), default_segment_params()
    full = synth.outdoor_pair(711)[0]
    full = np.concatenate([full] * (R // len(full) + 1))[:R]
    labelled = _scene(9)
    labelled[::97, 2] = np.nan
    labelled[5::113, 2] = -0.0
    labelled[7::131, 0] = -0.0
    scans = [_generator_scans(1, small=True)[0], np.zeros((0, 4), np.float32), np.full((300, 4), np.nan, np.float32), full, _capacity_scan(),
             labelled, _generator_scans(1, 740, small=True)[0]]
    with capi.Handle(max_batch_slots=2, max_raw_points=R) as h:      # waves of 4: the edge scans share waves with ordinary ones
        _, counts, status = _check_batch(h, scans, pp, sp, oracle)
        assert list(status) == [0, 0, 0, 0, 3, 0, 0] and counts[4][1] > 0 and counts[3].sum() > 0 and counts[3][2] > 0
        assert counts[1].sum() == 0 and counts[2].sum() == 0
        # the scan above max_raw_points is refused with the whole call
        with pytest.raises(capi.QuatroB200Error) as e:
            h.preprocess_batch(scans + [np.zeros((R + 1, 4), np.float32)], pp, sp)
        assert e.value.code == -1
        # ground removal only
        _check_batch(h, scans, pp, None, oracle)
        # the second Patchwork parameter set
        pp2 = default_patchwork_params()
        pp2.num_iter, pp2.using_global_elevation, pp2.uprightness_thr, pp2.num_min_pts = 5, 1, 0.5, 10
        _check_batch(h, scans, pp2, sp, oracle)
        # VLP-16 constants in all three neighbour modes
        for mode in (0, 1, 2):
            sv = default_segment_params()
            sv.n_scan, sv.horizon_scan, sv.ang_res_x, sv.ang_res_y, sv.ang_bottom = 16, 1800, 0.2, 2.0, 15.1
            sv.neighbor_mode = mode
            _check_batch(h, scans, pp, sv, oracle)


@pytest.mark.gpu
def test_shuffled_batch_gives_every_scan_the_same_bytes():
    pp, sp = default_patchwork_params(), default_segment_params()
    scans = _generator_scans(9, 760) + [_scene(10), _capacity_scan()]
    with capi.Handle(max_batch_slots=2) as h:
        per, counts, status = h.preprocess_batch(scans, pp, sp)
        perm = np.random.default_rng(1).permutation(len(scans))
        per2, counts2, status2 = h.preprocess_batch([scans[i] for i in perm], pp, sp)
        for j, i in enumerate(perm):
            assert np.array_equal(counts2[j], counts[i]) and status2[j] == status[i]
            assert all(same_bits(a, b) for a, b in zip(per2[j], per[i])), (i, j)
        # one scan alone, and the batch again: nothing is left over from an earlier call or wave
        for i in (0, 10):
            one, c1, s1 = h.preprocess_batch([scans[i]], pp, sp)
            assert np.array_equal(c1[0], counts[i]) and s1[0] == status[i] and all(same_bits(a, b) for a, b in zip(one[0], per[i]))


@pytest.mark.gpu
def test_host_and_device_inputs_and_outputs_give_the_same_bytes():
    import torch
    pp, sp = default_patchwork_params(), default_segment_params()
    scans = _generator_scans(7, 780) + [np.zeros((0, 4), np.float32)]
    dev = [torch.from_numpy(np.ascontiguousarray(s)).cuda() if len(s) else None for s in scans]
    dev_in = [(d.data_ptr() if d is not None else 0, len(s)) for d, s in zip(dev, scans)]
    with capi.Handle(max_batch_slots=2) as h:
        ref, rc, rs = h.preprocess_batch(scans, pp, sp)
        for kind, inp in ((MEM_HOST, scans), (MEM_DEVICE, dev_in)):
            for dest in (MEM_HOST, MEM_DEVICE):
                per, counts, status = h.preprocess_batch(inp, pp, sp, kind=kind, dest=dest)
                assert np.array_equal(counts, rc) and np.array_equal(status, rs)
                for i in range(len(scans)):
                    assert all(same_bits(a, b) for a, b in zip(per[i], ref[i])), (kind, dest, i)


@pytest.mark.gpu
@pytest.mark.parametrize("dest", [MEM_HOST, MEM_DEVICE])
def test_clipped_cap_keeps_prefixes_and_writes_nothing_past_it(dest):
    import torch
    pp, sp = default_patchwork_params(), default_segment_params()
    scans = _generator_scans(5, 800)
    cap = 1500
    with capi.Handle(max_batch_slots=2) as h:
        full, counts, status = h.preprocess_batch(scans, pp, sp)
        n = len(scans)
        # ground and valid only: non-ground and outlier are NULL
        host = {k: np.full((n, cap, 4), CANARY, np.uint32).view(np.float32) for k in ("ground4", "valid4")}
        arrays = host if dest == MEM_HOST else {k: torch.from_numpy(a.copy()).cuda() for k, a in host.items()}
        per, c2, s2 = h.preprocess_batch(scans, pp, sp, cap=cap, dest=dest, arrays=arrays)
        assert np.array_equal(c2, counts) and np.array_equal(s2, status)
        assert (counts[:, 0] > cap).any() and (counts[:, 2] > cap).any()      # the cap clips
        got = {k: (a if dest == MEM_HOST else a.cpu().numpy()) for k, a in arrays.items()}
        for i in range(n):
            for k, j in (("ground4", 0), ("valid4", 2)):
                m = min(int(counts[i, j]), cap)
                assert same_bits(got[k][i, :m], full[i][j][:m]), (i, k)
                assert (got[k][i, m:].view(np.uint32) == CANARY).all(), (i, k, "written past the count or the cap")
            assert per[i][1] is None and per[i][3] is None


def _chain_records(h, scans, pairs, p, via):
    """valid segments of every scan by the batch (device outputs) or by the single calls, then registration of `pairs`."""
    import torch
    pp, sp = default_patchwork_params(), default_segment_params()
    if via == "single":
        valid = [h.segment_cloud(h.patchwork(s, pp)[1], sp)[0] for s in scans]
        return h.register_batch([(valid[a], valid[b]) for a, b in pairs], p)
    cap = sp.n_scan * sp.horizon_scan
    buf = {"valid4": torch.zeros((len(scans), cap, 4), dtype=torch.float32, device="cuda")}
    _, counts, status = h.preprocess_batch(scans, pp, sp, cap=cap, dest=MEM_DEVICE, arrays=buf)
    assert (status == 0).all()
    ptr = lambda i: buf["valid4"][i].data_ptr()
    if via == "batch":
        return h.register_batch([(ptr(a), int(counts[a, 2]), ptr(b), int(counts[b, 2])) for a, b in pairs], p, kind=MEM_DEVICE)
    h.cache_reserve(len(scans))
    h.cache_scans([(ptr(i), int(counts[i, 2])) for i in range(len(scans))], list(range(len(scans))), p, kind=MEM_DEVICE)
    return h.register_cached(np.array(pairs, np.int32), p)


@pytest.mark.gpu
def test_device_valid_segments_feed_registration_unchanged():
    p = capi.default_params()
    p.skip_flagged = 0
    scans, pairs = [], []
    for k in range(3):
        src, tgt, _ = synth.outdoor_pair(820 + k)
        scans += [src, tgt]
        pairs.append((2 * k, 2 * k + 1))
    pairs.append((1, 2))
    with capi.Handle(max_batch_slots=2) as h:
        ref = _chain_records(h, scans, pairs, p, "single")
        assert (ref["status"] == 0).sum() >= 3
        for via in ("batch", "cache"):
            got = _chain_records(h, scans, pairs, p, via)
            assert got.tobytes() == ref.tobytes(), via


@pytest.mark.gpu
def test_launches_per_wave_do_not_depend_on_the_scans_in_it():
    pp, sp = default_patchwork_params(), default_segment_params()
    scans = _generator_scans(5, 840)
    with capi.Handle(max_batch_slots=2) as h:      # waves of 4
        def launches(batch, spp):
            before = h.launch_count()
            h.preprocess_batch(batch, pp, spp)
            return h.launch_count() - before
        for spp in (sp, None):
            one, wave, two = launches(scans[:1], spp), launches(scans[:4], spp), launches(scans[:5], spp)
            assert one == wave and two == 2 * wave, (one, wave, two)
            assert launches([np.zeros((0, 4), np.float32)], spp) == one


@pytest.mark.gpu
def test_preprocess_batch_refuses_bad_arguments():
    pp, sp = default_patchwork_params(), default_segment_params()
    lib = capi.load_library()
    scans = _generator_scans(2, 860)
    with capi.Handle(max_batch_slots=2) as h:
        ptrs = (C.c_void_p * 2)(*[s.ctypes.data for s in scans])
        n = (C.c_int32 * 2)(*[len(s) for s in scans])
        counts, status = np.full((2, 4), -7, np.int32), np.full(2, -7, np.int32)
        g = np.full((2, 10, 4), CANARY, np.uint32)

        def call(ptrs=ptrs, n=n, n_scans=2, kind=MEM_HOST, pp=pp, sp=sp, cap=10, okind=MEM_HOST, counts=counts, status=status, nul=False):
            out = capi.PreprocessOut(cap, okind)
            out.ground4 = g.ctypes.data
            out.counts = counts.ctypes.data if counts is not None else None
            out.status = status.ctypes.data if status is not None else None
            return lib.qb200_preprocess_batch(h.h, ptrs, n, n_scans, kind, C.byref(pp) if pp is not None else None,
                                              C.byref(sp) if sp is not None else None, None if nul else C.byref(out))

        bad_pp = default_patchwork_params()
        bad_pp.num_zones = 3
        bad_sp = default_segment_params()
        bad_sp.n_scan = 65
        too_big = (C.c_int32 * 2)(len(scans[0]), 131073)
        null_scan = (C.c_void_p * 2)(scans[0].ctypes.data, None)
        for kw in ({"n_scans": -1}, {"kind": 2}, {"pp": None}, {"pp": bad_pp}, {"sp": bad_sp}, {"cap": 0}, {"okind": 5},
                   {"counts": None}, {"status": None}, {"nul": True}, {"n": too_big}, {"ptrs": null_scan}, {"okind": MEM_DEVICE}):
            assert call(**kw) == -1, kw
        assert (counts == -7).all() and (status == -7).all() and (g == CANARY).all()     # no work started
        assert call() == 0 and (counts[:, 0] > 0).all()
