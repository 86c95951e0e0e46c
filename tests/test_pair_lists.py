"""Per-pair lists of the batch entry points (qb200_pair_lists): correspondences, matched points, max clique, final inliers and the
inlier masks of every pair of qb200_register_batch_ex / _enqueue_ex, qb200_register_cached_ex and qb200_solve_batch_ex."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import (Handle, ListBuffers, LIST_LAYOUT, SET_LISTS, FLAG_LISTS_TRUNCATED, MEM_HOST, MEM_DEVICE, PMC_EXACT,
                              INLIER_NONE, RESULT_DTYPE, default_params)
from support import build_against_lib, host_lists, same_lists, sentinel_lists

FIXTURE = "tests/fixtures/pair_lists_shim.cpp"


# ---- CPU: the C++ fixture builds ----------------------------------------------------------------------------------------------------
def test_pair_lists_fixture_compiles(tmp_path):
    exe = build_against_lib(tmp_path, FIXTURE)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr


# ---- GPU --------------------------------------------------------------------------------------------------------------------------
STREET_SEEDS = range(60, 80)   # 20 pairs: three waves on an 8-slot handle


@pytest.fixture(scope="module")
def street():
    return [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in STREET_SEEDS]


@pytest.fixture(scope="module")
def oracle_lists(street, oracle):
    """Per pair, what the CPU oracle computes on its own voxelized clouds."""
    p = default_params()
    out = []
    for src, tgt in street:
        sv, _ = oracle.voxelize(src, p.voxel_size, p.skip_flagged)
        tv, _ = oracle.voxelize(tgt, p.voxel_size, p.skip_flagged)
        corr, sm, tm, _ = oracle.match_and_pack(sv, tv, p)
        _, _, clique, fin = oracle.solve_correspondences(sm, tm, p, want_sets=True)
        _, rm, tmask, _ = oracle.solve_pose(sm, tm, clique, p)
        out.append({"corr": corr, "src_matched4": sm, "tgt_matched4": tm, "clique": clique, "final_inliers": fin,
                    "rot_inlier_mask": rm, "trans_inlier_mask": tmask})
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("lanes", ["1", None])
def test_batch_lists_match_oracle_and_single_pair(street, oracle_lists, monkeypatch, lanes):
    if lanes:
        monkeypatch.setenv("QB200_LANES", lanes)
    else:
        monkeypatch.delenv("QB200_LANES", raising=False)
    p = default_params()
    with Handle(max_batch_slots=8) as h:
        recs, lists = h.register_batch_lists(street, p)
        assert recs.tobytes() == h.register_batch(street, p).tobytes()
        assert not (recs["flags"] & FLAG_LISTS_TRUNCATED).any()
        for (src, tgt), r, got, want in zip(street, recs, lists, oracle_lists):
            assert r["status"] == 0 and r["n_final_inliers"] > 0
            same_lists(got, want)
            one, _ = h.register_pair(src, tgt, p)
            assert bytes(one) == r.tobytes()
            corr, sm, tm = h.last_correspondences()
            same_lists(got, {"corr": corr, "src_matched4": sm, "tgt_matched4": tm, "clique": h.last_clique(),
                              "final_inliers": h.last_final_inliers()})
        # one pair through _ex also sets what the single-pair getters read
        h.register_pair(*street[1], p)
        r1, l1 = h.register_batch_lists(street[:1], p)
        assert np.array_equal(h.last_clique(), l1[0]["clique"]) and np.array_equal(h.last_final_inliers(), l1[0]["final_inliers"])


@pytest.mark.gpu
def test_destinations_and_input_kinds_give_identical_bytes(street):
    import torch
    p = default_params()
    pairs = street[:11]
    dev = [(torch.from_numpy(s).cuda(), torch.from_numpy(t).cuda()) for s, t in pairs]
    ptrs = [(a.data_ptr(), a.shape[0], b.data_ptr(), b.shape[0]) for a, b in dev]
    torch.cuda.synchronize()
    with Handle(max_batch_slots=8) as h:
        cap = h.cfg.max_corr
        runs = []
        for kind, inputs in ((MEM_HOST, pairs), (MEM_DEVICE, ptrs)):
            for dest in (MEM_HOST, MEM_DEVICE):
                lb = ListBuffers(len(pairs), cap, dest, device=h.cfg.device)
                recs, _ = h.register_batch_lists(inputs, p, kind=kind, buffers=lb)
                runs.append((recs.tobytes(), {n: lb.host(n).tobytes() for n in LIST_LAYOUT}))
    for r in runs[1:]:
        assert r == runs[0]


@pytest.mark.gpu
def test_enqueue_ex_batches_land_in_their_own_arrays(street):
    import torch
    p = default_params()
    batches = [street[0:11], street[11:16], street[16:20]]
    with Handle(max_batch_slots=4) as h:
        ref = [h.register_batch_lists(b, p) for b in batches]
        keep, outs, bufs = [], [], []
        for i, b in enumerate(batches):
            arr, k = h.pair_array(b)
            keep.append((arr, k))
            outs.append(np.zeros(len(b), RESULT_DTYPE))
            bufs.append(None if i == 1 else ListBuffers(len(b), h.cfg.max_corr, MEM_DEVICE if i == 2 else MEM_HOST, device=h.cfg.device))
        for (arr, _), out, lb in zip(keep, outs, bufs):
            if lb is None:
                h.register_batch_enqueue_raw(arr, len(out), p, MEM_HOST, out)
            else:
                h.register_batch_enqueue_lists_raw(arr, len(out), p, MEM_HOST, out, lb)
        h.register_batch_flush()
        torch.cuda.synchronize()
        for (recs, lists), out, lb in zip(ref, outs, bufs):
            assert out.tobytes() == recs.tobytes()
            if lb is not None:
                for got, want in zip(host_lists(lb.trimmed(out)), lists):
                    same_lists(got, want)


@pytest.mark.gpu
def test_cached_lists_equal_batch_lists(street):
    p = default_params()
    scans = [s for pr in street[:4] for s in pr]
    idx = [(0, 1), (2, 3), (4, 5), (6, 7), (0, 3), (5, 2)]
    with Handle(max_batch_slots=4) as h:
        recs, lists = h.register_batch_lists([(scans[a], scans[b]) for a, b in idx], p)
        h.cache_reserve(len(scans))
        h.cache_scans(scans, list(range(len(scans))), p)
        crecs, clists = h.register_cached_lists(idx, p)
        assert crecs.tobytes() == recs.tobytes()
        for (a, b), got, want in zip(idx, clists, lists):
            same_lists(got, want)
            va, vb = h.cache_read(a)[0], h.cache_read(b)[0]
            assert np.array_equal(va[got["corr"][:, 0], :3], got["src_matched4"][:, :3])
            assert np.array_equal(vb[got["corr"][:, 1], :3], got["tgt_matched4"][:, :3])


@pytest.mark.gpu
def test_solve_batch_lists(oracle):
    import torch
    sizes = (40, 0, 1, 2, 700, 5000, 3, 160, 33, 2)
    sets = []
    for i, L in enumerate(sizes):
        a4, b4, _, _ = synth.matched_pairs(500 + i, max(L, 1), inlier_ratio=0.95 if L == 5000 else 0.4, noise=0.03)
        sets.append((a4[:L], b4[:L]))
    with Handle(max_batch_slots=4, max_corr=8192) as h:
        for mode, chosen in ((None, range(len(sets))), (PMC_EXACT, [0, 1, 2, 3, 6, 7, 8]), (INLIER_NONE, [0, 1, 2, 4, 7])):
            p = default_params()
            if mode is not None:
                p.inlier_selection_mode = mode
            sub = [sets[i] for i in chosen]
            recs, lists = h.solve_batch_lists(sub, p)
            assert recs.tobytes() == h.solve_batch(sub, p).tobytes()
            for (a4, b4), r, got in zip(sub, recs, lists):
                assert set(got) == set(SET_LISTS)
                one, _ = h.solve_correspondences(a4, b4, p)
                assert bytes(one) == r.tobytes()
                same_lists(got, {"clique": h.last_clique(), "final_inliers": h.last_final_inliers()})
                if len(a4) < 2:
                    # the oracle returns before it fills its sets; a degenerate clique has no solved masks
                    assert not got["rot_inlier_mask"].any() and not got["trans_inlier_mask"].any()
                    continue
                _, _, clique, fin = oracle.solve_correspondences(a4, b4, p, want_sets=True)
                _, rm, tm, _ = oracle.solve_pose(a4, b4, clique, p)
                same_lists(got, {"clique": clique, "final_inliers": fin, "rot_inlier_mask": rm, "trans_inlier_mask": tm})
            if mode is None:
                assert recs["clique_size"][sizes.index(5000)] > 4096
                dev = [(torch.from_numpy(np.ascontiguousarray(a)).cuda(), torch.from_numpy(np.ascontiguousarray(b)).cuda()) for a, b in sub]
                torch.cuda.synchronize()
                drecs, dlists = h.solve_batch_lists([(a.data_ptr() if len(a) else 0, b.data_ptr() if len(b) else 0, len(a)) for a, b in dev], p,
                                                    kind=MEM_DEVICE, dest=MEM_DEVICE)
                assert drecs.tobytes() == recs.tobytes()
                for got, want in zip(host_lists(dlists), lists):
                    same_lists(got, want)
        # the caller supplied the correspondences: asking for them back is refused
        lb = ListBuffers(2, 64, MEM_HOST, ("corr", "clique"))
        with pytest.raises(capi.QuatroB200Error) as e:
            h.solve_batch_lists(sets[:2], default_params(), buffers=lb)
        assert e.value.code == -1


@pytest.mark.gpu
@pytest.mark.parametrize("dest", [MEM_HOST, MEM_DEVICE])
def test_truncated_lists_are_prefixes_and_flagged(street, dest):
    p = default_params()
    pairs = street[:10]
    with Handle(max_batch_slots=8) as h:
        full_recs, full = h.register_batch_lists(pairs, p)
        cap = int(np.median(full_recs["clique_size"]))
        for names in (SET_LISTS, tuple(LIST_LAYOUT)):
            lb = ListBuffers(len(pairs), cap, dest, tuple(LIST_LAYOUT), h.cfg.device)
            sentinel_lists(lb)
            d = lb.descriptor()
            for n in set(LIST_LAYOUT) - set(names):
                setattr(d, n, None)                       # not asked for: must stay all sentinel
            out = np.zeros(len(pairs), RESULT_DTYPE)
            arr, keep = h.pair_array(pairs)
            h._check(h.lib.qb200_register_batch_ex(h.h, arr, len(pairs), C.byref(p), MEM_HOST, capi._ptr(out), C.byref(d)), "ex")
            want_flag = np.zeros(len(pairs), bool)
            for n in names:
                want_flag |= full_recs[LIST_LAYOUT[n][2]] > cap
            assert 0 < want_flag.sum() <= len(pairs)
            assert np.array_equal((out["flags"] & FLAG_LISTS_TRUNCATED) != 0, want_flag)
            assert (out["flags"] & ~FLAG_LISTS_TRUNCATED).tobytes() == full_recs["flags"].tobytes()
            plain = out.copy()
            plain["flags"] &= ~FLAG_LISTS_TRUNCATED
            assert plain.tobytes() == full_recs.tobytes()
            for n in LIST_LAYOUT:
                a = lb.host(n)
                raw = a.reshape(len(pairs), cap, -1).view(np.uint8).reshape(len(pairs), -1)
                per = raw.shape[1] // cap
                for i in range(len(pairs)):
                    m = min(int(full_recs[i][LIST_LAYOUT[n][2]]), cap) if n in names else 0
                    assert (raw[i, m * per:] == 0xA5).all(), (n, i)          # nothing past min(count, cap)
                    assert a[i, :m].tobytes() == full[i][n][:m].tobytes()   # a prefix of the full list


@pytest.mark.gpu
def test_capacity_exceeded_pair_gets_no_entries(street):
    p = default_params()
    small = synth.outdoor_pair(90, rings=8, azimuths=200)[:2]
    pairs = [street[0], small, street[1]]
    with Handle(max_batch_slots=4, max_corr=64) as h:
        lb = ListBuffers(len(pairs), 64, MEM_HOST)
        sentinel_lists(lb)
        recs, _ = h.register_batch_lists(pairs, p, buffers=lb)
        assert recs.tobytes() == h.register_batch(pairs, p).tobytes()
        over = recs["status"] == 3
        assert over.any()
        for n in LIST_LAYOUT:
            raw = lb.arrays[n].reshape(len(pairs), -1).view(np.uint8)
            for i in np.flatnonzero(over):
                assert (raw[i] == 0xA5).all(), n


@pytest.mark.gpu
def test_lists_cost_one_launch_per_wave_and_nothing_without(street):
    p = default_params()
    pairs = street[:11]                      # three waves of 4
    with Handle(max_batch_slots=4) as h:
        h.register_batch(pairs, p)           # lanes allocated, kernels warmed
        arr, keep = h.pair_array(pairs)
        out = np.zeros(len(pairs), RESULT_DTYPE)

        def launches(fn):
            before = h.launch_count()
            fn()
            return h.launch_count() - before

        plain = launches(lambda: h.register_batch(pairs, p))
        null = launches(lambda: h._check(h.lib.qb200_register_batch_ex(h.h, arr, len(pairs), C.byref(p), MEM_HOST, capi._ptr(out), None), "ex"))
        with_lists = launches(lambda: h.register_batch_lists(pairs, p))
        dev_lists = launches(lambda: h.register_batch_lists(pairs, p, dest=MEM_DEVICE))
        assert plain == null and with_lists == dev_lists == plain + 3


@pytest.mark.gpu
def test_fixture_reads_inliers_of_a_sweep(tmp_path, street):
    exe = build_against_lib(tmp_path, FIXTURE)
    scans = [street[0][0], street[0][1], street[2][1]]
    files = []
    for i, s in enumerate(scans):
        f = tmp_path / f"s{i}.bin"
        f.write_bytes(np.ascontiguousarray(s, np.float32).tobytes())
        files.append(str(f))
    r = subprocess.run([str(exe), *files], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "PAIR_LISTS_SHIM_OK" in r.stdout, r.stdout + r.stderr
    p = default_params()
    with Handle(max_batch_slots=4) as h:
        recs, lists = h.register_batch_lists([(scans[0], scans[1]), (scans[0], scans[2])], p)
    lines = [ln.split() for ln in r.stdout.splitlines() if ln.startswith("pair ")]
    for ln, rec, l in zip(lines, recs, lists):
        assert list(map(int, ln[2:7])) == [rec["status"], rec["n_corr"], rec["clique_size"], rec["n_final_inliers"], rec["flags"]]
        if rec["n_final_inliers"] > 0:
            assert list(map(int, ln[7:9])) == l["corr"][l["final_inliers"][0]].tolist()
