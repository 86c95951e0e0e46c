"""One params entry per pair, front end included: qb200_register_batch_mixed, _enqueue_mixed, qb200_register_cached_mixed and
qb200_cache_scans_each.  Pair i of a _mixed call is byte-identical to pair i of the _ex call made with params[i] for the whole batch and
matches the oracle run with its own params; a cached slot equals qb200_cache_scans of its scan with its entry; a rejected call writes
nothing."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import (COTE_WEIGHTED_MEAN, INLIER_NONE, KCORE_HEU, LIST_LAYOUT, MEM_DEVICE, MEM_HOST, RESULT_DTYPE, Handle,
                              ListBuffers, default_params)
from support import ROOT, assert_same_record, build_against_lib, host_lists, make_handle, make_params, same_lists, sentinel, sentinel_lists

MIXED = {"qb200_register_batch_mixed": "qb200_register_batch_each", "qb200_register_batch_enqueue_mixed": "qb200_register_batch_enqueue_each",
         "qb200_register_cached_mixed": "qb200_register_cached_each", "qb200_cache_scans_each": "qb200_cache_scans"}


# ---- CPU: declarations, bindings and the INTEGRATION.md snippet ---------------------------------------------------------------------
def test_header_declares_the_mixed_calls_and_compiles_as_c(tmp_path):
    """Each new function has its sibling's type (a pointer of the sibling's type takes its address without a warning)."""
    body = "".join(f"__typeof__(&{sib}) f{i} = {new};\n" for i, (new, sib) in enumerate(MIXED.items()))
    (tmp_path / "mixed.c").write_text('#include "quatro_b200.h"\n' + body + "int main(void) { return f0 == 0; }\n")
    r = subprocess.run(["/usr/bin/gcc", "-std=gnu11", "-Wall", "-Werror", "-Wincompatible-pointer-types", f"-I{ROOT / 'include'}", "-c",
                        str(tmp_path / "mixed.c"), "-o", str(tmp_path / "mixed.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_ctypes_signatures_match_the_siblings():
    lib = capi.load_library()
    for new, sib in MIXED.items():
        assert new in capi.EXPORTED_SYMBOLS
        assert getattr(lib, new).argtypes == getattr(lib, sib).argtypes, new
        assert getattr(lib, new).restype == getattr(lib, sib).restype, new


def test_mixed_sweep_fixture_compiles(tmp_path):
    build_against_lib(tmp_path, "tests/fixtures/frontend_mixed_shim.cpp")


def test_mixed_calls_refuse_a_null_handle():
    lib = capi.load_library()
    assert lib.qb200_register_batch_mixed(None, None, 0, None, MEM_HOST, None, None) == -1
    assert lib.qb200_register_cached_mixed(None, None, 0, None, None, None) == -1
    assert lib.qb200_cache_scans_each(None, None, None, None, 0, None, MEM_HOST) == -1


# ---- configurations -----------------------------------------------------------------------------------------------------------------
# Cycled over the pairs: bench.py's street and dense presets, three voxel sizes whose explicit lattice cell gives a lattice reach of 2
# for both radii (ceil(0.75 / 0.4), ceil(0.5 / 0.4), ...), equal radii, flagged points kept, the tuple test switched off by its scale,
# zero and 250 trials per correspondence; every entry its own seed, and solver fields varied alongside.
CONFIGS = [
    make_params(seed=11),
    make_params(voxel_size=0.22, use_tuple_test=0, seed=12, inlier_selection_mode=KCORE_HEU, kcore_heuristic_threshold=0.3),
    make_params(voxel_size=0.25, grid_cell=0.4, seed=13, noise_bound=0.35, cote_mode=COTE_WEIGHTED_MEAN),
    make_params(voxel_size=0.4, grid_cell=0.4, seed=14, rotation_gnc_factor=1.6, rotation_max_iterations=20),
    make_params(voxel_size=0.6, grid_cell=0.5, seed=15, normal_radius=0.6, fpfh_radius=0.9, noise_bound=0.4),
    make_params(normal_radius=0.75, fpfh_radius=0.75, seed=16, cote_noise_bound=0.35, using_rot_inliers_when_estimating_cote=1),
    make_params(skip_flagged=0, voxel_size=0.35, seed=17, inlier_selection_mode=INLIER_NONE),
    make_params(tuple_scale=0.0, seed=18, cbar2=0.8),
    make_params(tuple_trials_per_corr=0, seed=19, noise_bound=0.25),
    make_params(tuple_trials_per_corr=250, tuple_scale=0.9, seed=20, rotation_cost_threshold=1e-3),
]
LANES = 4
SLOTS = 4
N_PAIRS = 2 * SLOTS * LANES + 3   # more waves than lanes: every lane runs more than one wave of a batch


def cycled(n, offset=0, sets=CONFIGS):
    return [sets[(i + offset) % len(sets)] for i in range(n)]


def _untouched(out, lb):
    return (out.view(np.uint8) == 0xA5).all() and all((a.view(np.uint8) == 0xA5).all() for a in lb.arrays.values())


# ---- GPU fixtures --------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def street():
    return [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(300, 300 + N_PAIRS)]


@pytest.fixture(scope="module")
def h():
    with pytest.MonkeyPatch.context() as mp:
        mp.delenv("QB200_LANES", raising=False)
        handle = Handle(max_batch_slots=SLOTS)
    yield handle
    handle.close()


@pytest.fixture(scope="module")
def broadcast(h, street):
    """per configuration k: records and lists of qb200_register_batch_ex over every street pair with CONFIGS[k]"""
    return [h.register_batch_lists(street, p) for p in CONFIGS]


def _check_against_broadcast(recs, lists, broadcast, index, params_index):
    for j, (i, k) in enumerate(zip(index, params_index)):
        want_recs, want_lists = broadcast[k]
        assert recs[j].tobytes() == want_recs[i].tobytes(), (j, i, k)
        same_lists(lists[j], want_lists[i])


# ---- GPU 1: mixed configurations across waves ------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_mixed_configurations_equal_broadcast_and_oracle(h, street, broadcast, oracle):
    params = cycled(len(street))
    recs, lists = h.register_batch_mixed(street, params, buffers=ListBuffers(len(street), h.cfg.max_corr))
    ks = [i % len(CONFIGS) for i in range(len(street))]
    _check_against_broadcast(recs, lists, broadcast, range(len(street)), ks)
    # zero tuple trials mark no correspondence: those pairs are degenerate inputs, as in the reference; every other pair registers
    zero_trials = np.array([bool(p.use_tuple_test) and p.tuple_scale != 0 and p.tuple_trials_per_corr == 0 for p in params])
    assert (recs["status"][zero_trials] == 2).all() and (recs["status"][~zero_trials] == 0).all()
    # the configurations really differ: voxel counts of one scan under the first five presets are pairwise distinct
    assert len({int(broadcast[k][0][0]["n_src_vox"]) for k in range(5)}) == 5
    for (src, tgt), r, p in zip(street, recs, params):
        ref, st = oracle.register_pair(src, tgt, p)
        assert r["status"] == st
        assert_same_record(r, ref)


# ---- GPU 2: a seed sweep of one pair ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_seed_sweep_of_one_pair(h, street):
    pair = street[0]
    params = [make_params(seed=1000 + 7 * k) for k in range(8)]
    recs, lists = h.register_batch_mixed([pair] * 8, params, buffers=ListBuffers(8, h.cfg.max_corr))
    for k, p in enumerate(params):
        want, want_lists = h.register_batch_lists([pair], p)
        assert recs[k].tobytes() == want[0].tobytes(), k
        same_lists(lists[k], want_lists[0])
    assert len({r.tobytes() for r in recs}) > 1, "every seed gave the same record: the seed is not per pair"


# ---- GPU 3: a pair's size refusal stays its own ----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_size_faults_stay_per_pair(h, street, broadcast):
    overflow = make_params(voxel_size=1e-7, seed=31)                  # PCL's int voxel index would overflow
    too_many = make_params(voxel_size=0.08, skip_flagged=0, seed=32)  # > max_voxel_points voxels (~21.5 k)
    n = 2 * SLOTS + 3
    params = cycled(n)
    params[2], params[SLOTS + 1] = overflow, too_many
    pairs = street[:n]
    recs, lists = h.register_batch_mixed(pairs, params, buffers=ListBuffers(n, h.cfg.max_corr))
    assert recs["status"][2] == -5 and recs["status"][SLOTS + 1] == 3   # QB200_ERR_VOXEL_OVERFLOW, QB200_CAPACITY_EXCEEDED
    for i in (2, SLOTS + 1):
        want, want_lists = h.register_batch_lists([pairs[i]], params[i])
        assert recs[i].tobytes() == want[0].tobytes(), i
        same_lists(lists[i], want_lists[0])
    rest = [i for i in range(n) if i not in (2, SLOTS + 1)]
    _check_against_broadcast(recs[rest], [lists[i] for i in rest], broadcast, rest, [i % len(CONFIGS) for i in rest])


# ---- GPU 4: clouds above the shared-memory lattice sort in a mixed wave -------------------------------------------------------------
@pytest.mark.gpu
def test_indoor_and_street_pairs_in_one_large_v_wave(street):
    indoor = make_params(voxel_size=0.05, normal_radius=0.10, fpfh_radius=0.15, noise_bound=0.05, cote_noise_bound=0.05, skip_flagged=0,
                         seed=41)   # bench.py's indoor preset
    pairs = [street[0], synth.indoor_pair(5)[:2], street[1]]
    params = [CONFIGS[0], indoor, CONFIGS[1]]
    with make_handle(None, max_batch_slots=4, max_raw_points=524288, max_voxel_points=65536) as hb:
        recs, lists = hb.register_batch_mixed(pairs, params, buffers=ListBuffers(3, hb.cfg.max_corr))
        assert recs["n_src_vox"][1] > 17920
        for i, (pr, p) in enumerate(zip(pairs, params)):
            want, want_lists = hb.register_batch_lists([pr], p)
            assert recs[i].tobytes() == want[0].tobytes(), i
            same_lists(lists[i], want_lists[0])


# ---- GPU 5: the pipelined form ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_two_enqueued_mixed_batches_and_one_flush(h, street, broadcast):
    cut = 2 * SLOTS * 2 + 1
    parts = [(0, cut, 0), (cut, len(street), 3)]   # (first pair, end, configuration offset)
    keep, outs, bufs, plans = [], [], [], []
    for a, b, off in parts:
        arr, k = h.pair_array(street[a:b])
        pa = h.params_array(cycled(b - a, off))
        keep.append((arr, k, pa))
        outs.append(np.zeros(b - a, RESULT_DTYPE))
        bufs.append(ListBuffers(b - a, h.cfg.max_corr, MEM_DEVICE if off else MEM_HOST, device=h.cfg.device))
        plans.append((range(a, b), [(j + off) % len(CONFIGS) for j in range(b - a)]))
    for (arr, _, pa), out, lb in zip(keep, outs, bufs):
        h.register_batch_enqueue_mixed_raw(arr, len(out), pa, MEM_HOST, out, lb)
    h.register_batch_flush()
    import torch
    torch.cuda.synchronize()
    for out, lb, (index, ks) in zip(outs, bufs, plans):
        _check_against_broadcast(out, host_lists(lb.trimmed(out)), broadcast, index, ks)


# ---- GPU 6: the scan cache --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_cache_scans_each_and_register_cached_mixed(h, street):
    sets = [CONFIGS[0], CONFIGS[1], CONFIGS[2]]
    scans = [s for pr in street for s in pr]          # 2 N_PAIRS scans: more than 2S per call
    n = len(scans)
    cfg_of_scan = [(i // 2) % 3 for i in range(n)]    # both scans of a pair share a configuration
    h.cache_reserve(2 * n)
    try:
        h.cache_scans_each(scans, list(range(n)), [sets[k] for k in cfg_of_scan])
        for k in range(3):                            # slots n + i: the broadcast call, one configuration at a time
            idx = [i for i in range(n) if cfg_of_scan[i] == k]
            h.cache_scans([scans[i] for i in idx], [n + i for i in idx], sets[k])
        for i in range(n):
            got, want = h.cache_read(i), h.cache_read(n + i)
            assert all(g.tobytes() == w.tobytes() for g, w in zip(got, want)), i
        assert len({len(h.cache_read(i)[0]) for i in range(6)}) > 1
        pairs = [(2 * i, 2 * i + 1) for i in range(len(street))]
        pairs[4] = (8, 21)                            # scans of two pairs, both in configuration 1
        params = [sets[cfg_of_scan[a]] for a, _ in pairs]
        recs, lists = h.register_cached_mixed(pairs, params, buffers=ListBuffers(len(pairs), h.cfg.max_corr))
        for k in range(3):
            idx = [j for j in range(len(pairs)) if params[j] is sets[k]]
            want, want_lists = h.register_cached_lists([pairs[j] for j in idx], sets[k])
            for w, j in enumerate(idx):
                assert recs[j].tobytes() == want[w].tobytes(), (k, j)
                same_lists(lists[j], want_lists[w])
        # a pair whose entry does not match one of its slots (slot 2 holds configuration 1) rejects the whole call
        bad = [pairs[0], (0, 2), pairs[2]]
        sp = np.ascontiguousarray(np.asarray(bad, np.int32))
        out, lb = sentinel(3, RESULT_DTYPE), sentinel_lists(ListBuffers(3, 64))
        st = h.lib.qb200_register_cached_mixed(h.h, capi._ptr(sp), 3, h.params_array([sets[0], sets[0], sets[2]]), capi._ptr(out),
                                               C.byref(lb.descriptor()))
        assert st == -1 and _untouched(out, lb)
        assert "pair 1" in h.lib.qb200_last_error(h.h).decode()
        # qb200_cache_copy carries the signature: the copied slot is accepted with its source's entry only
        h.cache_copy(2, 0)
        got, _ = h.register_cached_mixed([(0, 3)], [sets[1]])
        assert got.tobytes() == h.register_cached_lists([(2, 3)], sets[1])[0].tobytes()
        out = sentinel(1, RESULT_DTYPE)
        sp = np.ascontiguousarray(np.asarray([(0, 3)], np.int32))
        assert h.lib.qb200_register_cached_mixed(h.h, capi._ptr(sp), 1, h.params_array([sets[0]]), capi._ptr(out), None) == -1
    finally:
        h.cache_reserve(0)


# ---- GPU 7: identical entries are the broadcast call, launch for launch ------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("k", [0, 1, 7])
def test_identical_entries_equal_the_broadcast_call(h, street, k):
    p = CONFIGS[k]
    pairs = street[:2 * SLOTS + 3]
    h.register_batch_lists(pairs, p)                  # lanes allocated, scratch and kernels warmed

    def run(fn):
        lb = ListBuffers(len(pairs), h.cfg.max_corr)
        before = h.launch_count()
        recs, _ = fn(lb)
        return recs.tobytes(), {n: lb.host(n).tobytes() for n in LIST_LAYOUT}, h.launch_count() - before

    ex = run(lambda lb: h.register_batch_lists(pairs, p, buffers=lb))
    assert run(lambda lb: h.register_batch_mixed(pairs, [p] * len(pairs), buffers=lb)) == ex


# ---- GPU 8: validation --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_bad_entry_rejects_the_whole_call(street):
    pairs = street[:SLOTS + 2]
    n = len(pairs)

    def good():
        return [make_params(seed=50 + i, voxel_size=0.25 + 0.05 * (i % 3), noise_bound=0.3 + 0.02 * i) for i in range(n)]

    def bad(k, **kw):
        ps = good()
        for f, v in kw.items():
            setattr(ps[k], f, v)
        ps[k].rot_noise_bound = 0.0       # would latch if it were resolved
        return ps

    cases = [(bad(3, normal_radius=float("nan")), -1), (bad(0, fpfh_radius=float("nan")), -1), (bad(n - 1, normal_radius=1.0), -1),
             (bad(2, voxel_size=0.0), -1), (bad(1, noise_bound=-1.0), -1), (bad(4, use_crosscheck=0), -4)]
    with make_handle(None, max_batch_slots=SLOTS) as h1, make_handle(None, max_batch_slots=SLOTS) as h2:
        scans = [s for pr in pairs for s in pr]
        h1.cache_reserve(2 * n)
        h1.cache_scans(scans, list(range(2 * n)), default_params())
        arr, keep = h1.pair_array(pairs)
        slots = np.ascontiguousarray(np.arange(2 * n, dtype=np.int32).reshape(n, 2))
        calls = {
            "register": lambda pa, out, lb: h1.lib.qb200_register_batch_mixed(h1.h, arr, n, pa, MEM_HOST, capi._ptr(out), lb),
            "enqueue": lambda pa, out, lb: h1.lib.qb200_register_batch_enqueue_mixed(h1.h, arr, n, pa, MEM_HOST, capi._ptr(out), lb),
            "cached": lambda pa, out, lb: h1.lib.qb200_register_cached_mixed(h1.h, capi._ptr(slots), n, pa, capi._ptr(out), lb),
        }
        for name, call in calls.items():
            for ps, code in cases:
                out, lb = sentinel(max(n, 1), RESULT_DTYPE), sentinel_lists(ListBuffers(n, 64))
                st = call(h1.params_array(ps), out, C.byref(lb.descriptor()))
                msg = h1.lib.qb200_last_error(h1.h).decode()
                h1.register_batch_flush()
                assert st == code, (name, st, msg)
                assert _untouched(out, lb), name
                bad_entry = next(i for i, p in enumerate(ps) if p.rot_noise_bound == 0.0)
                assert f"entry {bad_entry}" in msg, (name, msg)
        # qb200_cache_scans_each: a bad entry writes no slot
        h1.cache_reserve(2 * n)
        ptrs, cnts, keep_scans = capi._scan_arrays(scans, MEM_HOST)
        ids = (C.c_int32 * (2 * n))(*range(2 * n))
        for ps, code in cases[:5]:
            st = h1.lib.qb200_cache_scans_each(h1.h, ptrs, cnts, ids, 2 * n, h1.params_array(ps + ps), MEM_HOST)
            assert st == -1
            assert "entry" in h1.lib.qb200_last_error(h1.h).decode()
            assert all(len(h1.cache_read(s)[0]) == 0 for s in range(2 * n))
        # nothing the rejected calls saw was latched: h1's first accepted call latches as on a fresh handle
        ps = good()
        for p in ps:
            p.rot_noise_bound = 0.0
        want, _ = h2.register_batch_mixed(pairs, ps)
        got, _ = h1.register_batch_mixed(pairs, ps)
        assert got.tobytes() == want.tobytes()


# ---- GPU: the INTEGRATION.md snippet ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_mixed_sweep_fixture_matches_the_bindings(tmp_path, street):
    exe = build_against_lib(tmp_path, "tests/fixtures/frontend_mixed_shim.cpp")
    pairs = street[:4]
    args = []
    for k, (s, t) in enumerate(pairs):
        for j, a in enumerate((s, t)):
            f = tmp_path / f"scan{k}_{j}.bin"
            np.ascontiguousarray(a, np.float32).tofile(f)
            args.append(str(f))
    r = subprocess.run([str(exe), *args], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "FRONTEND_MIXED_SHIM_OK" in r.stdout, r.stderr
    lines = [ln.split() for ln in r.stdout.splitlines() if ln.startswith("pair ")]
    street_p, dense_p = default_params(), default_params()
    dense_p.voxel_size, dense_p.use_tuple_test = 0.22, 0
    with Handle(max_batch_slots=4) as hs:
        want = hs.register_batch_mixed(pairs, [street_p if k % 2 == 0 else dense_p for k in range(4)])[0]
    for k, ln in enumerate(lines[:4]):
        assert [int(x) for x in ln[2:]] == [int(want[k]["valid"]), int(want[k]["status"]), int(want[k]["n_corr"]),
                                            int(want[k]["clique_size"])], k
