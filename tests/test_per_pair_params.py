"""One params entry per pair: qb200_register_batch_each, _enqueue_each, qb200_register_cached_each and qb200_solve_batch_each.  Pair i of an
_each call is byte-identical to pair i of the _ex call made with params[i] for the whole batch, matches the oracle run with its own params,
and a rejected call writes nothing."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import (COTE_WEIGHTED_MEAN, FLAG_CLIQUE_TRUNCATED, INLIER_NONE, KCORE_HEU, LIST_LAYOUT, MEM_DEVICE, MEM_HOST,
                              PMC_EXACT, PMC_HEU, RESULT_DTYPE, SET_LISTS, Handle, ListBuffers, default_params)
from support import ROOT, assert_same_record, host_lists, make_handle, make_params, same_lists, sentinel

EACH = {"qb200_register_batch_each": "qb200_register_batch_ex", "qb200_register_batch_enqueue_each": "qb200_register_batch_enqueue_ex",
        "qb200_register_cached_each": "qb200_register_cached_ex", "qb200_solve_batch_each": "qb200_solve_batch_ex"}


# ---- CPU: declarations and bindings -------------------------------------------------------------------------------------------------
def test_header_declares_the_each_calls_and_compiles_as_c(tmp_path):
    """Each _each function has its _ex sibling's signature (a pointer of the sibling's type takes its address without a warning)."""
    body = ""
    for i, (each, ex) in enumerate(EACH.items()):
        body += f"__typeof__(&{ex}) f{i} = {each};\n"
    (tmp_path / "each.c").write_text('#include "quatro_b200.h"\n' + body + "int main(void) { return f0 == 0; }\n")
    r = subprocess.run(["/usr/bin/gcc", "-std=gnu11", "-Wall", "-Werror", "-Wincompatible-pointer-types", f"-I{ROOT / 'include'}", "-c",
                        str(tmp_path / "each.c"), "-o", str(tmp_path / "each.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_ctypes_signatures_match_the_ex_siblings():
    lib = capi.load_library()
    for each, ex in EACH.items():
        assert each in capi.EXPORTED_SYMBOLS
        assert getattr(lib, each).argtypes == getattr(lib, ex).argtypes, each
        assert getattr(lib, each).restype == getattr(lib, ex).restype, each


# ---- parameter sets ------------------------------------------------------------------------------------------------------------
def ryrx(roll_deg, pitch_deg):
    """Ry(pitch) Rx(roll), the Params.RyRx field: the roll/pitch prior an IMU gives for a scan (setPreEstaimatedRyRx)."""
    r, p = np.radians(roll_deg), np.radians(pitch_deg)
    rx = np.array([[1, 0, 0], [0, np.cos(r), -np.sin(r)], [0, np.sin(r), np.cos(r)]])
    ry = np.array([[np.cos(p), 0, np.sin(p)], [0, 1, 0], [-np.sin(p), 0, np.cos(p)]])
    return (C.c_double * 9)(*(ry @ rx).ravel())


# Six configurations cycled over the pairs: all four inlier modes (PMC_EXACT once with a one-node limit), both COTE modes with the
# rotation-inlier COTE on, noise_bound / cbar2 / cote_noise_bound at three values or more, different GNC factors and iteration caps, and
# the roll/pitch prior off and on with four matrices.
SETS = [
    make_params(),
    make_params(inlier_selection_mode=PMC_EXACT, max_clique_node_limit=1, noise_bound=0.6, cbar2=1.2, cote_noise_bound=0.25,
                cote_mode=COTE_WEIGHTED_MEAN, using_rot_inliers_when_estimating_cote=1, use_pre_estimated_RyRx=1, RyRx=ryrx(1.5, -0.8)),
    make_params(inlier_selection_mode=KCORE_HEU, kcore_heuristic_threshold=0.3, noise_bound=0.35, cbar2=0.8, cote_noise_bound=0.4,
                rotation_gnc_factor=1.6, rotation_max_iterations=20, use_pre_estimated_RyRx=1, RyRx=ryrx(-2.0, 1.0)),
    make_params(inlier_selection_mode=INLIER_NONE, cote_mode=COTE_WEIGHTED_MEAN, rotation_gnc_factor=1.2, rotation_max_iterations=8,
                use_pre_estimated_RyRx=1, RyRx=ryrx(0.5, 2.5)),
    make_params(inlier_selection_mode=PMC_EXACT, using_rot_inliers_when_estimating_cote=1),
    make_params(rotation_gnc_factor=1.8, rotation_max_iterations=30, rotation_cost_threshold=1e-3, cote_noise_bound=0.35,
                using_rot_inliers_when_estimating_cote=1, use_pre_estimated_RyRx=1, RyRx=ryrx(-1.2, -1.7), rot_noise_bound=0.5),
]
LANES = 4   # the default lane count (QB200_LANES unset)
SLOTS = 4
N_PAIRS = 2 * SLOTS * LANES + 3   # more waves than lanes: every lane runs more than one wave of a batch


def cycled(n, offset=0):
    return [SETS[(i + offset) % len(SETS)] for i in range(n)]


# ---- GPU fixtures ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def street():
    return [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(200, 200 + N_PAIRS)]


@pytest.fixture(scope="module")
def h():
    with pytest.MonkeyPatch.context() as mp:
        mp.delenv("QB200_LANES", raising=False)
        handle = Handle(max_batch_slots=SLOTS)
    yield handle
    handle.close()


@pytest.fixture(scope="module")
def broadcast(h, street):
    """per configuration k: records and lists of qb200_register_batch_ex over every street pair with SETS[k]"""
    return [h.register_batch_lists(street, p) for p in SETS]


def _check_against_broadcast(recs, lists, broadcast, index, params_index):
    """recs[j] / lists[j] against pair index[j] of the broadcast run of configuration params_index[j]"""
    for j, (i, k) in enumerate(zip(index, params_index)):
        want_recs, want_lists = broadcast[k]
        assert recs[j].tobytes() == want_recs[i].tobytes(), (j, i, k)
        same_lists(lists[j], want_lists[i])


# ---- GPU: every _each call equals its broadcast equivalent, pair by pair ------------------------------------------------------------
@pytest.mark.gpu
def test_register_batch_each_equals_broadcast_and_oracle(h, street, broadcast, oracle):
    params = cycled(len(street))
    lb = ListBuffers(len(street), h.cfg.max_corr)
    recs, lists = h.register_batch_each(street, params, buffers=lb)
    _check_against_broadcast(recs, lists, broadcast, range(len(street)), [i % len(SETS) for i in range(len(street))])
    modes = np.array([p.inlier_selection_mode for p in params])
    assert (recs["status"] == 0).all()
    assert (recs["clique_size"][modes == INLIER_NONE] == recs["n_corr"][modes == INLIER_NONE]).all()
    assert (recs["n_edges"][modes == INLIER_NONE] == 0).all() and (recs["n_edges"][modes != INLIER_NONE] > 0).all()
    for (src, tgt), r, p in zip(street, recs, params):
        ref, st = oracle.register_pair(src, tgt, p)
        # the solver part from the oracle's solve_correspondences on its own matched points: the oracle's register_pair searches
        # PMC_EXACT cliques with the default node limit, its solve_correspondences with the pair's own
        sv, _ = oracle.voxelize(src, p.voxel_size, p.skip_flagged)
        tv, _ = oracle.voxelize(tgt, p.voxel_size, p.skip_flagged)
        _, sm, tm, _ = oracle.match_and_pack(sv, tv, p)
        sol, _ = oracle.solve_correspondences(sm, tm, p)
        sol.n_src_vox, sol.n_tgt_vox, sol.n_mutual = ref.n_src_vox, ref.n_tgt_vox, ref.n_mutual
        assert r["status"] == st
        assert_same_record(r, sol)
        if p.max_clique_node_limit == 0:
            assert_same_record(r, ref)


@pytest.mark.gpu
def test_two_enqueued_each_batches_and_one_flush(h, street, broadcast):
    cut = 2 * SLOTS * 2 + 1
    parts = [(0, cut, 0), (cut, len(street), 3)]   # (first pair, end, configuration offset)
    keep, outs, bufs, plans = [], [], [], []
    for a, b, off in parts:
        arr, k = h.pair_array(street[a:b])
        pa = h.params_array(cycled(b - a, off))
        keep.append((arr, k, pa))
        outs.append(np.zeros(b - a, RESULT_DTYPE))
        bufs.append(ListBuffers(b - a, h.cfg.max_corr, MEM_DEVICE if off else MEM_HOST, device=h.cfg.device))
        plans.append((range(a, b), [(j + off) % len(SETS) for j in range(b - a)]))
    for (arr, _, pa), out, lb in zip(keep, outs, bufs):
        h.register_batch_enqueue_each_raw(arr, len(out), pa, MEM_HOST, out, lb)
    h.register_batch_flush()
    import torch
    torch.cuda.synchronize()
    for out, lb, (index, ks) in zip(outs, bufs, plans):
        _check_against_broadcast(out, host_lists(lb.trimmed(out)), broadcast, index, ks)


@pytest.mark.gpu
def test_register_cached_each_equals_cached_broadcast(h, street):
    scans = [s for pr in street for s in pr]
    idx = [(2 * i, 2 * i + 1) for i in range(len(street))]
    idx[3] = (0, 5)                                   # a scan against another pair's scan
    h.cache_reserve(len(scans))
    try:
        h.cache_scans(scans, list(range(len(scans))), default_params())
        ref = [h.register_cached_lists(idx, p) for p in SETS]
        recs, lists = h.register_cached_each(idx, cycled(len(idx)), buffers=ListBuffers(len(idx), h.cfg.max_corr))
        _check_against_broadcast(recs, lists, ref, range(len(idx)), [i % len(SETS) for i in range(len(idx))])
    finally:
        h.cache_reserve(0)


def solve_sets():
    """N_PAIRS correspondence sets on a 16384 handle: one above 8192 correspondences (K9's k-core arrays in global scratch), one whose
    clique has more than 4096 members (the pose workspace in global memory), one whose graph makes a one-node PMC_EXACT search stop
    (SETS[1]), the rest small; waves of four mix every case with small sets and other modes."""
    sets = []
    for i in range(N_PAIRS):
        L, ratio, noise, extent = 60 + 37 * i, 0.3, 0.05, 50.0
        if i == 5:
            L, ratio = 9000, 0.05
        elif i == 12:
            L, ratio, noise = 6000, 0.95, 0.03
        elif i == 7:
            L, ratio, extent = 200, 0.05, 4.0
        a4, b4, _, _ = synth.matched_pairs(700 + i, L, inlier_ratio=ratio, noise=noise, extent=extent)
        sets.append((a4, b4))
    return sets


@pytest.mark.gpu
def test_solve_batch_each_mixed_waves_equal_broadcast_and_oracle(oracle):
    sets = solve_sets()
    params = cycled(len(sets))
    with make_handle(None, max_batch_slots=SLOTS, max_corr=16384) as hs:
        ref = [hs.solve_batch_lists(sets, p) for p in SETS]
        recs, lists = hs.solve_batch_each(sets, params, buffers=ListBuffers(len(sets), hs.cfg.max_corr, MEM_HOST, SET_LISTS))
    _check_against_broadcast(recs, lists, ref, range(len(sets)), [i % len(SETS) for i in range(len(sets))])
    assert recs["n_corr"][5] > 8192 and recs["clique_size"][12] > 4096
    assert params[7].inlier_selection_mode == PMC_EXACT and recs["flags"][7] & FLAG_CLIQUE_TRUNCATED
    for (a4, b4), r, p in zip(sets, recs, params):
        r_o, st = oracle.solve_correspondences(a4, b4, p)
        assert r["status"] == st
        assert_same_record(r, r_o)


# ---- GPU: entries that are all equal are the existing call, launch for launch --------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [INLIER_NONE, PMC_HEU, PMC_EXACT])
def test_identical_entries_equal_the_broadcast_call(h, street, mode):
    p = make_params(inlier_selection_mode=mode)
    pairs = street[:2 * SLOTS + 3]
    h.register_batch_lists(pairs, p)                  # lanes allocated, scratch and kernels warmed

    def run(fn):
        lb = ListBuffers(len(pairs), h.cfg.max_corr)
        before = h.launch_count()
        recs, _ = fn(lb)
        return recs.tobytes(), {n: lb.host(n).tobytes() for n in LIST_LAYOUT}, h.launch_count() - before

    ex = run(lambda lb: h.register_batch_lists(pairs, p, buffers=lb))
    each = run(lambda lb: h.register_batch_each(pairs, [p] * len(pairs), buffers=lb))
    assert each == ex


# ---- GPU: the rotation noise latch ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_latch_resolves_in_pair_order(street):
    pairs = street[:SLOTS + 3]
    params = []
    for i, nb in enumerate((0.35, 0.25, 0.3, 0.4, 0.25, 0.3, 0.35)):
        params.append(make_params(noise_bound=nb, rot_noise_bound=0.0 if i != 2 else 0.45))
    with make_handle(None, max_batch_slots=SLOTS) as h1, make_handle(None, max_batch_slots=SLOTS) as h2:
        recs, _ = h1.register_batch_each(pairs, params)
        single = b"".join(bytes(h2.register_pair(s, t, p)[0]) for (s, t), p in zip(pairs, params))
        assert recs.tobytes() == single
        # the latch took 2 * 0.35 from entry 0: entry 1 (noise bound 0.25) is solved with 0.7, not with 0.5
        p1 = make_params(noise_bound=0.25, rot_noise_bound=0.7)
        assert recs[1].tobytes() == h2.register_batch([pairs[1]], p1).tobytes()


# ---- GPU: validation -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_bad_entries_reject_the_whole_call(street):
    pairs = street[:SLOTS + 2]
    n = len(pairs)
    good = [make_params(noise_bound=nb, rot_noise_bound=0.0) for nb in (0.3, 0.25, 0.35, 0.3, 0.25, 0.35)]
    sets = [(s[:300, :].copy(), t[:300, :].copy()) for s, t in pairs]   # any points: only the validation matters here

    def bad_solver(k, field, value):
        ps = [make_params(noise_bound=p.noise_bound, rot_noise_bound=0.0) for p in good]
        setattr(ps[k], field, value)
        return ps

    def frontend_mismatch(k):
        ps = [make_params(noise_bound=p.noise_bound, rot_noise_bound=0.0) for p in good]
        ps[k].voxel_size = 0.31
        return ps

    with make_handle(None, max_batch_slots=SLOTS) as h1, make_handle(None, max_batch_slots=SLOTS) as h2:
        h1.cache_reserve(2 * n)
        h1.cache_scans([s for pr in pairs for s in pr], list(range(2 * n)), default_params())
        arr, keep = h1.pair_array(pairs)
        sarr, skeep = h1._set_array(sets, MEM_HOST)
        slots = np.ascontiguousarray(np.arange(2 * n, dtype=np.int32).reshape(n, 2))
        calls = {
            "register": lambda pa, out, lb: h1.lib.qb200_register_batch_each(h1.h, arr, n, pa, MEM_HOST, capi._ptr(out), lb),
            "enqueue": lambda pa, out, lb: h1.lib.qb200_register_batch_enqueue_each(h1.h, arr, n, pa, MEM_HOST, capi._ptr(out), lb),
            "cached": lambda pa, out, lb: h1.lib.qb200_register_cached_each(h1.h, capi._ptr(slots), n, pa, capi._ptr(out), lb),
            "solve": lambda pa, out, lb: h1.lib.qb200_solve_batch_each(h1.h, sarr, n, pa, MEM_HOST, capi._ptr(out), lb),
        }
        bad = [bad_solver(4, "noise_bound", -1.0), bad_solver(0, "cbar2", 0.0), bad_solver(n - 1, "inlier_selection_mode", 4),
               bad_solver(2, "cote_mode", 7), bad_solver(3, "max_clique_node_limit", -5), bad_solver(1, "rotation_max_iterations", -1)]
        for name, call in calls.items():
            cases = bad + ([frontend_mismatch(3), frontend_mismatch(n - 1)] if name != "solve" else [])
            for ps in cases:
                out = sentinel(n, RESULT_DTYPE)
                lb = ListBuffers(n, 64, MEM_HOST, SET_LISTS)
                for a in lb.arrays.values():
                    a.view(np.uint8)[...] = 0xA5
                st = call(h1.params_array(ps), out, C.byref(lb.descriptor()))
                h1.register_batch_flush()
                assert st == -1, (name, st)
                assert (out.view(np.uint8) == 0xA5).all(), name
                assert all((a.view(np.uint8) == 0xA5).all() for a in lb.arrays.values()), name
        # the front-end fields do not matter to qb200_solve_batch_each: the mismatch is accepted and changes nothing
        want, _ = h1.solve_batch_each(sets, good)
        got, _ = h1.solve_batch_each(sets, frontend_mismatch(3))
        assert got.tobytes() == want.tobytes()
        # nothing the rejected calls saw was latched: h1's first accepted call latched 2 * 0.3, as on a fresh handle
        assert want.tobytes() == h2.solve_batch_each(sets, good)[0].tobytes()
