"""Cached pairs and correspondence sets on every lane, and their stream forms: qb200_register_cached_enqueue_mixed and
qb200_solve_batch_enqueue_each.  Records and lists never depend on the lane count; a stream of raw, cached and set batches completed by
one flush equals the blocking calls, latching rotation noise bounds in enqueue order; a queued cached batch registers the slot contents
it was enqueued against; a rejected enqueue writes nothing and leaves the batches queued before it intact."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import (COTE_WEIGHTED_MEAN, INLIER_NONE, KCORE_HEU, LIST_LAYOUT, MEM_DEVICE, MEM_HOST, RESULT_DTYPE, SET_LISTS,
                              ListBuffers)
from support import ROOT, device_copies, host_lists, make_handle, make_params, same_lists, sentinel, sentinel_lists

NEW = {"qb200_register_cached_enqueue_mixed": "qb200_register_cached_mixed", "qb200_solve_batch_enqueue_each": "qb200_solve_batch_each"}


# ---- CPU: declarations, bindings, a null handle ------------------------------------------------------------------------------------
def test_header_declares_the_enqueue_calls_and_compiles_as_c(tmp_path):
    """Each new function has the type of its blocking sibling."""
    body = "".join(f"__typeof__(&{sib}) f{i} = {new};\n" for i, (new, sib) in enumerate(NEW.items()))
    (tmp_path / "enq.c").write_text('#include "quatro_b200.h"\n' + body + "int main(void) { return f0 == 0; }\n")
    r = subprocess.run(["/usr/bin/gcc", "-std=gnu11", "-Wall", "-Werror", "-Wincompatible-pointer-types", f"-I{ROOT / 'include'}", "-c",
                        str(tmp_path / "enq.c"), "-o", str(tmp_path / "enq.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_library_exports_the_enqueue_calls_with_their_siblings_signatures():
    lib = capi.load_library()
    for new, sib in NEW.items():
        assert new in capi.EXPORTED_SYMBOLS
        assert getattr(lib, new).argtypes == getattr(lib, sib).argtypes, new
        assert getattr(lib, new).restype == getattr(lib, sib).restype, new


def test_enqueue_calls_refuse_a_null_handle():
    lib = capi.load_library()
    assert lib.qb200_register_cached_enqueue_mixed(None, None, 0, None, None, None) == -1
    assert lib.qb200_solve_batch_enqueue_each(None, None, 0, None, MEM_HOST, None, None) == -1


# ---- configurations ----------------------------------------------------------------------------------------------------------------
SLOTS, LANES = 4, 4
N = 2 * SLOTS * LANES + 3   # more waves than lanes: every lane runs more than one wave of a batch
BASE = make_params(seed=11)
# the front end of BASE, solver fields varied (the _each forms)
SOLVERS = [BASE, make_params(seed=11, noise_bound=0.35, cote_mode=COTE_WEIGHTED_MEAN),
           make_params(seed=11, inlier_selection_mode=KCORE_HEU, kcore_heuristic_threshold=0.3),
           make_params(seed=11, inlier_selection_mode=INLIER_NONE), make_params(seed=11, cbar2=0.8, rotation_max_iterations=20)]
# front ends varied too (the _mixed forms)
FRONTS = [BASE, make_params(voxel_size=0.4, grid_cell=0.4, seed=14, rotation_gnc_factor=1.6),
          make_params(voxel_size=0.25, grid_cell=0.4, seed=13, noise_bound=0.35)]
SET_SIZES = [0, 1, 40, 300, 1200, 2500, 700]


def cycled(n, sets):
    return [sets[i % len(sets)] for i in range(n)]


def _untouched(out, lb):
    return (out.view(np.uint8) == 0xA5).all() and all((a.view(np.uint8) == 0xA5).all() for a in lb.arrays.values())


# ---- GPU fixtures ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def street():
    return [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(400, 400 + N)]


@pytest.fixture(scope="module")
def sets():
    return [tuple(a[:L] for a in synth.matched_pairs(700 + i, max(L, 1), inlier_ratio=0.35, noise=0.03)[:2])
            for i, L in enumerate(cycled(N, SET_SIZES))]


# slot pairs: [0, 2N) hold every scan cached with BASE, [2N, 4N) every scan cached with FRONTS[(scan // 2) % 3]
PLAIN = [(2 * i, 2 * i + 1) for i in range(N)]
PLAIN[5] = (10, 23)   # scans of two different pairs
MIXED = [(2 * N + 2 * i, 2 * N + 2 * i + 1) for i in range(N)]
MIXED_PARAMS = [FRONTS[i % 3] for i in range(N)]


def _cache(h, street):
    scans = [s for pr in street for s in pr]
    h.cache_reserve(4 * N)
    h.cache_scans(scans, list(range(2 * N)), BASE)
    h.cache_scans_each(scans, list(range(2 * N, 4 * N)), [FRONTS[(i // 2) % 3] for i in range(2 * N)])


@pytest.fixture(scope="module")
def h4(street):
    h = make_handle(LANES, max_batch_slots=SLOTS)
    _cache(h, street)
    yield h
    h.close()


@pytest.fixture(scope="module")
def h1(street):
    h = make_handle(1, max_batch_slots=SLOTS)
    _cache(h, street)
    yield h
    h.close()


def _device_sets(sets):
    ptrs, keep = device_copies([x for s in sets for x in s])
    return [(a, b, n) for (a, n), (b, _) in zip(ptrs[0::2], ptrs[1::2])], keep


def _flat(recs, lb):
    return recs.tobytes(), (None if lb is None else [{k: v.tobytes() for k, v in d.items()} for d in host_lists(lb.trimmed(recs))])


def _cached_calls(h):
    """every cached form, lists on the host and on the device: name -> (record bytes, list bytes)"""
    out = {"plain": _flat(h.register_cached(PLAIN, BASE), None)}
    for dest in (MEM_HOST, MEM_DEVICE):
        lb = ListBuffers(N, h.cfg.max_corr, dest, device=h.cfg.device)
        out[f"ex{dest}"] = _flat(h.register_cached_lists(PLAIN, BASE, buffers=lb)[0], lb)
        lb = ListBuffers(N, h.cfg.max_corr, dest, device=h.cfg.device)
        out[f"each{dest}"] = _flat(h.register_cached_each(PLAIN, cycled(N, SOLVERS), buffers=lb)[0], lb)
        lb = ListBuffers(N, h.cfg.max_corr, dest, device=h.cfg.device)
        out[f"mixed{dest}"] = _flat(h.register_cached_mixed(MIXED, MIXED_PARAMS, buffers=lb)[0], lb)
    return out


def _set_calls(h, sets):
    dev, keep = _device_sets(sets)
    out = {}
    for kind, ss in ((MEM_HOST, sets), (MEM_DEVICE, dev)):
        for dest in (MEM_HOST, MEM_DEVICE):
            lb = ListBuffers(N, h.cfg.max_corr, dest, SET_LISTS, h.cfg.device)
            out[f"ex{kind}{dest}"] = _flat(h.solve_batch_lists(ss, BASE, kind, buffers=lb)[0], lb)
            lb = ListBuffers(N, h.cfg.max_corr, dest, SET_LISTS, h.cfg.device)
            out[f"each{kind}{dest}"] = _flat(h.solve_batch_each(ss, cycled(N, SOLVERS), kind, buffers=lb)[0], lb)
    return out


# ---- GPU 1: the lane count changes nothing -----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_cached_forms_do_not_depend_on_the_lane_count(h1, h4):
    one, four = _cached_calls(h1), _cached_calls(h4)
    assert one.keys() == four.keys()
    for name in one:
        assert one[name] == four[name], name
    recs = np.frombuffer(four["plain"][0], RESULT_DTYPE)
    assert (recs["status"] == 0).sum() >= N - 2 and len(set(recs["n_corr"])) > 1
    assert len(set(np.frombuffer(four[f"mixed{MEM_HOST}"][0], RESULT_DTYPE)["n_src_vox"][:3])) == 3   # the front ends really differ


@pytest.mark.gpu
def test_set_forms_do_not_depend_on_the_lane_count(h1, h4, sets):
    one, four = _set_calls(h1, sets), _set_calls(h4, sets)
    for name in one:
        assert one[name] == four[name], name
    assert four[f"ex{MEM_HOST}{MEM_HOST}"] == four[f"ex{MEM_DEVICE}{MEM_DEVICE}"]
    recs = np.frombuffer(four[f"each{MEM_HOST}{MEM_HOST}"][0], RESULT_DTYPE)
    assert len(set(recs["clique_size"])) > 3


# ---- GPU 2: raw, cached and set batches in one stream --------------------------------------------------------------------------------
@pytest.mark.gpu
def test_one_stream_of_cached_raw_and_set_batches(street, sets):
    """Three batches, one flush; entries with rot_noise_bound = 0 latch in enqueue order (the cached batch's first such entry)."""
    cached_p = [make_params(voxel_size=p.voxel_size, grid_cell=p.grid_cell, seed=p.seed, rotation_gnc_factor=p.rotation_gnc_factor,
                            noise_bound=0.45 if i % 4 == 1 else p.noise_bound, rot_noise_bound=0.0 if i % 4 == 1 else 2 * p.noise_bound)
                for i, p in enumerate(MIXED_PARAMS)]
    raw_p = [make_params(seed=20 + i % 3, noise_bound=0.6 if i % 2 else 0.3, rot_noise_bound=0.0 if i % 3 == 0 else 1.0) for i in range(N)]
    set_p = [make_params(noise_bound=0.5, rot_noise_bound=0.0 if i % 2 else 0.9, inlier_selection_mode=SOLVERS[i % 5].inlier_selection_mode)
             for i in range(N)]
    latch = 2 * cached_p[1].noise_bound
    assert latch not in (2 * raw_p[0].noise_bound, 2 * set_p[1].noise_bound)

    def resolved(ps):
        out = [capi.Params.from_buffer_copy(p) for p in ps]
        for q in out:
            q.rot_noise_bound = q.rot_noise_bound or latch
        return out

    with make_handle(LANES, max_batch_slots=SLOTS) as h, make_handle(LANES, max_batch_slots=SLOTS) as ref:
        for hh in (h, ref):
            _cache(hh, street)
        dev, keep_dev = _device_sets(sets)
        slot_arr = capi._slot_array(MIXED)
        pair_arr, keep_pairs = h.pair_array(street)
        set_arr, _ = h._set_array(dev, MEM_DEVICE)
        outs = [np.zeros(N, RESULT_DTYPE) for _ in range(3)]
        bufs = [ListBuffers(N, h.cfg.max_corr, MEM_HOST), ListBuffers(N, h.cfg.max_corr, MEM_DEVICE, device=h.cfg.device),
                ListBuffers(N, h.cfg.max_corr, MEM_HOST, SET_LISTS)]
        pas = [h.params_array(ps) for ps in (cached_p, raw_p, set_p)]
        h.register_cached_enqueue_mixed_raw(slot_arr, N, pas[0], outs[0], bufs[0])
        h.register_batch_enqueue_mixed_raw(pair_arr, N, pas[1], MEM_HOST, outs[1], bufs[1])
        h.solve_batch_enqueue_each_raw(set_arr, N, pas[2], MEM_DEVICE, outs[2], bufs[2])
        h.register_batch_flush()
        got = [_flat(o, b) for o, b in zip(outs, bufs)]
        # the blocking calls on a fresh handle, in the same order
        want = []
        for fn, ps in ((lambda lb, ps: ref.register_cached_mixed(MIXED, ps, buffers=lb), cached_p),
                       (lambda lb, ps: ref.register_batch_mixed(street, ps, buffers=lb), raw_p),
                       (lambda lb, ps: ref.solve_batch_each(dev, ps, MEM_DEVICE, buffers=lb), set_p)):
            lb = ListBuffers(N, ref.cfg.max_corr, MEM_HOST, SET_LISTS if ps is set_p else tuple(LIST_LAYOUT))
            want.append(_flat(fn(lb, ps)[0], lb))
        for k in range(3):
            assert got[k] == want[k], k
        # ... and with every zero bound replaced by the cached batch's latch: the first batch enqueued latched
        for k, (ps, fn) in enumerate(((cached_p, lambda ps: h.register_cached_mixed(MIXED, ps)),
                                      (raw_p, lambda ps: h.register_batch_mixed(street, ps)),
                                      (set_p, lambda ps: h.solve_batch_each(dev, ps, MEM_DEVICE)))):
            assert fn(resolved(ps))[0].tobytes() == got[k][0], k


# ---- GPU 3: a queued cached batch sees the slots it was enqueued against --------------------------------------------------------------
@pytest.mark.gpu
def test_a_queued_cached_batch_keeps_its_slot_contents(h4, street):
    old = [(0, 2 * i + 1) for i in range(N)]
    new_scan = street[7][1]                       # cached with BASE in slot 15 already
    want_old = h4.register_cached(old, BASE)
    want_new = h4.register_cached([(15, b) for _, b in old], BASE)
    assert want_old.tobytes() != want_new.tobytes()
    out = np.zeros(N, RESULT_DTYPE)
    slot_arr = capi._slot_array(old)
    try:
        h4.register_cached_enqueue_mixed_raw(slot_arr, N, h4.params_array([BASE] * N), out)
        h4.cache_scans([new_scan], [0], BASE)     # flushes first: the queued batch ran against the old scan
        h4.register_batch_flush()
        assert out.tobytes() == want_old.tobytes()
        assert h4.register_cached(old, BASE).tobytes() == want_new.tobytes()
    finally:
        h4.cache_scans([street[0][0]], [0], BASE)


# ---- GPU 4: rejections ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_rejected_enqueue_writes_nothing_and_keeps_the_queue(h4, sets):
    n = 2 * SLOTS * LANES + 1
    good_slots = capi._slot_array(PLAIN[:n])
    good_params = h4.params_array([BASE] * n)
    want_cached = h4.register_cached(PLAIN[:n], BASE)
    set_arr, keep_sets = h4._set_array(sets[:n], MEM_HOST)
    want_sets, _ = h4.solve_batch_each(sets[:n], [BASE] * n)
    lib = h4.lib

    def cached(slot_pairs, ps, n_=None, cap=64):
        sp = capi._slot_array(slot_pairs)
        out, lb = sentinel(max(len(sp), 1), RESULT_DTYPE), sentinel_lists(ListBuffers(len(sp), 64))
        d = lb.descriptor()
        d.cap_per_pair = cap
        st = lib.qb200_register_cached_enqueue_mixed(h4.h, capi._ptr(sp), len(sp) if n_ is None else n_, h4.params_array(ps),
                                                     capi._ptr(out), C.byref(d))
        return st, out, lb

    def set_call(n_=None, cap=64, ps=None):
        out, lb = sentinel(3, RESULT_DTYPE), sentinel_lists(ListBuffers(3, 64, MEM_HOST, SET_LISTS))
        d = lb.descriptor()
        d.cap_per_pair = cap
        st = lib.qb200_solve_batch_enqueue_each(h4.h, set_arr, 3 if n_ is None else n_, h4.params_array(ps or [BASE] * 3), MEM_HOST,
                                                capi._ptr(out), C.byref(d))
        return st, out, lb

    no_cross = make_params(seed=11, use_crosscheck=0)
    cases = {
        "n < 0": (lambda: cached(PLAIN[:3], [BASE] * 3, n_=-1), -1),
        "slot outside": (lambda: cached([(0, 1), (4 * N, 1), (2, 3)], [BASE] * 3), -1),
        "signature": (lambda: cached([(0, 1), (2 * N + 2, 3)], [BASE] * 2), -1),   # slot 2N + 2 holds FRONTS[1]
        "cap 0": (lambda: cached(PLAIN[:3], [BASE] * 3, cap=0), -1),
        "cap > max_corr": (lambda: cached(PLAIN[:3], [BASE] * 3, cap=h4.cfg.max_corr + 1), -1),
        "crosscheck": (lambda: cached(PLAIN[:3], [BASE, no_cross, BASE]), -4),
        "sets n < 0": (lambda: set_call(n_=-1), -1),
        "sets cap 0": (lambda: set_call(cap=0), -1),
        "sets bad entry": (lambda: set_call(ps=[BASE, make_params(noise_bound=-1.0), BASE]), -1),
    }
    for name, (call, code) in cases.items():
        out1, out2 = np.zeros(n, RESULT_DTYPE), np.zeros(n, RESULT_DTYPE)
        assert lib.qb200_register_cached_enqueue_mixed(h4.h, capi._ptr(good_slots), n, good_params, capi._ptr(out1), None) == 0
        st, out, lb = call()
        assert st == code, (name, st, lib.qb200_last_error(h4.h).decode())
        assert lib.qb200_solve_batch_enqueue_each(h4.h, set_arr, n, good_params, MEM_HOST, capi._ptr(out2), None) == 0
        h4.register_batch_flush()
        assert _untouched(out, lb), name
        assert out1.tobytes() == want_cached.tobytes(), name
        assert out2.tobytes() == want_sets.tobytes(), name
