"""Scan-cache writes in the batch stream: qb200_cache_scans_enqueue_each.  Queued writes leave every slot byte-identical to the blocking
qb200_cache_scans_each, whatever the lane count or the scans' memory kind; cached batches queued around writes to their slots register
the contents they were enqueued against, and their signatures; a rejected write queues and writes nothing and keeps the queue; the calls
that flush first see every queued write."""
import ctypes as C
import hashlib
import json
import subprocess

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import MEM_DEVICE, MEM_HOST, RESULT_DTYPE, ListBuffers, default_params
from support import ROOT, device_copies, host_lists, make_handle, make_params

NEW, SIBLING = "qb200_cache_scans_enqueue_each", "qb200_cache_scans_each"


# ---- CPU: declaration, binding, a null handle ----------------------------------------------------------------------------------------
def test_header_declares_the_cache_enqueue_and_compiles_as_c(tmp_path):
    """The new function has the type of qb200_cache_scans_each."""
    (tmp_path / "enq.c").write_text(f'#include "quatro_b200.h"\n__typeof__(&{SIBLING}) f = {NEW};\n'
                                    "int main(void) { return f == 0; }\n")
    r = subprocess.run(["/usr/bin/gcc", "-std=gnu11", "-Wall", "-Werror", "-Wincompatible-pointer-types", f"-I{ROOT / 'include'}", "-c",
                        str(tmp_path / "enq.c"), "-o", str(tmp_path / "enq.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_library_exports_the_cache_enqueue_with_its_siblings_signature():
    lib = capi.load_library()
    assert NEW in capi.EXPORTED_SYMBOLS
    assert getattr(lib, NEW).argtypes == getattr(lib, SIBLING).argtypes
    assert getattr(lib, NEW).restype == getattr(lib, SIBLING).restype


def test_cache_enqueue_refuses_a_null_handle():
    assert capi.load_library().qb200_cache_scans_enqueue_each(None, None, None, None, 0, None, MEM_HOST) == -1


# ---- configurations ----------------------------------------------------------------------------------------------------------------
SLOTS, LANES, RAW_CAP = 2, 4, 32768          # a write wave holds 2 * SLOTS = 4 scans
N = 2 * SLOTS * LANES + 3                    # pairs of a reader batch: more waves than lanes
BASE = make_params(seed=11)
CFG = dict(max_batch_slots=SLOTS, max_raw_points=RAW_CAP)
FRONTS = [BASE, make_params(voxel_size=0.4, grid_cell=0.4, seed=14), make_params(voxel_size=0.25, grid_cell=0.4, seed=13, noise_bound=0.35)]


def _read(h, slot):
    v, n, d = h.cache_read(slot)
    return v.tobytes() + n.tobytes() + d.tobytes() + np.int64(len(v)).tobytes()


def _enqueue(h, scans, slots, params, kind=MEM_HOST):
    """queue a cache write; returns what must stay alive until the flush"""
    ptrs, cnts, keep = capi._scan_arrays(scans, kind)
    ids = (C.c_int32 * max(len(slots), 1))(*slots)
    h.cache_scans_enqueue_each_raw(ptrs, cnts, ids, len(scans), h.params_array(params), kind)
    return keep


# ---- GPU fixtures ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scans():
    """3N street scans: N scenes, two poses each, and a third set of scenes written over slots later"""
    pairs = [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(500, 500 + N)]
    extra = [synth.outdoor_pair(s, rings=32, azimuths=900)[0] for s in range(600, 600 + N)]
    return [c for pr in pairs for c in pr] + extra


@pytest.fixture(scope="module")
def h1():
    h = make_handle(1, **CFG)
    yield h
    h.close()


@pytest.fixture(scope="module")
def h4():
    h = make_handle(LANES, **CFG)
    yield h
    h.close()


@pytest.fixture(scope="module")
def ref():
    h = make_handle(LANES, **CFG)
    yield h
    h.close()


# ---- GPU 1: slot contents --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_queued_writes_fill_every_slot_like_the_blocking_call_alone(h1, h4, ref, scans):
    n = 2 * SLOTS * LANES + 5                 # 6 write waves
    entries = [FRONTS[i % 3] for i in range(n)]
    ref.cache_reserve(n)
    want = []
    for i in range(n):
        ref.cache_scans_each([scans[i]], [i], [entries[i]])
        want.append(_read(ref, i))
    assert len(set(want)) == n and len({len(w) for w in want}) > 1
    dev, keep_dev = device_copies(scans[:n])
    for h in (h1, h4):
        for kind, ss in ((MEM_HOST, scans[:n]), (MEM_DEVICE, dev)):
            h.cache_reserve(n)
            slots = list(range(n))[::-1]    # slot order differs from scan order
            keep = _enqueue(h, ss[::-1], slots, entries[::-1], kind)
            h.register_batch_flush()
            del keep
            for i in range(n):
                assert _read(h, i) == want[i], (h.cfg, kind, i)


@pytest.mark.gpu
def test_every_cache_path_matches_the_golden_slots(h1, h4):
    """tests/golden/cache_slots.json holds the slot digests an earlier tree's qb200_cache_scans_each computed (tools/gen_golden_cache.py):
    three waves, three front ends, slot 5 named in the first and the last wave.  The blocking call and the queued write, with host and
    device scans, on one lane and on four, give those slots byte for byte."""
    g = json.loads((ROOT / "tests" / "golden" / "cache_slots.json").read_text())
    assert g["config"] == {"max_batch_slots": SLOTS, "max_raw_points": RAW_CAP}
    ss = [c for s in g["seeds"] for c in synth.outdoor_pair(s, rings=32, azimuths=900)[:2]]
    entries = []
    for i in range(len(g["slots"])):
        p = default_params()
        for k, v in g["fronts"][i % 3].items():
            setattr(p, k, v)
        entries.append(p)
    dev, keep_dev = device_copies(ss)
    for h in (h1, h4):
        for kind, scan_in in ((MEM_HOST, ss), (MEM_DEVICE, dev)):
            for queued in (False, True):
                h.cache_reserve(len(g["digests"]))
                if queued:
                    keep = _enqueue(h, scan_in, g["slots"], entries, kind)
                    h.register_batch_flush()
                    del keep
                else:
                    h.cache_scans_each(scan_in, g["slots"], entries, kind)
                got = [hashlib.sha256(_read(h, s)).hexdigest() for s in range(len(g["digests"]))]
                assert got == g["digests"], (h.cfg.max_batch_slots, kind, queued)


# ---- GPU 2: hazards in one stream ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_one_stream_orders_writes_and_readers_of_a_slot(h4, ref, scans):
    """One flush completes: a raw batch, reader A of slot 0, write 1, reader B of slot 15, writes 2 and 3, reader C of slot 15 and a set
    batch; each equals the blocking calls made in the same order, and so does every slot.

    Every call here spans at least LANES waves, so the rotation carries on across the calls, and each wave is submitted while the three
    waves before it are still in flight on the other lanes (a lane is collected only when it is reused).  A write wave holds 4 scans, a
    reader wave 2 pairs.  So each step below needs the device-side wait named beside it; without it the step would read or overwrite a
    slot before the wave in flight on another lane is done with it:
      write 1, wave 0 (slots 0..3)     WAR: waits for A's last three waves' copy-in of slot 0;
      B, wave 0 (slot 15)              RAW: waits for write 1's wave 3 (slots 12..15) to copy slot 15 out;
      write 2, wave 0 (slots 15..12)   WAR: waits for B's last three waves' copy-in of slot 15;
      write 3, wave 0 (slots 0..3)     WAW: waits for write 2's wave 3 (slots 3..0), a wave of the call before;
      C, wave 0 (slot 15)              RAW: waits for write 3's wave 3 (slots 12..15).
    The writes' scans are device-resident and the readers span ten waves each, so a missing RAW wait lets a reader's copy-in overtake
    the front end of the write it must follow.  Write 3's scans have 400 points, so its front end is far shorter than write 2's: without
    the WAW wait its first wave's copy-out would land before that of write 2's last wave, queued just before it on another lane.  A
    missing WAR wait cannot be made to show this way: a write's copy-out follows its own front end, which outlasts the copy-ins of the
    reader waves queued before it."""
    W = 4 * SLOTS * LANES // 2               # 16 scans in 4 waves
    assert N >= 2 * SLOTS * LANES and W == 4 * 2 * SLOTS
    read_0 = [(0, t) for t in range(W, W + N)]
    read_15 = [(15, t) for t in range(W, W + N)]  # slots W .. W + N - 1 are never written here
    writes = [(scans[2 * N:2 * N + W], list(range(W))),                          # 1: slot 15 in the last wave
              (scans[2 * N + 3:2 * N + 3 + W], list(range(W))[::-1]),            # 2: slot 15 in the first wave, slots 3..0 in the last
              ([sc[:400] for sc in scans[20:20 + W]], list(range(W)))]          # 3: slots 0..3 first, slot 15 last; small scans
    raw_pairs = [(scans[2 * i], scans[2 * i + 1]) for i in range(N)]
    sets = [tuple(a[:L] for a in synth.matched_pairs(800 + i, L, inlier_ratio=0.35, noise=0.03)[:2])
            for i, L in enumerate([40, 300, 1200, 2500] * (N // 4) + [700] * (N % 4))]
    set_p = [make_params(noise_bound=0.5)] * N
    for h in (h4, ref):
        h.cache_reserve(2 * N)
        h.cache_scans(scans[:2 * N], list(range(2 * N)), BASE)
    dev = [device_copies(w[0]) for w in writes]

    # blocking, in order
    want = {"raw": ref.register_batch_mixed(raw_pairs, [BASE] * N)[0], "A": ref.register_cached(read_0, BASE)}
    ref.cache_scans(dev[0][0], writes[0][1], BASE, MEM_DEVICE)
    want["B"] = ref.register_cached(read_15, BASE)
    ref.cache_scans(dev[1][0], writes[1][1], BASE, MEM_DEVICE)
    ref.cache_scans(dev[2][0], writes[2][1], BASE, MEM_DEVICE)
    want["C"] = ref.register_cached(read_15, BASE)
    want["sets"] = ref.solve_batch_each(sets, set_p)[0]
    assert len({want[k].tobytes() for k in "ABC"}) == 3

    # streamed
    out = {k: np.zeros(N, RESULT_DTYPE) for k in want}
    arr_0, arr_15 = capi._slot_array(read_0), capi._slot_array(read_15)
    pa = h4.params_array([BASE] * N)
    pair_arr, keep_pairs = h4.pair_array(raw_pairs)
    set_arr, keep_sets = h4._set_array(sets, MEM_HOST)
    h4.register_batch_enqueue_mixed_raw(pair_arr, N, pa, MEM_HOST, out["raw"])
    h4.register_cached_enqueue_mixed_raw(arr_0, N, pa, out["A"])
    _enqueue(h4, dev[0][0], writes[0][1], [BASE] * W, MEM_DEVICE)       # device scans: nothing to keep
    h4.register_cached_enqueue_mixed_raw(arr_15, N, pa, out["B"])
    _enqueue(h4, dev[1][0], writes[1][1], [BASE] * W, MEM_DEVICE)
    _enqueue(h4, dev[2][0], writes[2][1], [BASE] * W, MEM_DEVICE)
    h4.register_cached_enqueue_mixed_raw(arr_15, N, pa, out["C"])
    h4.solve_batch_enqueue_each_raw(set_arr, N, h4.params_array(set_p), MEM_HOST, out["sets"])
    h4.register_batch_flush()
    for k in want:
        assert out[k].tobytes() == want[k].tobytes(), k
    for s in range(2 * N):
        assert _read(h4, s) == _read(ref, s), s


# ---- GPU 3: a keyframe ring --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("window", [2, 2 * SLOTS * LANES])
def test_keyframe_ring_streams_like_the_blocking_sequence(h1, h4, ref, scans, window):
    """Keyframe k is cached into slot k % RING and registered against the `window` keyframes before it; the ring is smaller than the
    sequence, so slots are overwritten while batches that read them are queued."""
    K, RING = 24, window + 3
    seq = scans[:K]
    entries = [FRONTS[(k // 6) % 3] for k in range(K)]
    batches = [[((k - d) % RING, k % RING) for d in range(1, min(window, k) + 1)] for k in range(K)]
    bparams = [[entries[k - d] for d in range(1, min(window, k) + 1)] for k in range(K)]
    # the pair's entry must match both slots: register keyframe k against earlier keyframes cached with the same front end
    batches = [[sp for sp, p in zip(b, ps) if p is entries[k]] for k, (b, ps) in enumerate(zip(batches, bparams))]

    def blocking(h):
        h.cache_reserve(RING)
        recs, lists = [], []
        for k in range(K):
            h.cache_scans_each([seq[k]], [k % RING], [entries[k]])
            if batches[k]:
                lb = ListBuffers(len(batches[k]), h.cfg.max_corr, MEM_HOST)
                recs.append(h.register_cached_mixed(batches[k], [entries[k]] * len(batches[k]), buffers=lb)[0].tobytes())
                lists.append(host_lists(lb.trimmed(np.frombuffer(recs[-1], RESULT_DTYPE))))
        return recs, lists

    want_recs, want_lists = blocking(ref)
    assert sum(len(b) for b in batches) >= K
    for h in (h1, h4):
        h.cache_reserve(RING)
        keep, outs = [], []
        for k in range(K):
            keep.append(_enqueue(h, [seq[k]], [k % RING], [entries[k]]))
            if batches[k]:
                sp = capi._slot_array(batches[k])
                out = np.zeros(len(sp), RESULT_DTYPE)
                lb = ListBuffers(len(sp), h.cfg.max_corr, MEM_HOST)
                h.register_cached_enqueue_mixed_raw(sp, len(sp), h.params_array([entries[k]] * len(sp)), out, lb)
                keep.append(sp)
                outs.append((out, lb))
        h.register_batch_flush()
        assert [o.tobytes() for o, _ in outs] == want_recs
        for (o, lb), want in zip(outs, want_lists):
            got = host_lists(lb.trimmed(o))
            assert [{k: v.tobytes() for k, v in d.items()} for d in got] == [{k: v.tobytes() for k, v in d.items()} for d in want]


# ---- GPU 4: signatures and rejections --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_queued_write_changes_the_signature_for_the_calls_after_it(h4, ref, scans):
    lib = h4.lib
    n = 2 * SLOTS * LANES + 1
    for h in (h4, ref):
        h.cache_reserve(2 * N)
        h.cache_scans(scans[:2 * N], list(range(2 * N)), BASE)
        h.cache_scans([scans[2 * N]], [0], FRONTS[1])
    reader = [(1, 0)] * n                    # slot 1 is rewritten with FRONTS[1] by the queued write below
    ref.cache_scans([scans[2 * N + 1]], [1], FRONTS[1])
    want = ref.register_cached_mixed(reader, [FRONTS[1]] * n)[0]
    sp = capi._slot_array(reader)
    out = np.zeros(n, RESULT_DTYPE)
    keep = _enqueue(h4, [scans[2 * N + 1]], [1], [FRONTS[1]])
    assert lib.qb200_register_cached_enqueue_mixed(h4.h, capi._ptr(sp), n, h4.params_array([BASE] * n), capi._ptr(out), None) == -1
    assert "slot 1" in lib.qb200_last_error(h4.h).decode()
    h4.register_cached_enqueue_mixed_raw(sp, n, h4.params_array([FRONTS[1]] * n), out)
    h4.register_batch_flush()
    assert out.tobytes() == want.tobytes()
    del keep


@pytest.mark.gpu
def test_a_rejected_write_writes_nothing_and_keeps_the_queue(h4, scans):
    lib = h4.lib
    n = 2 * SLOTS * LANES + 1
    h4.cache_reserve(2 * N)
    h4.cache_scans(scans[:2 * N], list(range(2 * N)), BASE)
    before = [_read(h4, s) for s in range(2 * N)]
    good_slots = capi._slot_array([(2 * i, 2 * i + 1) for i in range(n)])
    good_params = h4.params_array([BASE] * n)
    want_cached = h4.register_cached([(2 * i, 2 * i + 1) for i in range(n)], BASE)
    sets = [tuple(a[:L] for a in synth.matched_pairs(900 + i, L, inlier_ratio=0.35, noise=0.03)[:2]) for i, L in enumerate([300] * n)]
    set_arr, keep_sets = h4._set_array(sets, MEM_HOST)
    want_sets = h4.solve_batch_each(sets, [BASE] * n)[0]
    new = scans[2 * N:2 * N + 6]
    ptrs, cnts, keep = capi._scan_arrays(new, MEM_HOST)
    big = (C.c_int32 * 6)(*[len(s) for s in new])
    big[4] = RAW_CAP + 1

    def write(slots, params, p=ptrs, c=cnts):
        ids = (C.c_int32 * 6)(*slots)
        return lib.qb200_cache_scans_enqueue_each(h4.h, p, c, ids, 6, params, MEM_HOST)

    fresh = [FRONTS[1]] * 6                   # would change the signature of every slot it names
    cases = {
        "slot outside": (lambda: write([0, 2, 4, 2 * N, 6, 8], h4.params_array(fresh)), "scan 3"),
        "negative slot": (lambda: write([0, -1, 4, 5, 6, 8], h4.params_array(fresh)), "scan 1"),
        "bad entry": (lambda: write([0, 2, 4, 5, 6, 8], h4.params_array(fresh[:2] + [make_params(voxel_size=0.0)] + fresh[3:])), "entry 2"),
        "beyond max_raw_points": (lambda: write([0, 2, 4, 5, 6, 8], h4.params_array(fresh), c=big), "scan 4"),
        "null scans": (lambda: write([0, 2, 4, 5, 6, 8], h4.params_array(fresh), p=None), "null"),
        "null params": (lambda: write([0, 2, 4, 5, 6, 8], None), "entry 0"),
    }
    for name, (call, why) in cases.items():
        out1, out2, out3 = np.zeros(n, RESULT_DTYPE), np.zeros(n, RESULT_DTYPE), np.zeros(n, RESULT_DTYPE)
        assert lib.qb200_register_cached_enqueue_mixed(h4.h, capi._ptr(good_slots), n, good_params, capi._ptr(out1), None) == 0
        assert call() == -1, name
        assert why in lib.qb200_last_error(h4.h).decode(), (name, lib.qb200_last_error(h4.h).decode())
        # the signatures are unchanged: a batch with the old entry is still accepted
        assert lib.qb200_solve_batch_enqueue_each(h4.h, set_arr, n, good_params, MEM_HOST, capi._ptr(out2), None) == 0
        h4.register_cached_enqueue_mixed_raw(good_slots, n, good_params, out3)
        h4.register_batch_flush()
        assert out1.tobytes() == want_cached.tobytes() == out3.tobytes(), name
        assert out2.tobytes() == want_sets.tobytes(), name
        assert [_read(h4, s) for s in range(2 * N)] == before, name


@pytest.mark.gpu
def test_a_slot_named_twice_in_one_call_ends_like_the_blocking_call(h4, ref, scans):
    """Slot 0 twice in one wave, slot 1 in the first and the last wave: each ends with the last scan that names it."""
    new = scans[2 * N:2 * N + 10]
    slots = [0, 0, 2, 1, 3, 4, 5, 6, 1, 7]
    entries = [FRONTS[i % 3] for i in range(10)]
    for h in (h4, ref):
        h.cache_reserve(8)
    ref.cache_scans_each(new, slots, entries)
    want = [_read(ref, s) for s in range(8)]
    for s, i in ((0, 1), (1, 8)):
        ref.cache_scans_each([new[i]], [s], [entries[i]])
        assert _read(ref, s) == want[s]
    keep = _enqueue(h4, new, slots, entries)
    h4.register_batch_flush()
    assert [_read(h4, s) for s in range(8)] == want
    # the signature is the last entry's too
    assert len(h4.register_cached_mixed([(1, 1)], [entries[8]])[0]) == 1
    with pytest.raises(capi.QuatroB200Error):
        h4.register_cached_mixed([(1, 1)], [entries[3]])
    del keep


# ---- GPU 5: the calls that flush first -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_cache_read_copy_and_reserve_see_the_queued_writes(h4, ref, scans):
    n = 2 * SLOTS * LANES + 1
    new = scans[2 * N:2 * N + n]
    ref.cache_reserve(n + 1)
    ref.cache_scans(new, list(range(n)), BASE)
    want = [_read(ref, s) for s in range(n)]
    h4.cache_reserve(n + 1)
    h4.cache_scans(scans[:n], list(range(n)), BASE)
    keep = [_enqueue(h4, new, list(range(n)), [BASE] * n)]
    assert [_read(h4, s) for s in range(n)] == want                # qb200_cache_read
    keep.append(_enqueue(h4, new[::-1], list(range(n)), [BASE] * n))
    h4.cache_copy(0, n)                                             # qb200_cache_copy of the second write's slot 0
    assert _read(h4, n) == want[n - 1]
    out = np.zeros(n, RESULT_DTYPE)
    sp = capi._slot_array([(0, s) for s in range(1, n)] + [(0, 0)])
    h4.register_cached_enqueue_mixed_raw(sp, n, h4.params_array([BASE] * n), out)
    keep.append(_enqueue(h4, scans[:n], list(range(n)), [BASE] * n))
    h4.cache_reserve(n + 1)                                         # qb200_cache_reserve: the queue completes before the cache goes
    ref.cache_scans(new[::-1], list(range(n)), BASE)
    assert out.tobytes() == ref.register_cached(capi._slot_array([(0, s) for s in range(1, n)] + [(0, 0)]), BASE).tobytes()
    assert all(len(h4.cache_read(s)[0]) == 0 for s in range(n + 1))
