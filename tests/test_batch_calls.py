"""Every batch entry point (raw scan pairs, cached slot pairs, correspondence sets; plain, _ex, _each and _enqueue forms) is one call
description checked by one function and run by one wave driver (csrc/api.cu: check_call, enqueue_call).  So the three inputs agree on
empty calls (no rotation noise bound is latched), on the memory kinds they accept, and on naming every rejected argument in
qb200_last_error; qb200_solve_correspondences is a qb200_solve_batch of one set."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import MEM_DEVICE, MEM_HOST, PMC_EXACT, INLIER_NONE, RESULT_DTYPE, Handle, default_params
from support import sentinel

CSRC = Path(__file__).resolve().parent.parent / "quatro_b200" / "csrc"
DELETED = ("run_waves", "solve_batch_impl", "enqueue_impl", "register_batch_impl", "register_cached_impl", "device_array_ok",
           "cache_write", "describe_call", "describe_points_call", "feature_call", "match_call")


def _sources():
    return {p.name: p.read_text() for p in sorted(CSRC.iterdir()) if p.suffix in (".cu", ".cuh")}


# ---- CPU: one checked call, one driver ----------------------------------------------------------------------------------------------
def test_per_input_drivers_and_validators_are_gone():
    found = [f"{name}: {d}" for name, text in _sources().items() for d in DELETED if re.search(rf"\b{d}\b", text)]
    assert not found, "\n".join(found)


def test_batch_call_names_its_source_and_sink():
    """A call says what it reads and what it produces in two fields, not in flags beside its input pointers."""
    body = re.search(r"struct BatchCall \{(.*?)\n\};", _sources()["api.cu"], re.S).group(1)
    code = re.sub(r"//[^\n]*", "", body)
    assert re.search(r"\bSource src\b", code) and re.search(r"\bSink sink\b", code), code
    assert not re.findall(r"\b(describe|points|match)\s*[=;,]", code), code


def test_one_wave_submit_call_site_and_one_pointer_query():
    text = "".join(_sources().values())
    calls = re.findall(r"(?<!int )\bwave_submit\(", text)
    assert len(calls) == 1, calls
    assert len(re.findall(r"\bcudaPointerGetAttributes\(", text)) == 1


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------
def _params(noise_bound, **kw):
    p = default_params()
    p.noise_bound, p.rot_noise_bound = noise_bound, 0.0
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _bound_sensitive_set():
    """a set whose record depends on the rotation noise bound: noisy inliers and outliers"""
    a4, b4, _, _ = synth.matched_pairs(4242, 300, inlier_ratio=0.5, noise=0.2)
    return a4, b4


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["register_batch", "register_cached", "solve_batch"])
def test_empty_call_latches_nothing(family):
    s = _bound_sensitive_set()
    wide, narrow = _params(0.9), _params(0.3)
    with Handle(max_batch_slots=2) as fresh, Handle(max_batch_slots=2) as latched, Handle(max_batch_slots=2) as h:
        want = fresh.solve_batch([s], narrow)
        latched.solve_batch([s], wide)   # latches 2 * 0.9
        assert latched.solve_batch([s], narrow).tobytes() != want.tobytes(), "the record does not depend on the latched bound"
        empty = {"register_batch": lambda: h.register_batch([], wide), "register_cached": lambda: h.register_cached([], wide),
                 "solve_batch": lambda: h.solve_batch([], wide)}[family]
        assert len(empty()) == 0
        assert h.solve_batch([s], narrow).tobytes() == want.tobytes()


@pytest.mark.gpu
def test_unknown_memory_kind_is_rejected_before_any_work():
    import torch
    src, tgt, _ = synth.outdoor_pair(5, rings=16, azimuths=400)
    a4, b4, _, _ = synth.matched_pairs(5, 64)
    dev = [torch.from_numpy(x).cuda() for x in (src, tgt, a4, b4)]
    torch.cuda.synchronize()
    p = default_params()
    with Handle(max_batch_slots=2) as h:
        h.register_batch([(src, tgt)], p)   # kernels warmed
        pairs, _ = h.pair_array([(dev[0].data_ptr(), len(src), dev[1].data_ptr(), len(tgt))], MEM_DEVICE)
        sets, _ = h._set_array([(dev[2].data_ptr(), dev[3].data_ptr(), len(a4))], MEM_DEVICE)
        lib = h.lib
        calls = {
            "register_batch": lambda n, out: lib.qb200_register_batch(h.h, pairs, n, C.byref(p), 2, capi._ptr(out)),
            "register_batch_enqueue": lambda n, out: lib.qb200_register_batch_enqueue(h.h, pairs, n, C.byref(p), 2, capi._ptr(out)),
            "solve_batch": lambda n, out: lib.qb200_solve_batch(h.h, sets, n, C.byref(p), 2, capi._ptr(out)),
        }
        for name, call in calls.items():
            for n in (0, 1):
                out = sentinel(max(n, 1), RESULT_DTYPE)
                before = h.launch_count()
                st = call(n, out)
                h.register_batch_flush()
                assert st == -1, (name, n, st)
                assert "memory kind" in lib.qb200_last_error(h.h).decode(), name
                assert h.launch_count() == before and (out.view(np.uint8) == 0xA5).all(), name


@pytest.mark.gpu
def test_every_rejection_names_its_fault():
    p = default_params()
    big = np.zeros((1025, 4), np.float32)
    with Handle(max_batch_slots=2, max_raw_points=1024) as h:
        lib = h.lib
        pairs, _ = h.pair_array([(big[:8], big[:8])])
        sets, _ = h._set_array([(big[:8], big[:8])], MEM_HOST)
        slots = np.zeros((1, 2), np.int32)
        out = np.zeros(1, RESULT_DTYPE)
        # per family: its input array and the call with (input, n, results)
        families = {
            "register_batch": (pairs, lambda x, n, res: lib.qb200_register_batch(h.h, x, n, C.byref(p), MEM_HOST, res)),
            "register_batch_enqueue": (pairs, lambda x, n, res: lib.qb200_register_batch_enqueue(h.h, x, n, C.byref(p), MEM_HOST, res)),
            "register_batch_each": (pairs, lambda x, n, res: lib.qb200_register_batch_each(h.h, x, n, h.params_array([p]), MEM_HOST, res, None)),
            "register_cached": (capi._ptr(slots), lambda x, n, res: lib.qb200_register_cached(h.h, x, n, C.byref(p), res)),
            "solve_batch": (sets, lambda x, n, res: lib.qb200_solve_batch(h.h, x, n, C.byref(p), MEM_HOST, res)),
            "solve_batch_ex": (sets, lambda x, n, res: lib.qb200_solve_batch_ex(h.h, x, n, C.byref(p), MEM_HOST, res, None)),
        }
        for name, (x, call) in families.items():
            for args, fault in (((x, -1, capi._ptr(out)), "n < 0"), ((None, 1, capi._ptr(out)), "input array is null"),
                                ((x, 1, None), "results array is null")):
                with pytest.raises(capi.QuatroB200Error):
                    h.register_batch([(big, big[:8])], p)   # leaves a known message: the cloud exceeds max_raw_points
                known = lib.qb200_last_error(h.h).decode()
                assert "max_raw_points" in known
                st = call(*args)
                h.register_batch_flush()
                msg = lib.qb200_last_error(h.h).decode()
                assert st == -1 and msg != known and fault in msg, (name, fault, st, msg)


@pytest.mark.gpu
def test_solve_correspondences_is_a_batch_of_one():
    sizes_modes = ((0, None), (1, None), (2, None), (40, None), (700, None), (300, PMC_EXACT), (300, INLIER_NONE), (2500, None))
    with Handle(max_batch_slots=4, max_corr=4096) as h:
        for i, (L, mode) in enumerate(sizes_modes):
            a4, b4, _, _ = synth.matched_pairs(900 + i, max(L, 1), inlier_ratio=0.4, noise=0.03)
            a4, b4 = a4[:L], b4[:L]
            p = default_params()
            if mode is not None:
                p.inlier_selection_mode = mode
            h.solve_batch([(a4, b4)], p)   # warmed: the scratch of the mode allocated

            def run(fn):
                before = h.launch_count()
                rec = fn()
                return rec, h.launch_count() - before, h.last_clique().tobytes(), h.last_final_inliers().tobytes()

            (one, st), *single = run(lambda: h.solve_correspondences(a4, b4, p))
            rec, *batch = run(lambda: h.solve_batch([(a4, b4)], p))
            assert st == one.status and bytes(one) == rec.tobytes() and single == batch, (L, mode)
