"""Poses of batches of caller inlier sets: qb200_solve_pose_batch_each and its queued form.  Street sets with the cliques
qb200_solve_batch_ex lists and the adversarial families of test_pose_adversarial equal qb200_solve_pose on each set alone and the
oracle; clique sizes on both sides of the shared-memory / workspace switch up to 32768, per-set params with the latch, unsorted and
repeated ids, the chains solve_batch -> pose and match -> graph -> clique -> pose on the device, refused sets, whole-call rejections,
memory kinds, lanes and wave sizes, the shared enqueue stream and the stage times."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import (COTE_MEDIAN, COTE_WEIGHTED_MEAN, GRAPH_LISTS, MATCH_LISTS, MEM_DEVICE, MEM_HOST, RESULT_DTYPE, SET_LISTS,
                              GraphBuffers, Handle, InlierSet, ListBuffers, default_params)
from support import P4, ROOT, device_copy, host_lists, make_handle

NEW = ("qb200_solve_pose_batch_each", "qb200_solve_pose_batch_enqueue_each")
SIZES = (0, 1, 2, 31, 32, 33, 4095, 4096, 4097, 8192, 32768)
BAD_ARG = -1
LISTS_TRUNCATED = 2
SENT = 0x5A
INT32_MAX = 2 ** 31 - 1
ZERO = ("valid", "n_src_vox", "n_tgt_vox", "n_mutual", "max_core", "clique_size", "gnc_iters", "n_rot_inliers", "n_final_inliers",
        "flags", "n_edges", "cost")


# ---- CPU: layout, prototypes, the INTEGRATION.md snippet -------------------------------------------------------------------------------
def test_inlier_set_mirror_matches_the_c_layout(tmp_path):
    fields = ("a", "b", "inliers", "L", "n_inliers")
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "quatro_b200.h"\nint main(void) {\n'
                   '  printf("%zu' + " %zu" * len(fields) + '\\n", sizeof(qb200_inlier_set)' +
                   "".join(f", offsetof(qb200_inlier_set, {f})" for f in fields) + ");\n  return 0;\n}\n")
    exe = tmp_path / "layout"
    r = subprocess.run(["/usr/bin/gcc", "-std=c11", "-Wall", "-Werror", f"-I{ROOT / 'include'}", str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(InlierSet)] + [getattr(InlierSet, f).offset for f in fields]


def test_header_declares_both_entry_points(tmp_path):
    header = (ROOT / "include" / "quatro_b200.h").read_text()
    for n in NEW:
        decl = header[header.index(f"int {n}("):]
        decl = decl[:decl.index(");")]
        assert decl.count(",") + 1 == len(capi._SIGNATURES[n][1]), n
    body = "".join(f"  __typeof__(&{NEW[0]}) p{i} = {n};\n  (void)p{i};\n" for i, n in enumerate(NEW))
    (tmp_path / "proto.c").write_text('#include "quatro_b200.h"\nint main(void) {\n' + body + "  return 0;\n}\n")
    r = subprocess.run(["/usr/bin/gcc", "-std=gnu11", "-Wall", "-Werror", "-Wincompatible-pointer-types", f"-I{ROOT / 'include'}", "-c",
                        str(tmp_path / "proto.c"), "-o", str(tmp_path / "proto.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = capi.load_library()
    for n in NEW:
        assert n in capi.EXPORTED_SYMBOLS and hasattr(lib, n)


def test_a_null_handle_is_refused():
    lib = capi.load_library()
    for n in NEW:
        assert getattr(lib, n)(None, None, 0, None, MEM_HOST, None, None) == BAD_ARG, n


def test_the_integration_chain_snippet_compiles(tmp_path):
    """The match -> graph -> clique -> pose example of INTEGRATION.md, with the names it takes from the steps before it as
    parameters, compiles as C++ against the header."""
    text = (ROOT / "INTEGRATION.md").read_text()
    blocks = [b for b in re.findall(r"```cpp\n(.*?)```", text, re.S) if "qb200_solve_pose_batch_each" in b]
    assert len(blocks) == 1
    src = ("#include <vector>\n#include \"quatro_b200.h\"\n"
           "void chain(qb200_handle* h, float* d_sm, float* d_tm, int32_t cap, int n_pairs, const std::vector<qb200_result>& rec,\n"
           "           const std::vector<qb200_params>& ps, int32_t* d_clique, const std::vector<qb200_result>& crec,\n"
           "           const double (*RyRx)[9]) {\n" + blocks[0] + "}\n")
    (tmp_path / "chain.cpp").write_text(src)
    r = subprocess.run(["/usr/bin/g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", f"-I{ROOT / 'include'}", "-fsyntax-only",
                        str(tmp_path / "chain.cpp")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


# ---- sets and what they must give ------------------------------------------------------------------------------------------------------
def pose_params(**kw):
    """Default params with rot_noise_bound explicit unless given (0 latches on the handle)."""
    p = default_params()
    p.rot_noise_bound = 0.6
    for k, v in kw.items():
        if k == "RyRx":
            p.use_pre_estimated_RyRx = 1
            for i, e in enumerate(np.asarray(v, float).ravel()):
                p.RyRx[i] = float(e)
        else:
            setattr(p, k, v)
    return p


def scene(seed, c, L=None):
    """(a4, b4, ids): a random street-scale set of L points (30 % outliers) and an ascending c-subset of its ids"""
    from test_pose_adversarial import _scene
    if c < 2:
        rng = np.random.default_rng(seed)
        L = c + 3 if L is None else L
        a = rng.uniform(-20, 20, (L, 3))
        return P4(a), P4(a + [1.0, -2.0, 0.5]), np.sort(rng.choice(L, c, replace=False)).astype(np.int32)
    a4, b4, ids = _scene(seed, c, L=L or c + c // 7 + 1)
    return a4, b4, ids.astype(np.int32)


def single(h, a4, b4, ids, p):
    """qb200_solve_pose on one set: (record bytes, rotation mask, translation mask, final inliers)"""
    res, rm, tm, _ = h.solve_pose(a4, b4, ids, p)
    return bytes(res), rm.copy(), tm.copy(), h.last_final_inliers()


def check_set(rec, lists, want, ids, cap, label):
    """one set of the batch (record, its trimmed lists) against qb200_solve_pose's outputs on it, lists clipped to cap"""
    res, rm, tm, fin = want
    w = np.frombuffer(res, RESULT_DTYPE)[0].copy()
    clipped = w["clique_size"] > cap or w["n_final_inliers"] > cap
    w["flags"] |= LISTS_TRUNCATED if clipped else 0
    assert rec.tobytes() == w.tobytes(), (label, rec, w)
    mq, mf = min(int(w["clique_size"]), cap), min(int(w["n_final_inliers"]), cap)
    assert lists["clique"].tobytes() == np.asarray(ids, np.int32)[:mq].tobytes(), label
    assert lists["rot_inlier_mask"].tobytes() == rm[:mq].tobytes(), label
    assert lists["trans_inlier_mask"].tobytes() == tm[:mq].tobytes(), label
    assert lists["final_inliers"].tobytes() == fin[:mf].tobytes(), label


def sentinel_lists(n, cap, kind=MEM_HOST, names=SET_LISTS):
    lb = ListBuffers(n, cap, kind, names)
    for a in lb.arrays.values():
        if kind == MEM_HOST:
            a.view(np.uint8)[...] = SENT
        else:
            import torch
            a.view(torch.uint8).fill_(SENT)
    return lb


def untouched(lb, i):
    return all((lb.host(n)[i].view(np.uint8) == SENT).all() for n in lb.arrays)


def device_sets(sets, inliers):
    """the same sets and ids in device memory: (sets, inliers as the call takes them, the tensors that hold them)"""
    keep = [(device_copy(a), device_copy(b), device_copy(np.asarray(i, np.int32).reshape(-1) if len(i) else np.zeros(1, np.int32)))
            for (a, b), i in zip(sets, inliers)]
    return ([(ta.data_ptr(), tb.data_ptr(), len(a)) for (ta, tb, _), (a, _) in zip(keep, sets)],
            [(ti.data_ptr() if len(i) else None, len(i)) for (_, _, ti), i in zip(keep, inliers)], keep)


def street_sets(h, seeds, p):
    """matched sets of street pairs and the cliques qb200_solve_batch_ex lists for them with p"""
    from test_graph_batch import street_sets as matched
    sets = matched(h, seeds)
    _, lists = h.solve_batch_lists(sets, p)
    return sets, [l["clique"] for l in lists]


# ---- GPU 1: a mixed batch equals the single call and the oracle ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mixed():
    """(sets, inliers, params, oracle-comparable): street sets with their solve_batch cliques and the adversarial cases of at most
    8192 points, each with its own COTE mode, rotation-inlier, RyRx and GNC knobs"""
    from test_pose_adversarial import CASES, ILL_CONDITIONED, case
    sets, inliers, params, cmp = [], [], [], []
    sp = pose_params()
    with Handle(max_batch_slots=8) as h:
        ss, cl = street_sets(h, range(2500, 2506), sp)
    for s, c in zip(ss, cl):
        sets.append(s), inliers.append(c), params.append(sp), cmp.append(True)
    for i, name in enumerate(CASES):
        a4, b4, clique, p, g = case(name, "median" if i % 2 else "mean")
        if len(a4) > 8192:
            continue
        sets.append((a4, b4)), inliers.append(clique), params.append(p)
        cmp.append(g["dev"]["safe"] and g["ora"]["safe"] and name not in ILL_CONDITIONED and not name.startswith("cote_far"))
    return sets, inliers, params, cmp


@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 4])
def test_mixed_batch_equals_single_calls_and_the_oracle(mixed, oracle, lanes):
    sets, inliers, params, cmp = mixed
    h = make_handle(lanes, max_batch_slots=8, max_corr=8192)
    try:
        assert len(sets) > 3 * 8 and any(len(i) > 4096 for i in inliers)
        recs, lists = h.solve_pose_batch_each(sets, inliers, params, buffers=ListBuffers(len(sets), 8192, MEM_HOST, SET_LISTS))
        for i, ((a4, b4), ids, p) in enumerate(zip(sets, inliers, params)):
            want = single(h, a4, b4, ids, p)
            check_set(recs[i], lists[i], want, ids, 8192, (lanes, i))
            if not cmp[i]:
                continue
            ro, rmo, tmo, st, fin = oracle.solve_pose(a4, b4, ids, p, want_final=True)
            r = recs[i]
            assert (r["status"], r["valid"], r["gnc_iters"], r["n_rot_inliers"], r["n_final_inliers"]) == \
                (st, ro.valid, ro.gnc_iters, ro.n_rot_inliers, ro.n_final_inliers), i
            assert np.allclose(np.asarray(r["T"]), np.asarray(ro.T[:]), atol=1e-9, rtol=0), i
            assert lists[i]["rot_inlier_mask"].tobytes() == rmo.tobytes() and lists[i]["trans_inlier_mask"].tobytes() == tmo.tobytes(), i
            assert lists[i]["final_inliers"].tobytes() == fin.tobytes(), i
    finally:
        h.close()


# ---- GPU 2: clique sizes across the shared-memory / workspace switch ------------------------------------------------------------------
@pytest.mark.gpu
def test_clique_sizes_up_to_32768_members():
    sets, inliers = [], []
    for k, c in enumerate(SIZES):
        a4, b4, ids = scene(300 + k, c, L=min(c + c // 7 + 1, 32768) if c >= 2 else None)
        sets.append((a4, b4)), inliers.append(ids)
    for L in (0, 1):   # fewer than two correspondences: DEGENERATE_INPUT
        a4, b4, ids = scene(310 + L, L, L=L)
        sets.append((a4, b4)), inliers.append(ids)
    params = [pose_params(cote_mode=(COTE_MEDIAN, COTE_WEIGHTED_MEAN)[k % 2]) for k in range(len(sets))]
    with Handle(max_batch_slots=2, max_corr=32768) as h:   # two slots: about 0.5 GB of adjacency
        want = [single(h, a, b, i, p) for (a, b), i, p in zip(sets, inliers, params)]
        statuses = [np.frombuffer(w[0], RESULT_DTYPE)[0]["status"] for w in want]
        assert statuses[:2] == [1, 1] and statuses[-2:] == [2, 2] and all(s == 0 for s in statuses[2:-2]), statuses
        dsets, dids, keep = device_sets(sets, inliers)
        for kind, ss, ii in ((MEM_HOST, sets, inliers), (MEM_DEVICE, dsets, dids)):
            recs, lists = h.solve_pose_batch_each(ss, ii, params, kind, ListBuffers(len(sets), 32768, MEM_HOST, SET_LISTS))
            for i, ids in enumerate(inliers):
                check_set(recs[i], lists[i], want[i], ids, 32768, (kind, SIZES[i] if i < len(SIZES) else "L<2"))
        del keep


# ---- GPU 3: per-set params in one batch, the latch in set order ---------------------------------------------------------------------
@pytest.mark.gpu
def test_per_set_params_and_the_latch_follow_set_order():
    from test_pose_adversarial import _Ry
    base = [scene(400 + k, c) for k, c in enumerate((300, 120, 700, 64, 450, 900, 33, 250, 500, 180))]
    knobs = [dict(rot_noise_bound=0.0, noise_bound=0.2), dict(cote_mode=COTE_WEIGHTED_MEAN), dict(using_rot_inliers_when_estimating_cote=1),
             dict(RyRx=_Ry(3.0)), dict(rotation_max_iterations=3), dict(rot_noise_bound=0.0, noise_bound=0.45),
             dict(rot_noise_bound=0.2, cote_noise_bound=0.5), dict(RyRx=_Ry(-2.0), using_rot_inliers_when_estimating_cote=1,
                                                                    cote_mode=COTE_WEIGHTED_MEAN),
             dict(rot_noise_bound=0.0, rotation_gnc_factor=1.2), dict(rotation_cost_threshold=1e-6, cbar2=2.0)]
    params = [pose_params(**kw) for kw in knobs]
    sets, inliers = [(a, b) for a, b, _ in base], [i for _, _, i in base]
    with Handle(max_batch_slots=4) as seq:
        want = [single(seq, a, b, i, p) for (a, b), i, p in zip(sets, inliers, params)]
    with make_handle(4, max_batch_slots=4) as h:
        recs, lists = h.solve_pose_batch_each(sets, inliers, params, buffers=ListBuffers(len(sets), 1024, MEM_HOST, SET_LISTS))
        for i, ids in enumerate(inliers):
            check_set(recs[i], lists[i], want[i], ids, 1024, i)
    # the latch is 2 x 0.2 from the first zero entry, not 2 x 0.45 of the sixth: a different latch changes the pose of set 5
    with Handle(max_batch_slots=4) as other:
        q = pose_params(rot_noise_bound=0.0, noise_bound=0.45)
        alone = single(other, *sets[5], inliers[5], q)
    assert alone[0] != want[5][0]


# ---- GPU 4: unsorted lists and repeated ids ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_unsorted_lists_and_repeated_ids_equal_the_single_call(handle):
    rng = np.random.default_rng(44)
    sets, inliers = [], []
    for k, c in enumerate((200, 50, 600, 33)):
        a4, b4, ids = scene(440 + k, c)
        sets += [(a4, b4)] * 3
        inliers += [ids, rng.permutation(ids), np.concatenate([ids[:c // 2], ids[c // 4:c // 2], ids[[0, 0, 0]]])[:len(a4)]]
    params = [pose_params()] * len(sets)
    recs, lists = handle.solve_pose_batch_each(sets, inliers, params, buffers=ListBuffers(len(sets), 1024, MEM_HOST, SET_LISTS))
    for i, ((a4, b4), ids) in enumerate(zip(sets, inliers)):
        check_set(recs[i], lists[i], single(handle, a4, b4, ids, params[i]), ids, 1024, i)


# ---- GPU 5: chains --------------------------------------------------------------------------------------------------------------------
POSE_FIELDS = ("valid", "status", "n_corr", "clique_size", "gnc_iters", "n_rot_inliers", "n_final_inliers", "cost", "T")


@pytest.mark.gpu
def test_solve_batch_cliques_fed_back_reproduce_it(handle):
    p = pose_params(rot_noise_bound=0.0)   # the handle's latch, as the solve batch resolved it
    sets = [synth.matched_pairs(s, L)[:2] for s, L in zip(range(450, 462), (300, 40, 1000, 2, 700, 64, 1500, 120, 33, 900, 3, 400))]
    want, wl = handle.solve_batch_lists(sets, p)
    for kind in (MEM_HOST, MEM_DEVICE):
        cliques = [l["clique"] for l in wl]
        ss, ii, keep = (sets, cliques, None) if kind == MEM_HOST else device_sets(sets, cliques)
        got, gl = handle.solve_pose_batch_each(ss, ii, [p] * len(sets), kind, ListBuffers(len(sets), handle.cfg.max_corr, MEM_HOST, SET_LISTS))
        for i in range(len(sets)):
            for k in POSE_FIELDS:
                assert np.asarray(got[i][k]).tobytes() == np.asarray(want[i][k]).tobytes(), (kind, i, k)
            for n in SET_LISTS:
                assert gl[i][n].tobytes() == wl[i][n].tobytes(), (kind, i, n)


@pytest.mark.gpu
def test_match_graph_clique_pose_on_the_device_equals_register(handle):
    import torch
    pairs = [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(2600, 2606)]
    n, cap = len(pairs), handle.cfg.max_corr
    p = default_params()
    p.rot_noise_bound = 0.6
    ml = ListBuffers(n, cap, MEM_DEVICE, MATCH_LISTS)
    mrec, _ = handle.match_batch_mixed(pairs, [p] * n, buffers=ml)
    sa, sb = ml.arrays["src_matched4"], ml.arrays["tgt_matched4"]
    sets = [(sa[i].data_ptr(), sb[i].data_ptr(), int(mrec[i]["n_corr"])) for i in range(n)]
    m = int(mrec["n_corr"].max())
    gb = GraphBuffers(n, m, (m + 31) // 32, 1, MEM_DEVICE, ("adj",))
    grec = handle.build_graph_batch_each(sets, [p] * n, MEM_DEVICE, gb)
    cl = ListBuffers(n, cap, MEM_DEVICE, GRAPH_LISTS)
    crec, _ = handle.max_clique_batch_each(gb.graphs(grec, "adj"), [p] * n, MEM_DEVICE, buffers=cl)
    d_clique = cl.arrays["clique"]
    ids = [(d_clique[i].data_ptr(), int(crec[i]["clique_size"])) for i in range(n)]
    got, gl = handle.solve_pose_batch_each(sets, ids, [p] * n, MEM_DEVICE, ListBuffers(n, cap, MEM_DEVICE, SET_LISTS))
    want, wl = handle.register_batch_mixed(pairs, [p] * n, buffers=ListBuffers(n, cap, MEM_HOST, SET_LISTS))
    gl = host_lists(gl)
    assert (want["valid"] == 1).sum() >= n // 2
    for i in range(n):
        for k in ("T", "cost", "gnc_iters", "n_rot_inliers", "n_final_inliers", "clique_size", "status", "valid"):
            assert np.asarray(got[i][k]).tobytes() == np.asarray(want[i][k]).tobytes(), (i, k)
        for name in SET_LISTS:
            assert gl[i][name].tobytes() == wl[i][name].tobytes(), (i, name)
    torch.cuda.synchronize()


# ---- GPU 6: refused sets ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", [MEM_HOST, MEM_DEVICE])
def test_out_of_range_ids_refuse_only_their_set(kind):
    good = [scene(460 + k, c) for k, c in enumerate((300, 64, 500, 120, 33))]
    sets = [(a, b) for a, b, _ in good]
    ids = [i for _, _, i in good]
    params = [pose_params(cote_mode=(COTE_MEDIAN, COTE_WEIGHTED_MEAN)[k % 2]) for k in range(5)]
    with Handle(max_batch_slots=4) as h:
        ref_lb = sentinel_lists(4, 1024)
        ref, _ = h.solve_pose_batch_each(sets[:1] + sets[2:], ids[:1] + ids[2:], params[:1] + params[2:], buffers=ref_lb)
        L = len(sets[1][0])
        for bad in (-1, L, INT32_MAX):
            for pos in (0, len(ids[1]) - 1):
                b_ids = ids[1].copy()
                b_ids[pos] = bad
                ii = ids[:1] + [b_ids] + ids[2:]
                ss, dd, keep = (sets, ii, None) if kind == MEM_HOST else device_sets(sets, ii)
                lb = sentinel_lists(5, 1024)
                recs, _ = h.solve_pose_batch_each(ss, dd, params, kind, lb)
                r = recs[1]
                assert r["status"] == BAD_ARG and r["n_corr"] == L, (bad, pos, r)
                for k in ZERO:
                    assert r[k] == 0, (bad, pos, k)
                assert np.array_equal(np.asarray(r["T"]), np.eye(4).reshape(-1))
                assert untouched(lb, 1), (bad, pos)
                for j, jr in ((0, 0), (2, 1), (3, 2), (4, 3)):   # the neighbours: as in the batch without the refused set
                    assert recs[j].tobytes() == ref[jr].tobytes(), (bad, pos, j)
                    for n in SET_LISTS:
                        assert lb.host(n)[j].tobytes() == ref_lb.host(n)[jr].tobytes(), (bad, pos, j, n)


# ---- GPU 7: whole-call rejections ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rejections_write_nothing_and_name_the_set(handle):
    import torch
    a4, b4, ids = scene(470, 40)
    ta, tb, ti = device_copy(a4), device_copy(b4), device_copy(ids)
    p = pose_params()
    bad_p = pose_params(cote_noise_bound=0.0)
    lb = sentinel_lists(2, 64)

    def arr(*sets):
        out = (InlierSet * max(len(sets), 1))()
        for i, s in enumerate(sets):
            out[i] = InlierSet(*s)
        return out

    ok = (a4.ctypes.data, b4.ctypes.data, ids.ctypes.data, len(a4), len(ids))
    dok = (ta.data_ptr(), tb.data_ptr(), ti.data_ptr(), len(a4), len(ids))
    lists_with_corr = lb.descriptor()
    lists_with_corr.corr = lb.arrays["clique"].ctypes.data
    lists_cap0 = lb.descriptor()
    lists_cap0.cap_per_pair = 0
    cases = [   # (what the error names, sets, n, params, kind, results?, lists)
        ("n < 0", arr(ok), -1, [p], MEM_HOST, True, lb.descriptor()),
        ("set 1: its L is outside", arr(ok, (*ok[:3], -1, 0)), 2, [p, p], MEM_HOST, True, lb.descriptor()),
        ("set 0: its L is outside", arr((*ok[:3], handle.cfg.max_corr + 1, 0)), 1, [p], MEM_HOST, True, lb.descriptor()),
        ("set 1: its n_inliers", arr(ok, (*ok[:4], -1)), 2, [p, p], MEM_HOST, True, lb.descriptor()),
        ("set 1: its n_inliers", arr(ok, (*ok[:4], len(a4) + 1)), 2, [p, p], MEM_HOST, True, lb.descriptor()),
        ("set 0: its points are null", arr((None, ok[1], ok[2], len(a4), len(ids))), 1, [p], MEM_HOST, True, lb.descriptor()),
        ("set 1: its inlier list is null", arr(ok, (ok[0], ok[1], None, len(a4), 3)), 2, [p, p], MEM_HOST, True, lb.descriptor()),
        ("results array is null", arr(ok), 1, [p], MEM_HOST, False, lb.descriptor()),
        ("unknown memory kind of the inputs", arr(ok), 1, [p], 3, True, lb.descriptor()),
        ("params entry 1", arr(ok, ok), 2, [p, bad_p], MEM_HOST, True, lb.descriptor()),
        ("no corr / matched points", arr(ok), 1, [p], MEM_HOST, True, lists_with_corr),
        ("cap_per_pair", arr(ok), 1, [p], MEM_HOST, True, lists_cap0),
        ("set 0: its points are misaligned", arr(ok), 1, [p], MEM_DEVICE, True, lb.descriptor()),
        ("set 1: its points are misaligned", arr(dok, (dok[0] + 4, *dok[1:])), 2, [p, p], MEM_DEVICE, True, lb.descriptor()),
        ("set 0: its inlier list is misaligned", arr((*dok[:2], dok[2] + 2, *dok[3:])), 1, [p], MEM_DEVICE, True, lb.descriptor()),
        ("set 0: its inlier list is misaligned", arr((*dok[:2], ids.ctypes.data, *dok[3:])), 1, [p], MEM_DEVICE, True, lb.descriptor()),
    ]
    # a queued batch before the rejected calls still completes on the flush
    qsets = [scene(471 + k, c) for k, c in enumerate((50, 300, 7))]
    qs, qi = [(a, b) for a, b, _ in qsets], [i for _, _, i in qsets]
    want, wl = handle.solve_pose_batch_each(qs, qi, [p] * 3, buffers=ListBuffers(3, 512, MEM_HOST, SET_LISTS))
    qrec = np.zeros(3, RESULT_DTYPE)
    qlb = ListBuffers(3, 512, MEM_HOST, SET_LISTS)
    qarr, qkeep = handle.inlier_array(qs, qi, MEM_HOST)
    qpa = handle.params_array([p] * 3)
    handle.solve_pose_batch_enqueue_each_raw(qarr, 3, qpa, MEM_HOST, qrec, qlb)
    lib = handle.lib
    for why, sets, n, ps, kind, with_results, d in cases:
        rec = np.zeros(max(n, 1), RESULT_DTYPE)
        rec.view(np.uint8)[...] = 0xA5
        for fn in NEW[::-1]:
            rc = getattr(lib, fn)(handle.h, sets, n, handle.params_array(ps), kind, rec.ctypes.data if with_results else None, C.byref(d))
            assert rc == BAD_ARG, (why, fn)
            assert why in lib.qb200_last_error(handle.h).decode(), (why, lib.qb200_last_error(handle.h))
            assert (rec.view(np.uint8) == 0xA5).all(), why
            assert untouched(lb, 0) and untouched(lb, 1), why
    handle.register_batch_flush()
    assert qrec.tobytes() == want.tobytes()
    for i, l in enumerate(qlb.trimmed(qrec)):
        for n in SET_LISTS:
            assert l[n].tobytes() == wl[i][n].tobytes(), (i, n)
    torch.cuda.synchronize()
    del ta, tb, ti


# ---- GPU 8: memory kinds, clipped lists, lanes and wave sizes -----------------------------------------------------------------------
@pytest.fixture(scope="module")
def wave_sets():
    """3 x 4 + 5 sets of mixed sizes and params, and what qb200_solve_pose gives for each"""
    rng = np.random.default_rng(48)
    base = [scene(480 + k, int(c)) for k, c in enumerate(rng.choice([0, 1, 2, 33, 120, 300, 650, 1000], 17))]
    sets, inliers = [(a, b) for a, b, _ in base], [i for _, _, i in base]
    params = [pose_params(cote_mode=(COTE_MEDIAN, COTE_WEIGHTED_MEAN)[k % 2], using_rot_inliers_when_estimating_cote=k % 3 == 0)
              for k in range(len(sets))]
    with Handle(max_batch_slots=4) as h:
        want = [single(h, a, b, i, p) for (a, b), i, p in zip(sets, inliers, params)]
    return sets, inliers, params, want


@pytest.mark.gpu
def test_memory_kinds_and_clipped_lists_give_the_same_bytes(wave_sets):
    sets, inliers, params, want = wave_sets
    dsets, dids, keep = device_sets(sets, inliers)
    sizes = sorted(np.frombuffer(w[0], RESULT_DTYPE)[0]["clique_size"] for w in want)
    with Handle(max_batch_slots=4) as h:
        for cap in (max(sizes) + 5, int(sizes[len(sizes) // 2])):
            for kind, ss, ii in ((MEM_HOST, sets, inliers), (MEM_DEVICE, dsets, dids)):
                for dest in (MEM_HOST, MEM_DEVICE):
                    lb = ListBuffers(len(sets), cap, dest, SET_LISTS)
                    recs, lists = h.solve_pose_batch_each(ss, ii, params, kind, lb)
                    lists = host_lists(lists)
                    for i, ids in enumerate(inliers):
                        check_set(recs[i], lists[i], want[i], ids, cap, (cap, kind, dest, i))
    del keep


@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 4])
def test_lanes_and_wave_sizes(wave_sets, lanes):
    sets, inliers, params, want = wave_sets
    S = 4
    h = make_handle(lanes, max_batch_slots=S)
    try:
        for n in (S - 1, S, S + 1, 3 * S + 5):
            recs, lists = h.solve_pose_batch_each(sets[:n], inliers[:n], params[:n], buffers=ListBuffers(n, 1024, MEM_HOST, SET_LISTS))
            for i in range(n):
                check_set(recs[i], lists[i], want[i], inliers[i], 1024, (lanes, n, i))
    finally:
        h.close()


# ---- GPU 9: one queued stream -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_enqueue_interleaved_with_graph_and_clique_batches(handle):
    from test_graph_batch import buffers as graph_buffers, graph_params, sized_set
    rng = np.random.default_rng(49)
    gsets = [sized_set(rng, L) for L in (50, 400, 33, 900, 128)]
    gparams = [graph_params(0.3)] * len(gsets)
    cgraphs = [np.ascontiguousarray(handle.build_graph(a, b, 0.3, 1.0)[0]) for a, b in gsets]
    cparams = [default_params()] * len(cgraphs)
    base = [scene(490 + k, c) for k, c in enumerate((300, 64, 500, 2, 700, 33, 120, 250, 40, 1000, 80))]
    psets, pids = [(a, b) for a, b, _ in base], [i for _, _, i in base]
    pparams = [pose_params(cote_mode=(COTE_MEDIAN, COTE_WEIGHTED_MEAN)[k % 2]) for k in range(len(psets))]
    shape = (len(gsets), 900, 29, 50_000)
    gref_buf = graph_buffers(*shape)
    gref = handle.build_graph_batch_each(gsets, gparams, MEM_HOST, gref_buf)
    cref, cl = handle.max_clique_batch_each(cgraphs, cparams, buffers=ListBuffers(len(cgraphs), 1024, MEM_HOST, GRAPH_LISTS))
    refs = {dest: handle.solve_pose_batch_each(psets, pids, pparams, buffers=ListBuffers(len(psets), 1024, dest, SET_LISTS))
            for dest in (MEM_HOST, MEM_DEVICE)}
    ga, gkeep = handle._set_array(gsets, MEM_HOST)
    ca, ckeep = handle.graph_array(cgraphs)
    pa, pkeep = handle.inlier_array(psets, pids, MEM_HOST)
    outs = [np.zeros(len(psets), RESULT_DTYPE), np.zeros(len(gsets), RESULT_DTYPE), np.zeros(len(cgraphs), RESULT_DTYPE),
            np.zeros(len(psets), RESULT_DTYPE)]
    plbs = [ListBuffers(len(psets), 1024, MEM_HOST, SET_LISTS), ListBuffers(len(psets), 1024, MEM_DEVICE, SET_LISTS)]
    gbuf = graph_buffers(*shape)
    clb = ListBuffers(len(cgraphs), 1024, MEM_HOST, GRAPH_LISTS)
    handle.solve_pose_batch_enqueue_each_raw(pa, len(psets), handle.params_array(pparams), MEM_HOST, outs[0], plbs[0])
    handle.build_graph_batch_enqueue_each_raw(ga, len(gsets), handle.params_array(gparams), MEM_HOST, outs[1], gbuf)
    handle.max_clique_batch_enqueue_each_raw(ca, len(cgraphs), handle.params_array(cparams), MEM_HOST, outs[2], clb)
    handle.solve_pose_batch_enqueue_each_raw(pa, len(psets), handle.params_array(pparams), MEM_HOST, outs[3], plbs[1])
    handle.register_batch_flush()
    assert outs[1].tobytes() == gref.tobytes() and outs[2].tobytes() == cref.tobytes()
    for n in gbuf.arrays:
        assert gbuf.host(n).tobytes() == gref_buf.host(n).tobytes(), n
    for i, l in enumerate(clb.trimmed(outs[2])):
        assert l["clique"].tobytes() == cl[i]["clique"].tobytes(), i
    for out, lb, dest in ((outs[0], plbs[0], MEM_HOST), (outs[3], plbs[1], MEM_DEVICE)):
        ref, rl = refs[dest]
        assert out.tobytes() == ref.tobytes(), dest
        for i, (g, w) in enumerate(zip(host_lists(lb.trimmed(out)), host_lists(rl))):
            for n in SET_LISTS:
                assert g[n].tobytes() == w[n].tobytes(), (dest, i, n)


# ---- GPU 10: stage times -----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_stage_times_are_h2d_pose_and_d2h():
    base = [scene(500 + k, c) for k, c in enumerate((300, 1000, 64, 2000))]
    with Handle(max_batch_slots=4) as h:
        h.solve_pose_batch_each([(a, b) for a, b, _ in base], [i for _, _, i in base], [pose_params()] * len(base))
        ms = h.stage_ms()
        assert ms[0] > 0 and ms[6] > 0 and ms[7] > 0 and ms[1] == ms[2] == ms[3] == ms[4] == ms[5] == 0, ms
        kms, calls = h.kernel_ms()
        assert (kms == 0).all() and (calls == 0).all()
