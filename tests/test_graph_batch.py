"""TIM consistency graphs of batches of correspondence sets: qb200_build_graph_batch_each and its queued form.  Adjacency rows, degrees
and edge counts of sets of every size class, street sets and the adversarial band families equal qb200_build_graph and the oracle, and
the edge lists equal the upper triangle of the oracle's matrix in (u, v) order; memory kinds, padded layouts, clipped and chunked edge
lists, a device-resident match -> graph -> clique chain, rejections, the shared enqueue stream and the call's side effects."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import (GRAPH_LISTS, INLIER_NONE, KCORE_HEU, MATCH_LISTS, MEM_DEVICE, MEM_HOST, PMC_EXACT, PMC_HEU, RESULT_DTYPE,
                              GraphBuffers, GraphOut, Handle, ListBuffers, default_params)
from support import P4, ROOT, device_copy, make_handle

NEW = ("qb200_build_graph_batch_each", "qb200_build_graph_batch_enqueue_each")
MODES = (PMC_EXACT, PMC_HEU, KCORE_HEU)
SIZES = (0, 1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 4095, 4096, 4097)
BAD_ARG = -1
LISTS_TRUNCATED = 2
SENT = 0x5A5A5A5A
ZERO = ("valid", "n_src_vox", "n_tgt_vox", "n_mutual", "max_core", "clique_size", "gnc_iters", "n_rot_inliers", "n_final_inliers", "cost")


# ---- CPU: layout, prototypes ----------------------------------------------------------------------------------------------------------
def test_graph_out_mirror_matches_the_c_layout(tmp_path):
    fields = ("kind", "rows_per_set", "words_per_row", "reserved", "cap_edges", "adj", "degree", "edges")
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "quatro_b200.h"\nint main(void) {\n'
                   '  printf("%zu' + " %zu" * len(fields) + '\\n", sizeof(qb200_graph_out)' +
                   "".join(f", offsetof(qb200_graph_out, {f})" for f in fields) + ");\n  return 0;\n}\n")
    exe = tmp_path / "layout"
    r = subprocess.run(["/usr/bin/gcc", "-std=c11", "-Wall", "-Werror", f"-I{ROOT / 'include'}", str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(GraphOut)] + [getattr(GraphOut, f).offset for f in fields]


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


# ---- sets and what they must give ------------------------------------------------------------------------------------------------------
def graph_params(noise_bound, cbar2=1.0, mode=PMC_HEU):
    p = default_params()
    p.noise_bound, p.cbar2, p.inlier_selection_mode, p.rot_noise_bound = noise_bound, cbar2, mode, 0.0
    return p


def sized_set(rng, L):
    """L matched points of a synthetic street-scale set, 10 % inliers"""
    if L < 2:
        a = rng.uniform(-20, 20, (L, 3))
        return P4(a), P4(a + rng.normal(0, 0.1, (L, 3)))
    a4, b4, _, _ = synth.matched_pairs(int(rng.integers(1 << 30)), L, inlier_ratio=0.1)
    return a4, b4


def street_sets(h, seeds):
    p = default_params()
    _, ml = h.match_batch_mixed([synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in seeds], [p] * len(seeds),
                                buffers=ListBuffers(len(seeds), h.cfg.max_corr, MEM_HOST, MATCH_LISTS))
    return [(m["src_matched4"], m["tgt_matched4"]) for m in ml]


def adversarial_sets():
    """a few sets of each band family of test_graph_adversarial, as (a4, b4, noise_bound) with cbar2 = 1"""
    from test_graph_adversarial import _placed, float_range_sets, overflow_sets, smin_net_sets, threshold_sets, tight_block_sets
    out = []
    for fam in (threshold_sets(), threshold_sets(step=2.0 ** -12), tight_block_sets(), smin_net_sets(), float_range_sets()):
        out += [(a, b, beta / 2) for a, b, beta in fam[::max(1, len(fam) // 6)]]
    ov = overflow_sets(1e9, 1e10, 40)
    out.append((np.concatenate([s[0] for s in ov]), np.concatenate([s[1] for s in ov]), 5e8))
    out.append((*_placed(257, 357), 0.3))
    return out


def upper_edges(adj, L):
    """every edge (u, v), u < v, of the adjacency rows in lexicographic order"""
    if L < 2:
        return np.zeros((0, 2), np.int32)
    bits = np.unpackbits(adj[:L].view(np.uint8), axis=1, bitorder="little")[:, :L].astype(bool)
    u, v = np.nonzero(np.triu(bits, 1))
    return np.stack([u, v], 1).astype(np.int32)


def check_set(i, rec, buf, adj, deg, n_edges, label):
    """set i of the call (record, GraphBuffers) against qb200_build_graph's adj (full rows of the buffers' words_per_row), degrees
    and edge count"""
    L = adj.shape[0]
    assert rec["status"] == 0 and rec["n_corr"] == L and rec["n_edges"] == n_edges, (label, rec)
    for k in ZERO:
        assert rec[k] == 0, (label, k)
    assert np.array_equal(np.asarray(rec["T"]), np.eye(4).reshape(-1)), label
    if "adj" in buf.arrays:
        got = buf.host("adj")[i]
        assert got[:L].tobytes() == adj.tobytes(), label
        assert (got[L:] == np.uint32(SENT)).all(), label
    if "degree" in buf.arrays:
        got = buf.host("degree")[i]
        assert got[:L].tobytes() == deg.tobytes() and (got[L:] == SENT).all(), label
    if "edges" in buf.arrays:
        got = buf.host("edges")[i]
        m = min(n_edges, buf.cap_edges)
        want = upper_edges(adj, L)
        assert len(want) == n_edges, label
        assert got[:m].tobytes() == want[:m].tobytes(), label
        assert (got[m:] == SENT).all(), label
        assert bool(rec["flags"] & LISTS_TRUNCATED) == (n_edges > buf.cap_edges), label
    else:
        assert rec["flags"] == 0, label


def buffers(n, rows, wpr, cap, kind=MEM_HOST, arrays=("adj", "degree", "edges")):
    return GraphBuffers(n, rows, wpr, cap, kind, arrays, fill=SENT)


# ---- GPU 1: a mixed batch equals the single call and the oracle ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mixed():
    """(sets, params): every size class, street sets and the adversarial families, each with its own noise_bound and cbar2; some
    entries in QB200_INLIER_NONE"""
    rng = np.random.default_rng(31)
    sets, params = [], []
    for k, L in enumerate(SIZES):
        sets.append(sized_set(rng, L))
        params.append(graph_params(float(rng.uniform(0.1, 0.6)), float(rng.uniform(0.5, 2.0)), (PMC_HEU, INLIER_NONE)[k % 2]))
    with Handle(max_batch_slots=8) as h:
        for a, b in street_sets(h, range(2000, 2004)):
            sets.append((a, b))
            params.append(graph_params(float(rng.uniform(0.2, 0.6)), float(rng.uniform(0.5, 1.5))))
    for a, b, nb in adversarial_sets():
        sets.append((a, b))
        params.append(graph_params(nb))
    return sets, params


@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 4])
def test_mixed_batch_equals_single_calls_and_the_oracle(mixed, oracle, lanes):
    sets, params = mixed
    h = make_handle(lanes, max_batch_slots=8, max_corr=8192)
    try:
        assert len(sets) > 3 * 8
        rows = max(len(a) for a, _ in sets)
        wpr = (rows + 31) // 32
        single = [h.build_graph(a, b, p.noise_bound, p.cbar2, wpr) for (a, b), p in zip(sets, params)]
        buf = buffers(len(sets), rows, wpr, max(ne for _, _, ne in single))
        recs = h.build_graph_batch_each(sets, params, MEM_HOST, buf)
        for i, ((a, b), p, (adj, deg, ne)) in enumerate(zip(sets, params, single)):
            oadj, odeg, one = oracle.build_graph(a, b, p.noise_bound, p.cbar2, wpr)
            assert adj.tobytes() == oadj.tobytes() and deg.tobytes() == odeg.tobytes() and ne == one, i
            check_set(i, recs[i], buf, adj, deg, ne, (lanes, i, len(a)))
    finally:
        h.close()


# ---- GPU 2: memory kinds and padded layouts ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_memory_kinds_give_the_same_bytes(handle):
    rng = np.random.default_rng(32)
    sizes = (40, 0, 300, 1, 33, 1000, 64, 2, 700, 129, 4096, 5)
    sets = [sized_set(rng, L) for L in sizes]
    params = [graph_params(float(rng.uniform(0.1, 0.5)), float(rng.uniform(0.5, 2))) for _ in sizes]
    rows = 4096 + 7
    wpr = (rows + 31) // 32 + 2
    single = [handle.build_graph(a, b, p.noise_bound, p.cbar2, wpr) for (a, b), p in zip(sets, params)]
    cap = max(ne for _, _, ne in single) + 5
    ref_buf = buffers(len(sets), rows, wpr, cap)
    ref = handle.build_graph_batch_each(sets, params, MEM_HOST, ref_buf)
    for i, (adj, deg, ne) in enumerate(single):
        check_set(i, ref[i], ref_buf, adj, deg, ne, i)
    keep = [(device_copy(a), device_copy(b)) for a, b in sets]
    dev_sets = [(ta.data_ptr(), tb.data_ptr(), len(a)) for (ta, tb), (a, _) in zip(keep, sets)]
    for kind, ss in ((MEM_HOST, sets), (MEM_DEVICE, dev_sets)):
        for dest in (MEM_HOST, MEM_DEVICE):
            buf = buffers(len(sets), rows, wpr, cap, dest)
            recs = handle.build_graph_batch_each(ss, params, kind, buf)
            assert recs.tobytes() == ref.tobytes(), (kind, dest)
            for name in buf.arrays:
                assert buf.host(name).tobytes() == ref_buf.host(name).tobytes(), (kind, dest, name)


# ---- GPU 3: clipped edge lists ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_clipped_edge_lists_carry_the_flag(handle):
    rng = np.random.default_rng(33)
    sets = [sized_set(rng, L) for L in (200, 3, 500, 64, 1500)]
    params = [graph_params(0.4)] * len(sets)
    full = buffers(len(sets), 1500, 47, 1500 * 1499 // 2, arrays=("edges",))
    recs = handle.build_graph_batch_each(sets, params, MEM_HOST, full)
    assert recs["flags"].sum() == 0
    cap = int(np.median(recs["n_edges"]))
    assert 0 < cap < recs["n_edges"].max() and (recs["n_edges"] < cap).any()
    for dest in (MEM_HOST, MEM_DEVICE):
        buf = buffers(len(sets), 0, 0, cap, dest, ("edges",))
        got = handle.build_graph_batch_each(sets, params, MEM_HOST, buf)
        edges = buf.host("edges")
        for i, r in enumerate(recs):
            m = min(int(r["n_edges"]), cap)
            assert got[i]["flags"] == (LISTS_TRUNCATED if r["n_edges"] > cap else 0), (dest, i)
            want = r.copy()
            want["flags"] = got[i]["flags"]
            assert got[i].tobytes() == want.tobytes(), (dest, i)
            assert edges[i, :m].tobytes() == full.host("edges")[i, :m].tobytes(), (dest, i)
            assert (edges[i, m:] == SENT).all(), (dest, i)


# ---- GPU 4: host edge lists larger than the edge staging -------------------------------------------------------------------------------
@pytest.mark.gpu
def test_host_edge_lists_cross_in_windows():
    """One slot per wave, one raw point per cloud, max_corr 4096: the edge staging (adjp, 4096 x 128 words) holds 262 144 edges, and a
    near-complete graph of 4096 vertices has about 8.4 M"""
    h = make_handle(2, max_batch_slots=1, max_raw_points=1, max_corr=4096)
    try:
        rng = np.random.default_rng(34)
        a = rng.uniform(-20, 20, (4096, 3))
        b = a + rng.normal(0, 0.01, (4096, 3))
        b[rng.choice(4096, 12, replace=False)] += 50.0      # a few outliers: not quite complete
        sets = [(P4(a), P4(b)), sized_set(rng, 900)]   # two waves
        params = [graph_params(0.5), graph_params(0.3)]
        buf = buffers(2, 4096, 128, 4096 * 4095 // 2, MEM_HOST, ("adj", "edges"))
        recs = h.build_graph_batch_each(sets, params, MEM_HOST, buf)
        assert recs[0]["n_edges"] > 8_000_000 and recs[0]["n_edges"] < 4096 * 4095 // 2
        for i, ((sa, sb), p) in enumerate(zip(sets, params)):
            adj, deg, ne = h.build_graph(sa, sb, p.noise_bound, p.cbar2, 128)
            assert ne == recs[i]["n_edges"] and buf.host("adj")[i][:len(sa)].tobytes() == adj.tobytes(), i
            want = upper_edges(adj, len(sa))
            assert buf.host("edges")[i][:ne].tobytes() == want.tobytes(), i
            assert (buf.host("edges")[i][ne:] == SENT).all(), i
    finally:
        h.close()


# ---- GPU 5: a device-resident chain -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_match_graph_clique_on_the_device_equals_register(handle):
    pairs = [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(2100, 2106)]
    cap = handle.cfg.max_corr
    p = default_params()
    p.rot_noise_bound = 0.6
    ml = ListBuffers(len(pairs), cap, MEM_DEVICE, MATCH_LISTS)
    mrec, _ = handle.match_batch_mixed(pairs, [p] * len(pairs), buffers=ml)
    sa, sb = ml.arrays["src_matched4"], ml.arrays["tgt_matched4"]
    sets = [(sa[i].data_ptr(), sb[i].data_ptr(), int(mrec[i]["n_corr"])) for i in range(len(pairs))]
    m = int(mrec["n_corr"].max())
    buf = buffers(len(pairs), m, (m + 31) // 32, m * (m - 1) // 2, MEM_DEVICE, ("adj", "edges"))
    grec = handle.build_graph_batch_each(sets, [p] * len(pairs), MEM_DEVICE, buf)
    for mode in MODES:
        q = default_params()
        q.inlier_selection_mode, q.rot_noise_bound = mode, 0.6
        rrec, rl = handle.register_batch_mixed(pairs, [q] * len(pairs), buffers=ListBuffers(len(pairs), cap, MEM_HOST, ("clique",)))
        cp = default_params()
        cp.inlier_selection_mode, cp.kcore_heuristic_threshold = mode, q.kcore_heuristic_threshold
        for use in ("edges", "adj"):
            crec, cl = handle.max_clique_batch_each(buf.graphs(grec, use), [cp] * len(pairs), MEM_DEVICE,
                                                    buffers=ListBuffers(len(pairs), cap, MEM_DEVICE, GRAPH_LISTS))
            for i in range(len(pairs)):
                for k in ("n_edges", "max_core", "clique_size", "flags"):
                    assert crec[i][k] == rrec[i][k], (mode, use, i, k)
                assert crec[i]["n_edges"] == grec[i]["n_edges"]
                assert cl[i]["clique"].cpu().numpy().tobytes() == rl[i]["clique"].tobytes(), (mode, use, i)


# ---- GPU 6: rejections ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rejections_write_nothing_and_name_the_entry(handle):
    import torch
    rng = np.random.default_rng(36)
    ok = sized_set(rng, 40)
    big = sized_set(rng, 70)
    t = torch.zeros(64, dtype=torch.int32, device="cuda")
    host = buffers(2, 64, 2, 100)

    def out(**kw):
        d = host.descriptor()
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    good = [graph_params(0.3)] * 2
    cases = [
        ("set 1", [ok, (ok[0], ok[1][:0])], MEM_HOST, good, out()),
        ("set 1", [ok, big], MEM_HOST, good, out()),                                   # L > rows_per_set
        ("set 0", [sized_set(rng, handle.cfg.max_corr + 1)], MEM_HOST, good[:1], out()),
        ("params entry 1", [ok, ok], MEM_HOST, [graph_params(0.3), graph_params(0.0)], out()),
        ("params entry 0", [ok], MEM_HOST, [graph_params(0.3, -1.0)], out()),
        ("null", [ok], MEM_HOST, good[:1], None),
        ("unknown memory kind of the outputs", [ok], MEM_HOST, good[:1], out(kind=5)),
        ("unknown memory kind of the inputs", [ok], 7, good[:1], out()),
        ("rows_per_set < 0", [ok], MEM_HOST, good[:1], out(rows_per_set=-1)),
        ("words_per_row", [ok], MEM_HOST, good[:1], out(words_per_row=1)),
        ("cap_edges", [ok], MEM_HOST, good[:1], out(cap_edges=0)),
        ("device adj", [ok], MEM_HOST, good[:1], out(kind=MEM_DEVICE, degree=None, edges=None)),
        ("device adj", [ok], MEM_HOST, good[:1], out(kind=MEM_DEVICE, adj=t.data_ptr() + 2, degree=None, edges=None)),
        ("device degree", [ok], MEM_HOST, good[:1], out(kind=MEM_DEVICE, adj=None, degree=t.data_ptr() + 1, edges=None)),
        ("device edges", [ok], MEM_HOST, good[:1], out(kind=MEM_DEVICE, adj=None, degree=None, edges=t.data_ptr() + 4)),
    ]
    # a queued batch before the rejected calls still completes on the flush
    qsets = [sized_set(rng, L) for L in (50, 7, 300)]
    qparams = [graph_params(0.35)] * 3
    want_buf = buffers(3, 300, 10, 50000)
    want = handle.build_graph_batch_each(qsets, qparams, MEM_HOST, want_buf)
    qbuf = buffers(3, 300, 10, 50000)
    qrec = np.zeros(3, RESULT_DTYPE)
    qarr, qkeep = handle._set_array(qsets, MEM_HOST)
    qpa = handle.params_array(qparams)
    handle.build_graph_batch_enqueue_each_raw(qarr, 3, qpa, MEM_HOST, qrec, qbuf)
    lib = handle.lib
    for why, ss, kind, ps, d in cases:
        arr, keep = handle._set_array(ss, MEM_HOST) if not (len(ss) == 2 and len(ss[1][1]) == 0) else _null_second(ss)
        rec = np.zeros(len(ss), RESULT_DTYPE)
        rec.view(np.uint8)[...] = 0xA5
        for fn in NEW[::-1]:
            rc = getattr(lib, fn)(handle.h, arr, len(ss), handle.params_array(ps), kind, rec.ctypes.data, None if d is None else C.byref(d))
            assert rc == BAD_ARG, (why, fn)
            assert why in lib.qb200_last_error(handle.h).decode(), (why, lib.qb200_last_error(handle.h))
            assert (rec.view(np.uint8) == 0xA5).all(), why
            assert all((host.host(n).view(np.uint32) == SENT).all() for n in host.arrays), why
    handle.register_batch_flush()
    assert qrec.tobytes() == want.tobytes()
    for n in qbuf.arrays:
        assert qbuf.host(n).tobytes() == want_buf.host(n).tobytes(), n
    assert lib.qb200_build_graph_batch_each(handle.h, None, -1, None, MEM_HOST, None, C.byref(host.descriptor())) == BAD_ARG
    assert lib.qb200_build_graph_batch_each(handle.h, handle._set_array([ok], MEM_HOST)[0], 1, handle.params_array(good[:1]), MEM_HOST,
                                            None, C.byref(host.descriptor())) == BAD_ARG
    del t


def _null_second(ss):
    """a set array whose second set has L points and null arrays"""
    arr, keep = capi._set_array([ss[0]], MEM_HOST)
    out = (capi.CorrSet * 2)()
    out[0] = arr[0]
    out[1].L = len(ss[1][0])
    return out, keep


# ---- GPU 7: one queued stream ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_enqueue_interleaved_with_raw_set_and_clique_batches(handle):
    rng = np.random.default_rng(37)
    gsets = [sized_set(rng, L) for L in (50, 400, 33, 900, 128, 7, 2000, 60, 300, 1000, 12)]
    gparams = [graph_params(float(rng.uniform(0.2, 0.5)), float(rng.uniform(0.5, 2))) for _ in gsets]
    pairs = [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(2200, 2203)]
    pp = default_params()
    pp.rot_noise_bound = 0.6
    sets = [synth.matched_pairs(s, 300)[:2] for s in range(2300, 2312)]
    cgraphs = [np.ascontiguousarray(handle.build_graph(a, b, 0.3, 1.0)[0]) for a, b in gsets[:5]]
    cparams = [default_params()] * len(cgraphs)
    shape = (len(gsets), 2000, 64, 100_000)
    refs = {}
    for dest in (MEM_HOST, MEM_DEVICE):
        b = buffers(*shape, dest)
        refs[dest] = (handle.build_graph_batch_each(gsets, gparams, MEM_HOST, b), b)
    raw_ref = handle.register_batch(pairs, pp)
    set_ref, _ = handle.solve_batch_each(sets, [pp] * len(sets))
    clq_ref, _ = handle.max_clique_batch_each(cgraphs, cparams)
    ga, gkeep = handle._set_array(gsets, MEM_HOST)
    gpa = handle.params_array(gparams)
    pa, pkeep = handle.pair_array(pairs)
    sa, skeep = handle._set_array(sets, MEM_HOST)
    ca, ckeep = handle.graph_array(cgraphs)
    outs = [np.zeros(len(gsets), RESULT_DTYPE), np.zeros(len(pairs), RESULT_DTYPE), np.zeros(len(gsets), RESULT_DTYPE),
            np.zeros(len(sets), RESULT_DTYPE), np.zeros(len(cgraphs), RESULT_DTYPE)]
    bufs = [buffers(*shape, MEM_HOST), buffers(*shape, MEM_DEVICE)]
    handle.build_graph_batch_enqueue_each_raw(ga, len(gsets), gpa, MEM_HOST, outs[0], bufs[0])
    handle.register_batch_enqueue_raw(pa, len(pairs), pp, MEM_HOST, outs[1])
    handle.build_graph_batch_enqueue_each_raw(ga, len(gsets), gpa, MEM_HOST, outs[2], bufs[1])
    handle.solve_batch_enqueue_each_raw(sa, len(sets), handle.params_array([pp] * len(sets)), MEM_HOST, outs[3])
    handle.max_clique_batch_enqueue_each_raw(ca, len(cgraphs), handle.params_array(cparams), MEM_HOST, outs[4])
    handle.register_batch_flush()
    assert outs[1].tobytes() == raw_ref.tobytes() and outs[3].tobytes() == set_ref.tobytes() and outs[4].tobytes() == clq_ref.tobytes()
    for out, b, dest in ((outs[0], bufs[0], MEM_HOST), (outs[2], bufs[1], MEM_DEVICE)):
        ref, rb = refs[dest]
        assert out.tobytes() == ref.tobytes(), dest
        for n in b.arrays:
            assert b.host(n).tobytes() == rb.host(n).tobytes(), (dest, n)


# ---- GPU 8: stage times and no latch ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_stage_times_and_nothing_latched():
    rng = np.random.default_rng(38)
    sets = [sized_set(rng, L) for L in (300, 1000, 64, 2000)]
    solve_sets = [synth.matched_pairs(s, 400)[:2] for s in range(2400, 2404)]
    sp = default_params()   # rot_noise_bound = 0: resolved by the first solve on the handle
    sp.noise_bound = 0.25
    with Handle(max_batch_slots=4) as fresh:
        want, _ = fresh.solve_batch_each(solve_sets, [sp] * len(solve_sets))
    with Handle(max_batch_slots=4) as h:
        h.build_graph_batch_each(sets, [graph_params(0.6)] * len(sets), MEM_HOST, buffers(len(sets), 2000, 63, 1, MEM_HOST, ("adj", "degree")))
        ms = h.stage_ms()
        assert ms[0] > 0 and ms[4] > 0 and ms[7] > 0 and ms[1] == ms[2] == ms[3] == ms[5] == ms[6] == 0, ms
        kms, calls = h.kernel_ms()
        assert kms[1] > 0 and calls[1] >= 1 and calls[0] == 0
        got, _ = h.solve_batch_each(solve_sets, [sp] * len(solve_sets))
        assert got.tobytes() == want.tobytes()
