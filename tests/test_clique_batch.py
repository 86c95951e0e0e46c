"""Maximum cliques of batches of caller graphs: qb200_max_clique_batch_each and its queued form, and the teaser/graph.h shim over them.
Adjacency and edge-list graphs of every size class in every mode equal qb200_max_clique_ex and the oracle; edge lists follow
teaser::Graph::addEdge; small graphs are checked against networkx; TIM graphs of street pairs give the cliques qb200_solve_batch_ex
lists; device kinds, padded rows, invalid graphs, rejections, the shared enqueue stream, clipped lists and the C++ shim."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import (GRAPH_LISTS, KCORE_HEU, MATCH_LISTS, MEM_DEVICE, MEM_HOST, PMC_EXACT, PMC_HEU, RESULT_DTYPE, Graph,
                              ListBuffers, default_params)
from support import ROOT, device_copy, make_handle

NEW = ("qb200_max_clique_batch_each", "qb200_max_clique_batch_enqueue_each")
MODES = (PMC_EXACT, PMC_HEU, KCORE_HEU)
SIZES = (0, 1, 2, 31, 32, 33, 4096, 4097, 8192, 8193, 20000, 32768)
BAD_ARG = -1
CLIQUE_TRUNCATED, LISTS_TRUNCATED = 1, 2
ZERO = ("valid", "n_src_vox", "n_tgt_vox", "n_mutual", "gnc_iters", "n_rot_inliers", "n_final_inliers", "cost")
SHIM = "tests/fixtures/clique_batch_shim.cpp"


# ---- CPU: layout, prototypes, the shim ---------------------------------------------------------------------------------------------
def test_graph_mirror_matches_the_c_layout(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "quatro_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(qb200_graph), offsetof(qb200_graph, edges), offsetof(qb200_graph, adj),\n'
                   '         offsetof(qb200_graph, n_edges), offsetof(qb200_graph, L), offsetof(qb200_graph, words_per_row));\n'
                   '  return 0;\n}\n')
    exe = tmp_path / "layout"
    r = subprocess.run(["/usr/bin/gcc", "-std=c11", "-Wall", "-Werror", f"-I{ROOT / 'include'}", str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(Graph)] + [getattr(Graph, f).offset for f in ("edges", "adj", "n_edges", "L", "words_per_row")]


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


def build_shim(tmp_path):
    """The fixture compiled as a caller of the reference would build it (INTEGRATION.md, Option A), linked to the library."""
    from quatro_b200 import _build
    lib = _build.build_cuda()
    exe = tmp_path / "clique_batch_shim"
    cmd = ["/usr/bin/g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", f"-I{ROOT / 'include'}", f"-I{ROOT / 'include' / 'quatro_b200'}",
           str(ROOT / SHIM), f"-L{lib.parent}", "-lquatro_b200", f"-Wl,-rpath,{lib.parent}", "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_the_graph_shim_compiles(tmp_path):
    build_shim(tmp_path)


def test_a_null_handle_is_refused():
    lib = capi.load_library()
    for n in NEW:
        assert getattr(lib, n)(None, None, 0, None, MEM_HOST, None, None) == BAD_ARG, n


# ---- graphs --------------------------------------------------------------------------------------------------------------------------
def params_for(mode, thr=0.5, node_limit=0):
    p = default_params()
    p.inlier_selection_mode, p.kcore_heuristic_threshold, p.max_clique_node_limit = mode, thr, node_limit
    return p


def pack(L, u, v, wpr=None):
    """(L, wpr) uint32 rows of the undirected graph with edges (u[k], v[k]), both bits of each"""
    wpr = wpr or max((L + 31) // 32, 1) if L else 1
    u, v = np.asarray(u, np.int64), np.asarray(v, np.int64)
    r, c = np.concatenate([u, v]), np.concatenate([v, u])
    a = np.zeros(max(L, 1) * wpr, np.uint32)
    np.bitwise_or.at(a, r * wpr + (c >> 5), np.uint32(1) << (c & 31).astype(np.uint32))
    return a.reshape(max(L, 1), wpr)[:L]


def random_graph(rng, L):
    """distinct undirected edges (u < v) of a sparse random graph with a planted clique"""
    if L < 2:
        return np.zeros((0, 2), np.int64)
    deg = 24 if L <= 4096 else 6
    m = L * deg // 2 if L > 64 else L * (L - 1) // 4
    u, v = rng.integers(0, L, m), rng.integers(0, L, m)
    k = min(L, 5 + L % 7 + (13 if L > 100 else 0))   # above the random part's core: the heuristic meets the k-core bound
    members = rng.choice(L, k, replace=False)
    a, b = np.triu_indices(k, 1)
    u, v = np.concatenate([u, members[a]]), np.concatenate([v, members[b]])
    keep = u != v
    e = np.stack([np.minimum(u, v), np.maximum(u, v)], 1)[keep]
    return np.unique(e, axis=0)


def shuffled_edges(rng, e):
    """the edge list with both orientations of some edges, duplicates, in random order"""
    if len(e) == 0:
        return e.astype(np.int32)
    flip = rng.random(len(e)) < 0.5
    out = np.where(flip[:, None], e[:, ::-1], e)
    both = e[rng.random(len(e)) < 0.3][:, ::-1]
    dup = e[rng.random(len(e)) < 0.2]
    out = np.concatenate([out, both, dup])
    return np.ascontiguousarray(out[rng.permutation(len(out))], np.int32)


def expected_record(h, adj, mode, thr=0.5, node_limit=0):
    clique, _, _, mc, fl = h.max_clique_ex(adj, mode, thr, node_limit)
    L = adj.shape[0]
    n_edges = int(np.unpackbits(adj.view(np.uint8)).sum()) // 2 if L else 0
    return dict(status=0, n_corr=L, n_edges=n_edges, max_core=mc, clique_size=len(clique), flags=fl), clique


def assert_record(r, want, label):
    for k, v in want.items():
        assert r[k] == v, (label, k, r[k], v)
    for k in ZERO:
        assert r[k] == 0, (label, k, r[k])
    assert np.array_equal(np.asarray(r["T"]), np.eye(4).reshape(-1)), label


def clique_lists(n, cap, kind=MEM_HOST):
    return ListBuffers(n, cap, kind, GRAPH_LISTS)


@pytest.fixture(scope="module")
def wide():
    """32768-vertex handle: 2 slots per wave over 2 lanes, so a batch of more than 4 graphs rotates"""
    h = make_handle(2, max_batch_slots=2, max_corr=32768)
    yield h
    h.close()


@pytest.fixture(scope="module")
def size_graphs():
    rng = np.random.default_rng(7)
    return [(L, random_graph(rng, L)) for L in SIZES]


@pytest.fixture(scope="module")
def size_batch(wide, size_graphs):
    """every size class in every mode, adjacency input, one call: (graphs, params, records, lists)"""
    graphs, params = [], []
    for mode in MODES:
        for L, e in size_graphs:
            graphs.append(pack(L, e[:, 0], e[:, 1]))
            params.append(params_for(mode))
    lb = clique_lists(len(graphs), wide.cfg.max_corr)
    recs, lists = wide.max_clique_batch_each(graphs, params, buffers=lb)
    return graphs, params, recs, lists


# ---- GPU 1, 2: every size class and mode, adjacency and edge lists -------------------------------------------------------------------
@pytest.mark.gpu
def test_adjacency_graphs_equal_the_single_call_and_the_oracle(wide, size_batch, oracle):
    graphs, params, recs, lists = size_batch
    assert len(graphs) > 2 * 2
    for i, (adj, p) in enumerate(zip(graphs, params)):
        label = (adj.shape[0], p.inlier_selection_mode)
        want, clique = expected_record(wide, adj, p.inlier_selection_mode)
        assert_record(recs[i], want, label)
        assert lists[i]["clique"].tobytes() == clique.astype(np.int32).tobytes(), label
        if adj.shape[0]:
            oc, _, _, omc, ofl = oracle.max_clique_ex(adj, p.inlier_selection_mode, 0.5, 0)
            assert np.array_equal(oc, clique) and omc == want["max_core"] and ofl == want["flags"], label


@pytest.mark.gpu
def test_edge_lists_equal_the_adjacency_input(wide, size_batch, size_graphs):
    graphs, params, recs, lists = size_batch
    rng = np.random.default_rng(8)
    edge_graphs = [(L, shuffled_edges(rng, e)) for _ in MODES for L, e in size_graphs]
    lb = clique_lists(len(edge_graphs), wide.cfg.max_corr)
    got, glists = wide.max_clique_batch_each(edge_graphs, params, buffers=lb)
    assert got.tobytes() == recs.tobytes()
    for i, (L, e) in enumerate(size_graphs * len(MODES)):
        assert got[i]["n_edges"] == len(e)
        assert glists[i]["clique"].tobytes() == lists[i]["clique"].tobytes()


# ---- GPU 3: small graphs against networkx ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_small_graphs_against_networkx(handle):
    import networkx as nx
    rng = np.random.default_rng(11)
    graphs, params, nxg = [], [], []
    for k in range(36):
        L = int(rng.integers(1, 201))
        p = (0.05, 0.15, 0.3, 0.5)[k % 4]
        u, v = np.triu_indices(L, 1)
        keep = rng.random(len(u)) < p
        e = np.stack([u[keep], v[keep]], 1)
        g = nx.Graph()
        g.add_nodes_from(range(L))
        g.add_edges_from(e.tolist())
        graphs.append((L, e))
        params.append(params_for(MODES[k % 3]))
        nxg.append(g)
    recs, lists = handle.max_clique_batch_each(graphs, params, buffers=clique_lists(len(graphs), 256))
    for i, g in enumerate(nxg):
        c = lists[i]["clique"].tolist()
        assert recs[i]["status"] == 0 and len(c) == recs[i]["clique_size"]
        assert all(g.has_edge(a, b) for a in c for b in c if a < b), i
        assert recs[i]["n_edges"] == g.number_of_edges()
        if params[i].inlier_selection_mode == PMC_EXACT:
            assert len(c) == len(nx.max_weight_clique(g, weight=None)[0]), i


@pytest.mark.gpu
def test_a_small_node_limit_truncates_as_the_single_call(handle):
    rng = np.random.default_rng(12)
    graphs, params = [], []
    for k in range(12):
        L = 120 + 7 * k
        u, v = np.triu_indices(L, 1)
        keep = rng.random(len(u)) < 0.6
        graphs.append(pack(L, u[keep], v[keep]))
        params.append(params_for(PMC_EXACT, node_limit=(1, 3, 20, 500)[k % 4]))
    recs, lists = handle.max_clique_batch_each(graphs, params, buffers=clique_lists(len(graphs), 256))
    assert any(r["flags"] & CLIQUE_TRUNCATED for r in recs)
    for i, (adj, p) in enumerate(zip(graphs, params)):
        want, clique = expected_record(handle, adj, PMC_EXACT, 0.5, p.max_clique_node_limit)
        assert_record(recs[i], want, i)
        assert lists[i]["clique"].tobytes() == clique.astype(np.int32).tobytes(), i


# ---- GPU 4: TIM graphs of street correspondence sets ----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_tim_graphs_give_the_cliques_of_solve_batch(handle):
    pairs = [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(1500, 1506)]
    mp = [default_params() for _ in pairs]
    for p in mp:
        p.rot_noise_bound = 0.6
    _, ml = handle.match_batch_mixed(pairs, mp, buffers=ListBuffers(len(pairs), handle.cfg.max_corr, MEM_HOST, MATCH_LISTS))
    sets = [(m["src_matched4"], m["tgt_matched4"]) for m in ml if len(m["src_matched4"]) > 1]
    assert len(sets) >= 4
    for mode in MODES:
        p = default_params()
        p.inlier_selection_mode, p.rot_noise_bound = mode, 0.6
        _, sl = handle.solve_batch_lists(sets, p, cap_per_pair=handle.cfg.max_corr, dest=MEM_HOST)
        graphs = [handle.build_graph(a, b, p.noise_bound, p.cbar2)[0] for a, b in sets]
        recs, gl = handle.max_clique_batch_each(graphs, [params_for(mode, p.kcore_heuristic_threshold)] * len(graphs),
                                                buffers=clique_lists(len(graphs), handle.cfg.max_corr))
        for i in range(len(sets)):
            assert gl[i]["clique"].tobytes() == sl[i]["clique"].tobytes(), (mode, i)


# ---- GPU 5: device kinds, padded rows -------------------------------------------------------------------------------------------------
def padded(adj, extra, rng):
    """adj with `extra` more words per row and every bit at columns >= L set"""
    L, w = adj.shape
    out = np.zeros((L, w + extra), np.uint32)
    out[:, :w] = adj
    out[:, w:] = rng.integers(0, 2**32, (L, extra), dtype=np.uint64).astype(np.uint32)
    if L % 32:
        out[:, w - 1] |= np.uint32(~((1 << (L % 32)) - 1) & 0xFFFFFFFF)
    return out


@pytest.mark.gpu
def test_device_inputs_device_lists_and_padded_rows(handle):
    rng = np.random.default_rng(13)
    sizes = (0, 5, 33, 100, 257, 1000, 2049, 4096, 70, 31, 64)
    edges = [random_graph(rng, L) for L in sizes]
    adjs = [pack(L, e[:, 0], e[:, 1]) for L, e in zip(sizes, edges)]
    params = [params_for(MODES[i % 3]) for i in range(len(sizes))]
    ref, rl = handle.max_clique_batch_each(adjs, params, buffers=clique_lists(len(sizes), 4096))
    pads = [padded(a, 1 + i % 3, rng) for i, a in enumerate(adjs)]
    host_pad, hl = handle.max_clique_batch_each(pads, params, buffers=clique_lists(len(sizes), 4096))
    assert host_pad.tobytes() == ref.tobytes()
    keep, dev_rows, dev_edges = [], [], []
    for L, e, pa in zip(sizes, edges, pads):
        tr, te = device_copy(pa), device_copy(shuffled_edges(rng, e))
        keep += [tr, te]
        dev_rows.append(Graph(None, tr.data_ptr() if L else None, 0, L, pa.shape[1]))
        dev_edges.append(Graph(te.data_ptr() if len(e) else None, None, te.shape[0], L, 0))
    for label, gs in (("rows", dev_rows), ("edges", dev_edges)):
        for dest in (MEM_HOST, MEM_DEVICE):
            recs, gl = handle.max_clique_batch_each(gs, params, MEM_DEVICE, buffers=clique_lists(len(sizes), 4096, dest))
            assert recs.tobytes() == ref.tobytes(), (label, dest)
            for i in range(len(sizes)):
                got = gl[i]["clique"] if dest == MEM_HOST else gl[i]["clique"].cpu().numpy()
                assert got.tobytes() == rl[i]["clique"].tobytes(), (label, dest, i)


# ---- GPU 6: invalid graphs ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_invalid_graphs_are_refused_alone(handle):
    rng = np.random.default_rng(14)
    good = [random_graph(rng, L) for L in (40, 300, 77, 500, 64)]
    L = 90
    e = random_graph(rng, L)
    asym = pack(L, e[:, 0], e[:, 1])
    asym[3, 1] ^= np.uint32(1 << 5)   # edge (3, 37) without (37, 3)
    diag = pack(L, e[:, 0], e[:, 1])
    diag[60, 1] |= np.uint32(1 << 28)  # bit (60, 60)
    bad = [(L, np.concatenate([e, [[17, 17]]])), (L, np.concatenate([e, [[5, L]]])), (L, np.concatenate([[[-1, 3]], e])), asym, diag]
    graphs, params = [], []
    for i, b in enumerate(bad):
        g = good[i]
        graphs += [(max(g.max() + 1, 1), g), b]
        params += [params_for(MODES[i % 3]), params_for(MODES[(i + 1) % 3])]
    ref, rl = handle.max_clique_batch_each(graphs[0::2], params[0::2], buffers=clique_lists(len(good), 512))
    for kind in (MEM_HOST, MEM_DEVICE):
        gs, keep = graphs, []
        if kind == MEM_DEVICE:
            gs = []
            for g in graphs:
                if isinstance(g, tuple):
                    t = device_copy(np.ascontiguousarray(g[1], np.int32))
                    gs.append(Graph(t.data_ptr(), None, len(g[1]), g[0], 0))
                else:
                    t = device_copy(g)
                    gs.append(Graph(None, t.data_ptr(), 0, g.shape[0], g.shape[1]))
                keep.append(t)
        lb = clique_lists(len(gs), 512)
        for a in lb.arrays.values():
            a[...] = -7
        recs, gl = handle.max_clique_batch_each(gs, params, kind, buffers=lb)
        for i in range(len(bad)):
            r = recs[2 * i + 1]
            assert r["status"] == BAD_ARG and r["n_corr"] == L and r["clique_size"] == 0 and r["n_edges"] == 0, (kind, i)
            assert (lb.arrays["clique"][2 * i + 1] == -7).all(), (kind, i)
            assert recs[2 * i].tobytes() == ref[i].tobytes(), (kind, i)
            assert gl[2 * i]["clique"].tobytes() == rl[i]["clique"].tobytes(), (kind, i)


# ---- GPU 6b: host edge lists larger than the edge staging --------------------------------------------------------------------------
def dense_edges(rng, L, p):
    u, v = np.triu_indices(L, 1)
    keep = rng.random(len(u)) < p
    return np.stack([u[keep], v[keep]], 1)


@pytest.mark.gpu
def test_host_edge_lists_cross_in_chunks():
    """A handle whose edge staging holds 2048 edges (2 slots, 1 raw point per cloud, max_corr 256: the larger idle buffer is adjp,
    2 x 256 x 8 words).  Waves of two: a packed list beside a streamed dense one; two streamed lists, the first with an out-of-range
    vertex in a late chunk; a packed list beside one that no longer fits beside it and crosses in a single chunk."""
    h = make_handle(2, max_batch_slots=2, max_raw_points=1, max_corr=256)
    try:
        rng = np.random.default_rng(21)
        distinct = [random_graph(rng, 40), dense_edges(rng, 256, 0.9), dense_edges(rng, 200, 0.5), dense_edges(rng, 256, 0.3),
                    random_graph(rng, 100), random_graph(rng, 60)]
        Ls = (40, 256, 200, 256, 100, 60)
        modes = (PMC_EXACT, PMC_HEU, KCORE_HEU, PMC_EXACT, PMC_HEU, KCORE_HEU)
        lists = [shuffled_edges(rng, e) for e in distinct]
        sizes = [len(e) for e in lists]
        assert sizes[0] + sizes[1] > 2048 and sizes[1] > 10 * 2048 and min(sizes[2], sizes[3]) > 3 * 2048
        assert sizes[4] <= 2048 < sizes[4] + sizes[5] and sizes[5] <= 2048
        bad = len(lists[2]) * 9 // 10   # in a late chunk of its list
        lists[2] = np.ascontiguousarray(np.insert(lists[2], bad, [[7, 200]], axis=0), np.int32)
        params = [params_for(m) for m in modes]
        adjs = [pack(L, e[:, 0], e[:, 1]) for L, e in zip(Ls, distinct)]
        ref, rl = h.max_clique_batch_each(adjs, params, buffers=clique_lists(len(adjs), 256))
        for i, (adj, m) in enumerate(zip(adjs, modes)):
            want, clique = expected_record(h, adj, m)
            assert_record(ref[i], want, i)
            assert rl[i]["clique"].tobytes() == clique.astype(np.int32).tobytes(), i
        keep = [device_copy(e) for e in lists]
        device = [Graph(t.data_ptr(), None, t.shape[0], L, 0) for t, L in zip(keep, Ls)]
        for kind, gs in ((MEM_HOST, list(zip(Ls, lists))), (MEM_DEVICE, device)):
            recs, gl = h.max_clique_batch_each(gs, params, kind, buffers=clique_lists(len(gs), 256))
            for i in range(len(Ls)):
                if i == 2:
                    r = recs[i]
                    assert r["status"] == BAD_ARG and r["n_corr"] == 200 and r["clique_size"] == 0 and r["n_edges"] == 0, kind
                    continue
                assert recs[i].tobytes() == ref[i].tobytes(), (kind, i)
                assert recs[i]["n_edges"] == len(distinct[i]), (kind, i)
                assert gl[i]["clique"].tobytes() == rl[i]["clique"].tobytes(), (kind, i)
    finally:
        h.close()


# ---- GPU 7: whole-call rejections -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rejections_write_nothing_and_name_the_entry(handle):
    import torch
    ok = pack(40, [1, 2], [2, 3])
    edges = np.array([[0, 1]], np.int32)
    t = torch.zeros(16, dtype=torch.int32, device="cuda")
    host_e = np.zeros(8, np.int32)
    cases = [
        ("L is outside", [ok, Graph(None, None, 0, handle.cfg.max_corr + 1, 0)], MEM_HOST, None, None),
        ("L is outside", [Graph(None, None, 0, -1, 0)], MEM_HOST, None, None),
        ("both given", [Graph(edges.ctypes.data, ok.ctypes.data, 1, 40, 2)], MEM_HOST, None, None),
        ("neither", [Graph(None, None, 3, 40, 0)], MEM_HOST, None, None),
        ("n_edges < 0", [Graph(edges.ctypes.data, None, -1, 40, 0)], MEM_HOST, None, None),
        ("words_per_row", [ok, Graph(None, ok.ctypes.data, 0, 40, 1)], MEM_HOST, None, None),
        ("not memory of the handle", [Graph(host_e.ctypes.data, None, 1, 40, 0)], MEM_DEVICE, None, None),
        ("misaligned", [Graph(t.data_ptr() + 4, None, 1, 40, 0)], MEM_DEVICE, None, None),
        ("misaligned", [Graph(None, t.data_ptr() + 2, 0, 8, 1)], MEM_DEVICE, None, None),
        ("params entry 1", [ok, ok], MEM_HOST, [params_for(PMC_HEU), params_for(3)], None),
        ("params entry 0", [ok], MEM_HOST, [params_for(7)], None),
        ("params entry 0", [ok], MEM_HOST, [params_for(PMC_EXACT, node_limit=-1)], None),
        ("only a clique", [ok], MEM_HOST, None, ListBuffers(1, 8, MEM_HOST, ("clique", "final_inliers"))),
        ("cap_per_pair", [ok], MEM_HOST, None, ListBuffers(1, handle.cfg.max_corr + 1, MEM_HOST, GRAPH_LISTS)),
    ]
    lib = handle.lib
    for why, gs, kind, ps, lb in cases:
        arr, keep = handle.graph_array(gs)
        ps = ps or [params_for(PMC_HEU)] * len(gs)
        out = np.zeros(len(gs), RESULT_DTYPE)
        out.view(np.uint8)[...] = 0xA5
        lb = lb or clique_lists(len(gs), 8)
        for a in lb.arrays.values():
            a.view(np.uint8)[...] = 0xA5
        for fn in NEW:
            rc = getattr(lib, fn)(handle.h, arr, len(gs), handle.params_array(ps), kind, out.ctypes.data, C.byref(lb.descriptor()))
            handle.register_batch_flush()
            assert rc == BAD_ARG, (why, fn)
            assert why in lib.qb200_last_error(handle.h).decode(), (why, lib.qb200_last_error(handle.h))
            assert (out.view(np.uint8) == 0xA5).all(), why
            assert all((a.view(np.uint8) == 0xA5).all() for a in lb.arrays.values()), why
    assert lib.qb200_max_clique_batch_each(handle.h, None, -1, None, MEM_HOST, None, None) == BAD_ARG
    assert lib.qb200_max_clique_batch_each(handle.h, handle.graph_array([ok])[0], 1, handle.params_array([params_for(PMC_HEU)]), MEM_HOST,
                                           None, None) == BAD_ARG
    del t


# ---- GPU 8: one queued stream -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_enqueue_interleaved_with_raw_and_set_batches(handle):
    rng = np.random.default_rng(15)
    graphs = [pack(L, *random_graph(rng, L).T) for L in (50, 400, 33, 900, 128, 7, 2000, 60, 300, 1000, 12)]
    gparams = [params_for(MODES[i % 3]) for i in range(len(graphs))]
    pairs = [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(1600, 1603)]
    pp = default_params()
    pp.rot_noise_bound = 0.6
    sets = [synth.matched_pairs(s, 300)[:2] for s in range(1700, 1712)]
    # blocking references
    g_ref, g_lists = handle.max_clique_batch_each(graphs, gparams, buffers=clique_lists(len(graphs), 4096))
    raw_ref = handle.register_batch(pairs, pp)
    set_ref, _ = handle.solve_batch_each(sets, [pp] * len(sets))
    # one stream: graphs, raw pairs, graphs again, sets; one flush
    ga, gkeep = handle.graph_array(graphs)
    pa, pkeep = handle.pair_array(pairs)
    sa, skeep = handle._set_array(sets, MEM_HOST)
    outs = [np.zeros(len(graphs), RESULT_DTYPE), np.zeros(len(pairs), RESULT_DTYPE), np.zeros(len(graphs), RESULT_DTYPE),
            np.zeros(len(sets), RESULT_DTYPE)]
    lbs = [clique_lists(len(graphs), 4096), clique_lists(len(graphs), 4096)]
    handle.max_clique_batch_enqueue_each_raw(ga, len(graphs), handle.params_array(gparams), MEM_HOST, outs[0], lbs[0])
    handle.register_batch_enqueue_raw(pa, len(pairs), pp, MEM_HOST, outs[1])
    handle.max_clique_batch_enqueue_each_raw(ga, len(graphs), handle.params_array(gparams), MEM_HOST, outs[2], lbs[1])
    handle.solve_batch_enqueue_each_raw(sa, len(sets), handle.params_array([pp] * len(sets)), MEM_HOST, outs[3])
    handle.register_batch_flush()
    assert outs[0].tobytes() == g_ref.tobytes() and outs[2].tobytes() == g_ref.tobytes()
    assert outs[1].tobytes() == raw_ref.tobytes() and outs[3].tobytes() == set_ref.tobytes()
    for lb in lbs:
        for i, d in enumerate(lb.trimmed(outs[0])):
            assert d["clique"].tobytes() == g_lists[i]["clique"].tobytes(), i


# ---- GPU 9: clipped lists, stage times ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_clipped_lists_carry_the_flag_and_stage_times(handle):
    rng = np.random.default_rng(16)
    graphs = [pack(L, *random_graph(rng, L).T) for L in (200, 500, 64, 1000)]
    params = [params_for(PMC_EXACT)] * len(graphs)
    full, fl = handle.max_clique_batch_each(graphs, params, buffers=clique_lists(len(graphs), 4096))
    ms = handle.stage_ms()
    assert ms[4] > 0 and ms[5] > 0 and ms[0] > 0 and ms[7] > 0 and ms[1] == ms[2] == ms[3] == ms[6] == 0, ms
    cap = int(min(full["clique_size"])) - 1
    assert cap >= 1
    recs, cl = handle.max_clique_batch_each(graphs, params, buffers=clique_lists(len(graphs), cap))
    for i in range(len(graphs)):
        assert recs[i]["flags"] == full[i]["flags"] | LISTS_TRUNCATED, i
        assert cl[i]["clique"].tobytes() == fl[i]["clique"][:cap].tobytes(), i
    recs, _ = handle.max_clique_batch_each(graphs, params)
    assert recs.tobytes() == full.tobytes()


# ---- GPU 10: the C++ shim --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_the_shim_equals_the_batch_call(tmp_path, wide):
    exe = build_shim(tmp_path)
    rng = np.random.default_rng(17)
    graphs = [(L, random_graph(rng, L)) for L in (0, 1, 30, 150, 700, 5000)]
    for mode in MODES:
        txt = [f"{len(graphs)} {mode} 1"]
        for L, e in graphs:
            txt.append(f"{L} {len(e)}")
            txt += [f"{a} {b}" if k % 2 else f"{b} {a}" for k, (a, b) in enumerate(e.tolist())]
        (tmp_path / "g.txt").write_text("\n".join(txt) + "\n")
        r = subprocess.run([str(exe), str(tmp_path / "g.txt")], capture_output=True, text=True)
        assert r.returncode == 0, (r.returncode, r.stderr)
        lines = r.stdout.split("\n")
        recs, gl = wide.max_clique_batch_each(graphs, [params_for(mode, 1.0)] * len(graphs), buffers=clique_lists(len(graphs), 4096))
        for i in range(len(graphs)):
            assert lines[2 * i] == f"edges {recs[i]['n_edges']}", (mode, i)
            want = " ".join(["clique", str(recs[i]["clique_size"])] + [str(x) for x in gl[i]["clique"]])
            assert lines[2 * i + 1] == want, (mode, i)
