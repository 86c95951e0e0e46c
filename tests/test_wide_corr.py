"""Pairs of up to QB200_MAX_CORR = 32768 correspondences and cliques of any size.

Graphs above 8192 vertices keep the k-core and clique arrays in a per-pair global scratch instead of shared memory, cliques above
4096 members the pose workspace; the choice is made per pair from its L (or clique size), so the sizes 8191 / 8192 / 8193 and
4095 / 4096 / 4097 sit on both sides of the switch.  Everything is compared bit for bit with the CPU oracle, whose results are
computed once per module (the graph alone is 5e8 literal fp64 tests at L = 32768)."""
import re
import subprocess

import numpy as np
import pytest

from quatro_b200 import synth
from quatro_b200.capi import (COTE_WEIGHTED_MEAN, FLAG_CLIQUE_TRUNCATED, INLIER_NONE, KCORE_HEU, PMC_EXACT, PMC_HEU, RESULT_DTYPE, Handle,
                              QuatroB200Error, default_params)
from support import ROOT, assert_same_record, build_against_lib
MAX_CORR = 32768
GRAPH_SIZES = (8193, 12000, 20000, 32768)


# ---- argument validation and the C++ layer (no GPU needed) -------------------------------------------------------------------

def test_largest_max_corr_passes_validation():
    try:
        h = Handle(max_batch_slots=1, max_corr=MAX_CORR)
    except QuatroB200Error as e:
        assert e.code == -2, e  # QB200_ERR_NO_DEVICE: validation passed, the device probe failed
    else:
        h.close()


@pytest.mark.parametrize("max_corr", [MAX_CORR + 32, 2 * MAX_CORR])
def test_max_corr_beyond_the_limit_is_refused(max_corr):
    with pytest.raises(QuatroB200Error) as e:
        Handle(max_batch_slots=1, max_corr=max_corr)
    assert e.value.code == -1  # QB200_ERR_BAD_ARG, decided before any device is probed


def test_header_defines_the_limit():
    txt = (ROOT / "include" / "quatro_b200.h").read_text()
    assert re.search(r"#define\s+QB200_MAX_CORR\s+32768\b", txt)


FIXTURE = "tests/fixtures/wide_corr_shim.cpp"


def test_wide_corr_shim_compiles(tmp_path):
    build_against_lib(tmp_path, FIXTURE)


# ---- graph helpers ---------------------------------------------------------------------------------------------------------

def pack_edges(n, i, j):
    """Symmetric packed adjacency ((n, ceil(n/32)) uint32, bit u of row v = edge) from an edge list; self loops dropped."""
    i, j = np.asarray(i, np.int64), np.asarray(j, np.int64)
    keep = i != j
    r, c = np.concatenate([i[keep], j[keep]]), np.concatenate([j[keep], i[keep]])
    W = (n + 31) // 32
    adj = np.zeros(n * W, np.uint32)
    np.bitwise_or.at(adj, r * W + (c >> 5), (np.uint32(1) << (c & 31).astype(np.uint32)))
    return adj.reshape(n, W)


def gnp_edges(rng, n, p):
    m = rng.binomial(n * (n - 1) // 2, p)
    return rng.integers(0, n, m), rng.integers(0, n, m)


def clique_edges(members):
    m = np.asarray(members)
    a, b = np.triu_indices(len(m), 1)
    return m[a], m[b]


def g_gnp(n, p, seed, planted=0):
    rng = np.random.default_rng(seed)
    i, j = gnp_edges(rng, n, p)
    if planted:
        ci, cj = clique_edges(np.sort(rng.choice(n, planted, replace=False)))
        i, j = np.concatenate([i, ci]), np.concatenate([j, cj])
    return pack_edges(n, i, j)


def g_hub(n, seed):
    """vertex n // 3 adjacent to every other vertex (degree n - 1, the largest u16 degree at n = 32768) over a sparse G(n, p)"""
    rng = np.random.default_rng(seed)
    i, j = gnp_edges(rng, n, 3.0 / n)
    hub = n // 3
    o = np.arange(n)
    return pack_edges(n, np.concatenate([i, np.full(n, hub)]), np.concatenate([j, o]))


def g_disjoint(n, k):
    """disjoint cliques of k vertices (the last one shorter): many vertices of equal degree in every bucket"""
    ii, jj = [], []
    for s in range(0, n, k):
        a, b = clique_edges(np.arange(s, min(n, s + k)))
        ii.append(a); jj.append(b)
    return pack_edges(n, np.concatenate(ii), np.concatenate(jj))


def reg_set(L, seed, ratio=0.05, shift=0.0):
    a4, b4, _, _ = synth.matched_pairs(seed, L, inlier_ratio=ratio, noise=0.05)
    a4[:, :3] += shift
    b4[:, :3] += shift
    return a4, b4


def tied_set(L, seed, ratio, dup=0):
    """A registration set whose inliers share one exact z offset (every inlier's z COTE value is the same double) and, with dup > 0,
    the first dup correspondences repeated: tied (value, index) keys all over the COTE sorts."""
    a4, b4, T, inl = synth.matched_pairs(seed, L, inlier_ratio=ratio, noise=0.05)
    a4[:, 2] = np.round(a4[:, 2] * 4) / 4
    b4[inl, 2] = a4[inl, 2] + np.float32(0.5)
    if dup:
        a4[L - dup:] = a4[:dup]
        b4[L - dup:] = b4[:dup]
    return a4, b4


def junction_set(L, seed):
    """z COTE values 1.0 for the first half of the set and 0.5 for the second: with a COTE range of 0.25 the first half's interval
    starts exactly where the second half's ends, and the stable (value, index) order puts those 2 x L/2 tied events in the order that
    makes every correspondence overlap -- the optimum of the sweep sits inside the tie"""
    a4, b4, _, _ = synth.matched_pairs(seed, L, inlier_ratio=0.5, noise=0.05)
    a4[:, 2] = np.round(a4[:, 2] * 4) / 4
    b4[:, 2] = a4[:, 2] + np.where(np.arange(L) < L // 2, np.float32(1.0), np.float32(0.5)).astype(np.float32)
    return a4, b4


# ---- fixtures ----------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def h1():
    """one slot, the hall pair's voxel capacity and 32768 correspondences"""
    with Handle(max_batch_slots=1, max_raw_points=524288, max_voxel_points=262144, max_corr=MAX_CORR) as h:
        yield h


@pytest.fixture(scope="module")
def h4():
    with Handle(max_batch_slots=4, max_corr=MAX_CORR) as h:
        yield h


@pytest.fixture(scope="module")
def reg_graphs(oracle):
    """registration sets and their oracle graphs at GRAPH_SIZES, plus one set shifted 400 m from the origin (wide K8 error band)"""
    out = {}
    for L in GRAPH_SIZES:
        a4, b4 = reg_set(L, 500 + L)
        out[L] = (a4, b4, *oracle.build_graph(a4, b4, 0.3, 1.0))
    a4, b4 = reg_set(12000, 77, ratio=0.2, shift=400.0)
    out["shifted"] = (a4, b4, *oracle.build_graph(a4, b4, 0.3, 1.0))
    return out


def _clique_graphs(reg_graphs):
    gs = [(f"registration L={L}", reg_graphs[L][2]) for L in GRAPH_SIZES]
    gs += [(f"G({n}, 0.003)", g_gnp(n, 0.003, n, planted=40)) for n in (8191, 8192, 8193)]   # the shared / global switch of K9
    gs += [("G(12000, 0.01)", g_gnp(12000, 0.01, 3)), ("G(32768, 0.002)", g_gnp(32768, 0.002, 4))]
    gs += [("planted 20000", g_gnp(20000, 0.002, 5, planted=300)), ("planted 32768", g_gnp(32768, 0.001, 6, planted=500))]
    gs += [("hub 32768", g_hub(32768, 7)), ("hub 8193", g_hub(8193, 8))]
    gs += [("disjoint 12000", g_disjoint(12000, 60)), ("disjoint 32768", g_disjoint(32768, 64))]
    return gs


@pytest.fixture(scope="module")
def clique_cases(reg_graphs, oracle):
    cases = []
    for name, adj in _clique_graphs(reg_graphs):
        cases.append((name, adj, PMC_HEU, 0.5, oracle.max_clique(adj, PMC_HEU)))
    for L in (8193, 32768):
        adj = reg_graphs[L][2]
        for thr in (0.5, 0.0005):
            cases.append((f"kcore-heu {thr} L={L}", adj, KCORE_HEU, thr, oracle.max_clique(adj, KCORE_HEU, thr)))
    return cases


# ---- 1. graph ----------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_graph_bit_exact_up_to_32768(h1, reg_graphs):
    for key, (a4, b4, adj_r, deg_r, ne_r) in reg_graphs.items():
        adj_g, deg_g, ne_g = h1.build_graph(a4, b4, 0.3, 1.0)
        assert np.array_equal(adj_g, adj_r), key
        assert np.array_equal(deg_g, deg_r) and ne_g == ne_r, key


# ---- 2. k-core + heuristic clique --------------------------------------------------------------------------------------------

def _check_clique(h, cases):
    for name, adj, mode, thr, ref in cases:
        got = h.max_clique(adj, mode, thr)
        assert got[3] == ref[3], f"{name}: max core"
        assert np.array_equal(got[1], ref[1]), f"{name}: core numbers differ"
        assert np.array_equal(got[2], ref[2]), f"{name}: peel order differs"
        assert np.array_equal(got[0], ref[0]), f"{name}: clique differs"


@pytest.mark.gpu
def test_kcore_and_clique_bit_exact_up_to_32768(h1, clique_cases):
    _check_clique(h1, clique_cases)


@pytest.mark.gpu
def test_kcore_and_cliques_on_a_16384_handle(clique_cases, exact_cases):
    """max_corr 16384: 512-word rows, 16 adjacency words per lane (kcore_kernel<16>, clique_descent<16>, clique_exact_kernel<16>)"""
    with Handle(max_batch_slots=1, max_corr=16384) as h:
        _check_clique(h, [c for c in clique_cases if len(c[1]) <= 16384])
        assert _check_exact(h, [c for c in exact_cases if c[0] <= 16384])[0] >= 1


def test_hub_reaches_the_largest_degree():
    adj = g_hub(MAX_CORR, 7)
    assert int(np.unpackbits(adj[MAX_CORR // 3].view(np.uint8)).sum()) == MAX_CORR - 1


# ---- 3. exact clique ---------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def exact_cases(oracle):
    """sparse wide graphs with a dense random core: the heuristic clique is not maximum there, the search improves it"""
    cases = []
    for n, core, p, seed, limit in ((9000, 150, 0.5, 11, 0), (20000, 120, 0.5, 12, 0), (32768, 150, 0.5, 13, 0), (20000, 120, 0.5, 12, 300)):
        rng = np.random.default_rng(seed)
        i, j = gnp_edges(rng, n, 4.0 / n)
        m = np.sort(rng.choice(n, core, replace=False))
        ci, cj = clique_edges(m)
        sel = rng.uniform(size=len(ci)) < p
        adj = pack_edges(n, np.concatenate([i, ci[sel]]), np.concatenate([j, cj[sel]]))
        ref = oracle.max_clique_ex(adj, PMC_EXACT, 0.5, limit)
        heu = oracle.max_clique(adj, PMC_HEU)
        cases.append((n, limit, adj, ref, len(heu[0])))
    return cases


def _check_exact(h, cases):
    improved = truncated = 0
    for n, limit, adj, ref, heu in cases:
        got = h.max_clique_ex(adj, PMC_EXACT, 0.5, limit)
        assert got[3] == ref[3] and got[4] == ref[4], (n, limit, got[3:], ref[3:])
        assert np.array_equal(got[1], ref[1]) and np.array_equal(got[2], ref[2]), (n, limit)
        assert np.array_equal(got[0], ref[0]), (n, limit)
        improved += len(ref[0]) > heu
        truncated += bool(ref[4] & FLAG_CLIQUE_TRUNCATED)
    return improved, truncated


@pytest.mark.gpu
def test_exact_clique_on_wide_graphs(h1, exact_cases):
    improved, truncated = _check_exact(h1, exact_cases)
    assert improved >= 3 and truncated >= 1, (improved, truncated)


# ---- 4. pose with large cliques ----------------------------------------------------------------------------------------------

def _trans_mask_len(res, rot_inl):
    """the translation mask covers the COTE inputs: the rotation inliers when they are used, else the whole clique"""
    return res.n_rot_inliers if rot_inl and res.n_rot_inliers > 0 else res.clique_size


@pytest.mark.gpu
@pytest.mark.parametrize("L", [4095, 4096, 4097, 6000, MAX_CORR])
def test_pose_of_every_correspondence(h1, oracle, L):
    """INLIER_NONE: the clique is all L correspondences; 4096 / 4097 sit on the shared / global switch of the pose workspace"""
    tied, junction = tied_set(L, 900 + L, 0.4, dup=L // 8), junction_set(L, 950 + L)
    for st, mode, rot_inl in ((tied, 0, 0), (tied, COTE_WEIGHTED_MEAN, 1), (junction, 0, 0), (junction, COTE_WEIGHTED_MEAN, 0)):
        a4, b4 = st
        p = default_params()
        p.inlier_selection_mode, p.cote_mode, p.using_rot_inliers_when_estimating_cote = INLIER_NONE, mode, rot_inl
        if st is junction:
            p.cote_noise_bound = 0.25
        r_g, st_g = h1.solve_correspondences(a4, b4, p)
        r_o, st_o, c_o, f_o = oracle.solve_correspondences(a4, b4, p, want_sets=True)
        assert st_g == st_o == 0 and r_g.clique_size == L
        assert_same_record(r_g, r_o)
        assert np.array_equal(h1.last_final_inliers(), f_o)
        clique = np.arange(L, dtype=np.int32)
        res_g, rm_g, tm_g, _ = h1.solve_pose(a4, b4, clique, p)
        res_o, rm_o, tm_o, _ = oracle.solve_pose(a4, b4, clique, p)
        n = _trans_mask_len(res_o, rot_inl)
        assert np.array_equal(rm_g, rm_o) and np.array_equal(tm_g[:n], tm_o[:n])
        assert_same_record(res_g, res_o)


@pytest.mark.gpu
def test_pose_of_a_clique_above_4096(h1, oracle):
    a4, b4 = tied_set(12000, 31, 0.6)
    for mode, rot_inl in ((0, 0), (COTE_WEIGHTED_MEAN, 0), (0, 1)):
        p = default_params()
        p.cote_mode, p.using_rot_inliers_when_estimating_cote = mode, rot_inl
        r_g, st_g = h1.solve_correspondences(a4, b4, p)
        r_o, st_o, c_o, f_o = oracle.solve_correspondences(a4, b4, p, want_sets=True)
        assert st_g == st_o == 0 and r_o.clique_size > 4096
        assert_same_record(r_g, r_o)
        assert np.array_equal(h1.last_clique(), c_o) and np.array_equal(h1.last_final_inliers(), f_o)
        res_g, rm_g, tm_g, _ = h1.solve_pose(a4, b4, c_o, p)
        res_o, rm_o, tm_o, _ = oracle.solve_pose(a4, b4, c_o, p)
        n = _trans_mask_len(res_o, rot_inl)
        assert np.array_equal(rm_g, rm_o) and np.array_equal(tm_g[:n], tm_o[:n])


# ---- 5. batch of mixed sizes -------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_solve_batch_mixed_sizes(h4, oracle):
    sets = [reg_set(100, 41, 0.3), reg_set(5000, 42, 0.1), tied_set(20000, 43, 0.3), reg_set(MAX_CORR, 44, 0.05)]
    p = default_params()
    out = h4.solve_batch(sets, p)
    single = np.frombuffer(b"".join(bytes(h4.solve_correspondences(a, b, p)[0]) for a, b in sets), RESULT_DTYPE)
    assert out.tobytes() == single.tobytes()
    for k, (a, b) in enumerate(sets):
        r_o, st_o = oracle.solve_correspondences(a, b, p)
        assert out[k]["status"] == st_o == 0 and out[k]["n_corr"] == len(a)
        assert (out[k]["clique_size"], out[k]["max_core"], out[k]["n_edges"], out[k]["n_final_inliers"], out[k]["gnc_iters"]) == \
               (r_o.clique_size, r_o.max_core, r_o.n_edges, r_o.n_final_inliers, r_o.gnc_iters)
        assert np.allclose(np.asarray(out[k]["T"]).reshape(4, 4).T, r_o.matrix(), atol=1e-9, rtol=0)


# ---- 6. the hall pair end to end, every mutual neighbour a correspondence --------------------------------------------------------

def hall_params():
    p = default_params()
    p.voxel_size, p.normal_radius, p.fpfh_radius, p.noise_bound, p.cote_noise_bound, p.skip_flagged = 0.05, 0.10, 0.15, 0.05, 0.05, 0
    p.use_tuple_test = 0
    p.rot_noise_bound = 2 * p.noise_bound   # what a fresh handle latches; h1 has latched the default pairs' bound already
    return p


@pytest.mark.gpu
def test_register_hall_pair_without_tuple_test(h1, oracle):
    src, tgt, T = synth.indoor_pair(0, extent=9.0)
    ref, st_ref = oracle.register_pair(src, tgt, hall_params())
    assert st_ref == 0 and 8192 < ref.n_corr <= MAX_CORR
    got, st = h1.register_pair(src, tgt, hall_params())
    assert st == 0 and got.valid == 1
    assert_same_record(got, ref)


# ---- 7. the C++ layer --------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_cpp_shim_grows_to_wide_sets(tmp_path, oracle):
    exe = build_against_lib(tmp_path, FIXTURE)
    a4, b4 = reg_set(10000, 61, 0.3)
    (tmp_path / "a.bin").write_bytes(np.ascontiguousarray(a4, np.float32).tobytes())
    (tmp_path / "b.bin").write_bytes(np.ascontiguousarray(b4, np.float32).tobytes())
    r = subprocess.run([str(exe), str(tmp_path / "a.bin"), str(tmp_path / "b.bin")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "WIDE_CORR_SHIM_OK" in r.stdout, r.stdout + r.stderr
    out = {ln.split()[0]: ln.split()[1:] for ln in r.stdout.splitlines() if ln and not ln.startswith("T ")}
    T_cpp = np.array([list(map(float, ln.split()[1:])) for ln in r.stdout.splitlines() if ln.startswith("T ")])
    ref, st = oracle.solve_correspondences(a4, b4, default_params())
    assert st == 0 and int(out["corr"][0]) == 10000 and int(out["clique"][0]) == ref.clique_size
    assert np.allclose(T_cpp, ref.matrix(), atol=1e-9)
