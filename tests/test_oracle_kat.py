"""Known-answer tests that pin the CPU oracle (SURVEY.md 8c, KAT-1..13).  The reference ships no
tests or golden vectors, so these hand-computable cases are the pins."""
import numpy as np
import pytest

from conftest import adj_to_dense, dense_to_adj
from quatro_b200 import synth
from quatro_b200.capi import default_params, PMC_HEU, KCORE_HEU, COTE_WEIGHTED_MEAN
from support import P4


# ---- KAT-1 voxel ------------------------------------------------------------------------------
def test_kat1_voxel_lattice(oracle):
    # two points in each cell of a 3x3x3 lattice (leaf 1.0): centroid = mean, order = ascending (k,j,i)
    pts, exp = [], []
    for k in range(3):
        for j in range(3):
            for i in range(3):
                a = np.array([i + 0.25, j + 0.25, k + 0.25])
                b = np.array([i + 0.75, j + 0.5, k + 0.25])
                pts += [a, b]
                exp.append((a.astype(np.float32) + b.astype(np.float32)) / np.float32(2))
    pts = np.array(pts)
    perm = np.random.default_rng(0).permutation(len(pts))
    out, st = oracle.voxelize(P4(pts[perm]), 1.0, 0)
    assert st == 0 and len(out) == 27
    np.testing.assert_array_equal(out[:, :3], np.array(exp, np.float32))
    assert np.all(out[:, 3] == 1.0)


def test_voxel_skips_nonfinite_and_flagged(oracle):
    pts = P4([[0.1, 0.1, 0.1], [np.nan, 0, 0], [0.2, 0.1, 0.1], [5, 5, 5]])
    pts[3, 3] = -1.0
    out, _ = oracle.voxelize(pts, 0.3, 1)
    assert len(out) == 1 and np.allclose(out[0, :3], [0.15, 0.1, 0.1])
    out, _ = oracle.voxelize(pts, 0.3, 0)
    assert len(out) == 2
    out, _ = oracle.voxelize(P4(np.zeros((0, 3))), 0.3, 1)
    assert len(out) == 0


def test_voxel_negative_coordinates_floor(oracle):
    # floor semantics: -0.1 and +0.1 are different cells at leaf 0.3
    out, _ = oracle.voxelize(P4([[-0.1, 0, 0], [0.1, 0, 0]]), 0.3, 0)
    assert len(out) == 2 and out[0, 0] < 0 < out[1, 0]


# ---- neighbour search vs brute force ---------------------------------------------------------------
def test_neighbors_match_bruteforce(oracle):
    rng = np.random.default_rng(3)
    pts = P4(rng.uniform(-3, 3, (800, 3)))
    for q in (0, 17, 799):
        for r, cell in ((0.5, 0.3), (0.75, 0.3), (0.6, 0.3), (0.5, 0.5)):
            idx, d2 = oracle.neighbors(pts, cell, q, r)
            d = pts[:, :3] - pts[q, :3]
            d2b = ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]).astype(np.float32) + d[:, 2] * d[:, 2]).astype(np.float32)
            ref = np.nonzero(d2b < np.float32(r * r))[0]
            assert sorted(idx.tolist()) == ref.tolist()
            assert q in idx


# ---- KAT-2 normals ---------------------------------------------------------------------------------
def test_default_lattice_cell_covers_the_radius_with_27_cells(oracle):
    """D8: the default cell (1 + 2^-9) r makes a 3 x 3 x 3 cell walk sufficient even when x / cell rounds across a cell
    boundary.  Adversarial clouds: points within a few ulps of cell boundaries, at KITTI-scale coordinates, pairs at
    distances just inside / outside the radius; the lattice walk must return exactly the brute-force set {d2 < r2}."""
    rng = np.random.default_rng(7)
    r = np.float32(0.75)
    cell = np.float32(r * np.float32(1.001953125))
    r2 = np.float32(np.float64(r) * np.float64(r))
    n = 4000
    base = rng.integers(-160, 160, (n, 3)).astype(np.float32) * cell          # exactly on cell boundaries ...
    jitter = rng.choice(np.array([0.0, 1e-6, -1e-6, 1e-4, -1e-4, 0.3, -0.3, 0.7499, -0.7499, 0.7501], np.float32), (n, 3))
    pts = (base + jitter).astype(np.float32)
    # a dense cluster so that many pairs sit right at the radius
    c0 = np.array([37, -12, 2], np.float32) * cell
    ring = rng.normal(size=(600, 3)).astype(np.float32)
    ring = c0 + ring / np.linalg.norm(ring, axis=1, keepdims=True) * rng.choice(np.array([0.7499995, 0.75, 0.7500005, 0.4], np.float32), (600, 1))
    pts = np.vstack([pts, c0[None], ring]).astype(np.float32)
    p4 = np.concatenate([pts, np.ones((len(pts), 1), np.float32)], 1)
    for q in list(rng.integers(0, len(pts), 60)) + [n]:                            # n = the cluster centre
        idx, d2 = oracle.neighbors(p4, float(cell), int(q), float(r), cap=len(pts))
        d = pts[q][None, :] - pts
        bf = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]).astype(np.float32) + (d[:, 2] * d[:, 2]).astype(np.float32)   # the walk's own expression
        want = np.nonzero(bf < r2)[0]
        assert np.array_equal(np.sort(idx), want), (q, len(idx), len(want))


def test_kat2_plane_normals(oracle):
    g = np.arange(-2, 2.01, 0.25)
    xx, yy = np.meshgrid(g, g)
    ground = np.stack([xx.ravel(), yy.ravel(), np.full(xx.size, -1.7)], 1)
    nrm, _ = oracle.compute_fpfh(P4(ground), 0.5, 0.75, 0.3)
    inner = (np.abs(ground[:, 0]) < 1.4) & (np.abs(ground[:, 1]) < 1.4)
    assert np.allclose(nrm[inner, :3], [0, 0, 1], atol=1e-3)  # flipped towards the origin (above the plane)
    wall = np.stack([np.full(xx.size, 5.0), xx.ravel(), yy.ravel()], 1)
    nrm, _ = oracle.compute_fpfh(P4(wall), 0.5, 0.75, 0.3)
    assert np.allclose(nrm[inner, :3], [-1, 0, 0], atol=1e-3)
    assert np.all(nrm[inner, 3] < 1e-3)  # curvature ~ 0 on a plane


def test_normals_need_three_neighbours(oracle):
    pts = P4([[0, 0, 0], [0.1, 0, 0], [10, 10, 10]])
    nrm, desc = oracle.compute_fpfh(pts, 0.5, 0.75, 0.3)
    assert np.all(np.isnan(nrm[:, :3]))
    assert np.all(desc[2] == 0)           # isolated point: all-zero descriptor
    assert np.all(np.isfinite(desc))      # NaN normals go to bin 0 (D6), never into the histogram values
    assert desc[0, 0] == pytest.approx(100.0) and desc[0, 11] == pytest.approx(100.0) and desc[0, 22] == pytest.approx(100.0)


# ---- KAT-3 pair features ---------------------------------------------------------------------------
def test_kat3_pair_features(oracle):
    # p1 at origin with n1 = +z, p2 at +x with n2 = +x.
    # angle1 = 0, angle2 = 1 -> acos(0) > acos(1): roles swap: n1c = +x, n2c = +z, dp = -x, f3 = -angle2 = -1
    # v = dp x n1c = 0 -> degenerate -> rejected
    ok, f = oracle.pair_features([0, 0, 0], [0, 0, 1], [1, 0, 0], [1, 0, 0])
    assert not ok
    # n1 = +z at origin, p2 = (1,0,0) n2 = (0, 1, 0): angle1 = angle2 = 0 -> no swap, f3 = 0
    # v = dp x n1 = (1,0,0)x(0,0,1) = (0,-1,0); w = n1 x v = (0,0,1)x(0,-1,0) = (1,0,0)
    # f2 = v.n2 = -1 ; f1 = atan2(w.n2, n1.n2) = atan2(0, 0) = 0
    ok, f = oracle.pair_features([0, 0, 0], [0, 0, 1], [1, 0, 0], [0, 1, 0])
    assert ok and f[0] == 0.0 and f[1] == -1.0 and f[2] == 0.0
    # coplanar parallel normals: f1 = atan2(0, 1) = 0, f2 = 0, f3 = 0
    ok, f = oracle.pair_features([0, 0, 0], [0, 0, 1], [0.5, 0.2, 0], [0, 0, 1])
    assert ok and np.allclose(f, 0, atol=1e-7)
    ok, _ = oracle.pair_features([1, 2, 3], [0, 0, 1], [1, 2, 3], [0, 0, 1])  # zero distance
    assert not ok


# ---- KAT-4 planar patch FPFH -----------------------------------------------------------------------
def test_kat4_plane_fpfh(oracle):
    g = np.arange(-3, 3.01, 0.3)
    xx, yy = np.meshgrid(g, g)
    pts = np.stack([xx.ravel(), yy.ravel(), np.full(xx.size, -1.7)], 1)
    nrm, desc, spfh = oracle.compute_fpfh(P4(pts), 0.5, 0.75, 0.3, want_spfh=True)
    inner = (np.abs(pts[:, 0]) < 1.5) & (np.abs(pts[:, 1]) < 1.5)
    d = desc[inner]
    # every third sums to 100; the mass sits in the bins containing f1 = 0, f2 = 0, f3 = 0 (bin 5 of each third)
    for t in range(3):
        assert np.allclose(d[:, 11 * t:11 * t + 11].sum(1), 100.0, atol=1e-3)
    assert np.all(d[:, 16] > 99.0) and np.all(d[:, 27] > 99.0)
    assert np.all(d[:, 5] + d[:, 4] + d[:, 6] > 99.0)  # f1 = atan2(~0, 1) sits on the bin-5 side of 0 +- rounding
    assert np.allclose(spfh[inner].reshape(-1, 3, 11).sum(2), 100.0, atol=1e-3)


# ---- KAT-5 / KAT-6 matcher -------------------------------------------------------------------------
def _rand_desc(rng, n):
    d = rng.uniform(0, 1, (n, 33)).astype(np.float32)
    for t in range(3):
        d[:, 11 * t:11 * t + 11] *= 100.0 / d[:, 11 * t:11 * t + 11].sum(1, keepdims=True)
    return d


def test_kat5_permuted_copy_gives_identity_matches(oracle):
    rng = np.random.default_rng(5)
    n = 300
    src = P4(rng.uniform(-20, 20, (n, 3)))
    desc = _rand_desc(rng, n)
    perm = rng.permutation(n)
    tgt, tdesc = src[perm].copy(), desc[perm].copy()
    p = default_params()
    corr, nm, st = oracle.match(src, desc, tgt, tdesc, p)
    assert nm == n and len(corr) == n          # rigid (identity) motion: every tuple passes
    assert np.array_equal(corr[:, 0], np.arange(n))
    assert np.array_equal(perm[corr[:, 1]], corr[:, 0])


def test_kat6_tuple_test_rejects_scaled_point(oracle):
    rng = np.random.default_rng(6)
    n = 60
    src = P4(rng.uniform(-20, 20, (n, 3)))
    desc = _rand_desc(rng, n)
    yaw = 0.7
    R = np.array([[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]])
    tgt = src.copy()
    tgt[:, :3] = src[:, :3] @ R.T + [3, -2, 0.5]
    bad = 7
    tgt[bad, :3] += [40.0, 40.0, 0]       # breaks every triangle through correspondence 7
    p = default_params()
    corr, nm, _ = oracle.match(src, desc, tgt, desc.copy(), p)
    assert nm == n
    assert bad not in corr[:, 0] and len(corr) == n - 1
    p2 = default_params(); p2.use_tuple_test = 0
    corr2, _, _ = oracle.match(src, desc, tgt, desc.copy(), p2)
    assert len(corr2) == n


def test_matcher_swaps_when_target_is_larger_and_sorts_by_source(oracle):
    rng = np.random.default_rng(8)
    n = 120
    src = P4(rng.uniform(-20, 20, (n, 3)))
    desc = _rand_desc(rng, n)
    extra = P4(rng.uniform(-20, 20, (30, 3)))
    tgt = np.concatenate([extra, src[::-1]])
    tdesc = np.concatenate([_rand_desc(rng, 30), desc[::-1]])
    corr, nm, _, mutual = oracle.match(src, desc, tgt, tdesc, default_params(), want_mutual=True)
    assert np.all(np.diff(mutual[:, 0]) > 0)                 # listed by index in the LARGER cloud (target)
    assert np.all(np.diff(corr[:, 0]) > 0)                   # output sorted by (src, tgt)
    assert np.array_equal(corr[:, 1], 30 + (n - 1 - corr[:, 0]))


def test_matcher_tie_break_lowest_index(oracle):
    src = P4([[0, 0, 0], [1, 0, 0], [0, 1, 0]])
    tgt = P4([[0, 0, 0], [1, 0, 0], [0, 1, 0]])
    d = np.zeros((3, 33), np.float32)    # all identical descriptors: only (0,0) is mutual under lowest-index ties
    p = default_params(); p.use_tuple_test = 0
    corr, nm, _ = oracle.match(src, d, tgt, d, p)
    assert corr.tolist() == [[0, 0]]


# ---- KAT-7 graph -----------------------------------------------------------------------------------
def test_kat7_graph_edges_and_boundary(oracle):
    a4, b4, T, inl = synth.matched_pairs(7, 200, inlier_ratio=0.4, noise=0.02)
    adj, deg, ne = oracle.build_graph(a4, b4, 0.3, 1.0)
    A = adj_to_dense(adj, 200)
    assert np.array_equal(A, A.T) and not A.diagonal().any()
    assert ne == A.sum() // 2 and np.array_equal(deg, A.sum(1))
    ii = np.nonzero(inl)[0]
    assert A[np.ix_(ii, ii)].sum() == len(ii) * (len(ii) - 1)      # inliers form a clique
    a, b = a4[:, :3].astype(np.float64), b4[:, :3].astype(np.float64)
    da = np.linalg.norm(a[:, None] - a[None], axis=2)
    db = np.linalg.norm(b[:, None] - b[None], axis=2)
    clear = np.abs(np.abs(db - da) - 0.6) > 1e-9
    np.fill_diagonal(clear, False)
    assert np.array_equal(A[clear], (np.abs(db - da) <= 0.6)[clear])
    # boundary: |db - da| = 0.6 -/+ 1e-6
    a4 = P4([[0, 0, 0], [10, 0, 0], [0, 0, 0], [10, 0, 0]])
    b4 = P4([[0, 0, 0], [10.599999, 0, 0], [50, 0, 0], [60.600002, 0, 0]])
    A = adj_to_dense(oracle.build_graph(a4, b4, 0.3, 1.0)[0], 4)
    assert A[0, 1] and not A[2, 3]


# ---- KAT-8 k-core ----------------------------------------------------------------------------------
def test_kat8_kcore(oracle):
    n = 7
    K = np.ones((n, n), bool); np.fill_diagonal(K, False)
    k, order, mc = oracle.kcore(dense_to_adj(K))
    assert mc == n - 1 and np.all(k == n)                         # pmc stores core + 1
    assert sorted(order.tolist()) == list(range(n))
    path = np.zeros((5, 5), bool)
    for i in range(4):
        path[i, i + 1] = path[i + 1, i] = True
    k, order, mc = oracle.kcore(dense_to_adj(path))
    assert mc == 1 and np.all(k == 2)
    G = np.zeros((6, 6), bool)
    G[:5, :5] = True; np.fill_diagonal(G, False)
    G[4, 5] = G[5, 4] = True                                       # K5 + pendant
    k, order, mc = oracle.kcore(dense_to_adj(G))
    assert mc == 4 and k.tolist() == [5, 5, 5, 5, 5, 2] and order[0] == 5
    import networkx as nx
    rng = np.random.default_rng(1)
    R = rng.uniform(size=(60, 60)) < 0.15
    R = np.triu(R, 1); R = R | R.T
    k, order, mc = oracle.kcore(dense_to_adj(R))
    cn = nx.core_number(nx.from_numpy_array(R))
    assert [cn[i] + 1 for i in range(60)] == k.tolist() and mc == max(cn.values())
    # the peel order is a valid degeneracy order: core numbers are non-decreasing along it
    assert np.all(np.diff(k[order]) >= 0)


# ---- KAT-9 clique ----------------------------------------------------------------------------------
def test_kat9_planted_clique(oracle):
    import networkx as nx
    rng = np.random.default_rng(9)
    n, q = 150, 25
    R = rng.uniform(size=(n, n)) < 0.03
    R = np.triu(R, 1); R = R | R.T
    members = np.sort(rng.choice(n, q, replace=False))
    R[np.ix_(members, members)] = True
    np.fill_diagonal(R, False)
    clique, k, order, mc = oracle.max_clique(dense_to_adj(R), PMC_HEU)
    assert clique.tolist() == members.tolist()
    assert mc == q - 1                                             # it is the (q-1)-core: lb == ub
    # validity on a random graph without planted structure
    R2 = rng.uniform(size=(80, 80)) < 0.3
    R2 = np.triu(R2, 1); R2 = R2 | R2.T
    c2, *_ = oracle.max_clique(dense_to_adj(R2), PMC_HEU)
    assert len(c2) >= 2 and R2[np.ix_(c2, c2)].sum() == len(c2) * (len(c2) - 1)
    best = max(len(c) for c in nx.find_cliques(nx.from_numpy_array(R2)))
    assert len(c2) <= best
    # empty graph -> no clique (lb = 0)
    c3, *_ = oracle.max_clique(dense_to_adj(np.zeros((10, 10), bool)), PMC_HEU)
    assert len(c3) == 0


# ---- KAT-9b exact clique (PMC_EXACT) against networkx's maximal-clique enumeration -----------------------------------
def test_kat9b_exact_clique_is_maximum(oracle):
    """src/graph.cc:106-127: the exact finder returns a MAXIMUM clique; its size is pinned by an independent enumeration
    (networkx, Bron-Kerbosch), membership is only required to be a clique (pmc's own choice depends on thread timing)."""
    import networkx as nx
    from quatro_b200.capi import PMC_EXACT, FLAG_CLIQUE_TRUNCATED
    rng = np.random.default_rng(91)
    improved = 0
    for n, p_, planted in ((40, 0.3, 0), (60, 0.5, 0), (150, 0.05, 12), (300, 0.1, 0), (600, 0.03, 9), (1200, 0.02, 0), (90, 0.6, 0)):
        R = rng.uniform(size=(n, n)) < p_
        R = np.triu(R, 1); R = R | R.T
        if planted:
            m = rng.choice(n, planted, replace=False)
            R[np.ix_(m, m)] = True
        np.fill_diagonal(R, False)
        adj = dense_to_adj(R)
        heu = oracle.max_clique(adj, PMC_HEU)[0]
        c, k, order, mc, flags = oracle.max_clique_ex(adj, PMC_EXACT)
        best = max(len(x) for x in nx.find_cliques(nx.from_numpy_array(R)))
        assert flags == 0 and len(c) == best, (n, p_, len(c), best)
        assert np.all(np.diff(c) > 0) and R[np.ix_(c, c)].sum() == len(c) * (len(c) - 1)
        assert len(heu) <= best <= mc + 1
        if len(heu) == best:
            assert c.tolist() == heu.tolist()          # only a strictly larger clique replaces the heuristic one (graph.cc:96-104)
        else:
            improved += 1
    assert improved >= 2                               # the branch and bound really ran
    # node limit: the search stops, says so, and still returns a clique at least as large as the heuristic one
    R = rng.uniform(size=(400, 400)) < 0.6
    R = np.triu(R, 1); R = R | R.T
    adj = dense_to_adj(R)
    heu = oracle.max_clique(adj, PMC_HEU)[0]
    c, *_, flags = oracle.max_clique_ex(adj, PMC_EXACT, 0.5, 2000)
    assert flags & FLAG_CLIQUE_TRUNCATED and len(c) >= len(heu) and R[np.ix_(c, c)].sum() == len(c) * (len(c) - 1)
    c2, *_, flags2 = oracle.max_clique_ex(adj, PMC_EXACT, 0.5, 20000)
    assert len(c2) >= len(c)
    # PMC_HEU / KCORE_HEU through the _ex entry are unchanged
    assert oracle.max_clique_ex(adj, PMC_HEU)[0].tolist() == heu.tolist()


def test_exact_mode_through_the_solver(oracle):
    from quatro_b200 import synth
    from quatro_b200.capi import PMC_EXACT, default_params
    a4, b4, T, inl = synth.matched_pairs(77, 400, inlier_ratio=0.3, noise=0.05)
    p = default_params()
    r_heu, st_heu = oracle.solve_correspondences(a4, b4, p)
    p.inlier_selection_mode = PMC_EXACT
    r_ex, st_ex = oracle.solve_correspondences(a4, b4, p)
    assert st_ex == 0 and r_ex.valid == 1 and r_ex.clique_size >= r_heu.clique_size and r_ex.flags == 0
    rot, tr = synth.pose_error(r_ex.matrix(), T)
    assert rot < 2.0 and tr < 0.3


def test_kcore_heuristic_mode(oracle):
    K = np.ones((8, 8), bool); np.fill_diagonal(K, False)
    G = np.zeros((10, 10), bool); G[:8, :8] = K
    c, *_ = oracle.max_clique(dense_to_adj(G), KCORE_HEU, 0.5)     # max_core 7 > 0.5 * 10 -> k-core shortcut
    assert c.tolist() == list(range(8))


# ---- KAT-10 svd ------------------------------------------------------------------------------------
def test_kat10_svd2x2_and_rotation(oracle):
    rng = np.random.default_rng(10)
    for _ in range(50):
        H = rng.normal(size=(2, 2))
        U, S, V = oracle.svd2x2(H)
        assert np.allclose(U @ np.diag(S) @ V.T, H, atol=1e-12)
        assert np.allclose(U @ U.T, np.eye(2), atol=1e-12) and np.allclose(V @ V.T, np.eye(2), atol=1e-12)
        assert S[0] >= S[1] >= 0
        assert np.allclose(S, np.linalg.svd(H, compute_uv=False), atol=1e-12)
    yaw = 2.1
    R = np.array([[np.cos(yaw), -np.sin(yaw)], [np.sin(yaw), np.cos(yaw)]])
    X = rng.normal(size=(2, 40)); Y = R @ X
    assert np.allclose(oracle.svd_rot2d(X, Y, np.ones(40)), R, atol=1e-12)
    # reflection: best ROTATION must still have det +1 (the V.col(1) fix)
    Y2 = np.diag([1.0, -1.0]) @ X
    R2 = oracle.svd_rot2d(X, Y2, np.ones(40))
    assert np.linalg.det(R2) == pytest.approx(1.0)
    # closed form used on the GPU: theta = atan2(H01 - H10, H00 + H11)
    W = rng.uniform(0.1, 1, 40)
    Y3 = R @ X + rng.normal(0, 0.1, (2, 40))
    H = (X * W) @ Y3.T
    th = np.arctan2(H[0, 1] - H[1, 0], H[0, 0] + H[1, 1])
    assert np.allclose(oracle.svd_rot2d(X, Y3, W), [[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]], atol=1e-12)


# ---- KAT-11 GNC ------------------------------------------------------------------------------------
def test_kat11_gnc(oracle):
    rng = np.random.default_rng(11)
    c = 200
    yaw = -1.3
    R = np.array([[np.cos(yaw), -np.sin(yaw)], [np.sin(yaw), np.cos(yaw)]])
    X = rng.uniform(-30, 30, (2, c))
    Y = R @ X + rng.normal(0, 0.02, (2, c))
    out = rng.uniform(size=c) < 0.5
    Y[:, out] = rng.uniform(-30, 30, (2, out.sum()))
    p = default_params()
    Rg, inl, cost, it = oracle.gnc(X, Y, p, 0.6)
    assert np.allclose(Rg, R, atol=2e-3)
    assert not inl[out].any() or inl[out].mean() < 0.05
    assert inl[~out].all() and 1 < it <= 50
    # noise-free: max residual ~ 0 -> mu <= 0 -> early exit after the first SVD, all weights 1
    Rg, inl, cost, it = oracle.gnc(X, R @ X, p, 0.6)
    assert it == 1 and inl.all() and np.allclose(Rg, R, atol=1e-12)


# ---- KAT-12 COTE -----------------------------------------------------------------------------------
def test_kat12_cote(oracle):
    rng = np.random.default_rng(12)
    X = np.concatenate([4.0 + rng.uniform(-0.2, 0.2, 30), rng.uniform(-50, 50, 20)])
    est, inl = oracle.cote(X, 0.3, median=True)
    assert abs(est - 4.0) < 0.3 and inl[:30].all()
    est_w, _ = oracle.cote(X, 0.3, median=False)
    assert abs(est_w - 4.0) < 0.3
    # literal "median" = mean of the two middle candidates among the events preceding the optimum
    assert oracle.cote(np.array([1.0, 1.2]), 0.3)[0] == pytest.approx(1.1)
    est3, inl3 = oracle.cote(np.array([1.0, 1.1, 1.2, 9.0]), 0.3)
    assert 1.0 <= est3 <= 1.2 and inl3.tolist() == [True, True, True, False]
    # n_card == 1 (isolated measurements): D5 -> that value
    est1, _ = oracle.cote(np.array([0.0, 10.0, 20.0]), 0.3)
    assert est1 in (0.0, 10.0, 20.0)


# ---- KAT-13 end to end -----------------------------------------------------------------------------
def test_kat13_solver_end_to_end(oracle):
    a4, b4, T, inl = synth.matched_pairs(13, 400, inlier_ratio=0.25, noise=0.03)
    res, st, clique, fin = oracle.solve_correspondences(a4, b4, default_params(), want_sets=True)
    assert st == 0 and res.valid == 1
    rot, tr = synth.pose_error(res.matrix(), T)
    assert rot < 0.5 and tr < 0.1
    assert set(clique.tolist()) <= set(np.nonzero(inl)[0].tolist()) | set(clique.tolist())
    assert len(clique) >= 0.9 * inl.sum()
    assert set(fin.tolist()) <= set(clique.tolist())
    M = res.matrix()
    assert M[2, 2] == 1.0 and M[0, 2] == 0 and M[3].tolist() == [0, 0, 0, 1]     # yaw-only rotation block
    # degenerate: no consistent pair -> clique <= 1 -> invalid, identity
    a = P4([[0, 0, 0], [10, 0, 0], [0, 10, 0]]); b = P4([[0, 0, 0], [50, 0, 0], [0, 90, 0]])
    res, st = oracle.solve_correspondences(a, b, default_params())
    assert st == 1 and res.valid == 0 and np.array_equal(res.matrix(), np.eye(4))
    res, st = oracle.solve_correspondences(a[:1], b[:1], default_params())
    assert st == 2 and res.valid == 0


def test_full_pipeline_on_synthetic_scan_pair(oracle):
    src, tgt, T = synth.outdoor_pair(1)
    res, st = oracle.register_pair(src, tgt, default_params())
    assert st == 0 and res.valid == 1
    rot, tr = synth.pose_error(res.matrix(), T)
    assert rot < 2.0 and tr < 0.5, (rot, tr)
    assert 3000 < res.n_src_vox < 12000 and res.n_corr > 50


def test_weighted_mean_cote_mode(oracle):
    a4, b4, T, inl = synth.matched_pairs(14, 300, inlier_ratio=0.3, noise=0.03)
    p = default_params(); p.cote_mode = COTE_WEIGHTED_MEAN
    res, st = oracle.solve_correspondences(a4, b4, p)
    assert st == 0 and synth.pose_error(res.matrix(), T)[1] < 0.1
