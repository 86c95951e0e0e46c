"""GPU parity: every stage of the CUDA path, called through the C-ABI, against the CPU oracle on the
same seeded inputs.  Integer outputs (voxel membership, correspondences, adjacency bits, core numbers,
clique membership) must be bit-exact; fp64 poses within 1e-9; end-to-end within 2 deg / 0.3 m."""
import numpy as np
import pytest

from conftest import adj_to_dense, dense_to_adj
from quatro_b200 import synth
from quatro_b200.capi import Handle, default_params, PMC_HEU, KCORE_HEU, INLIER_NONE, COTE_WEIGHTED_MEAN, RESULT_DTYPE
from support import P4, assert_same_record, fpfh_like, same_bits

pytestmark = pytest.mark.gpu

# the production default of the neighbour lattice: (1 + 2^-9) * fpfh_radius (api.cu lattice_cell(), oracle default)
DEFAULT_CELL = float(np.float32(0.75) * np.float32(1.001953125))


@pytest.fixture(scope="module")
def scan_pair():
    return synth.outdoor_pair(1)


@pytest.fixture(scope="module")
def small_pair():
    return synth.outdoor_pair(3, rings=32, azimuths=900)


# ---- K1 voxel ----------------------------------------------------------------------------------
def test_voxel_capacity_is_reported(oracle, scan_pair):
    from quatro_b200.capi import Handle
    with Handle(max_batch_slots=2, max_voxel_points=1024) as h:
        got, st = h.voxelize(scan_pair[0], 0.3, 1)
        assert st == 3 and len(got) == 1024     # QB200_CAPACITY_EXCEEDED, never silent truncation
        out = h.register_batch([scan_pair[:2]], default_params())
        assert out["valid"][0] == 0 and out["status"][0] == 3 and np.array_equal(out["T"][0], np.eye(4).ravel())


def test_voxelize_bit_exact(handle, oracle, scan_pair, small_pair):
    for cloud in (scan_pair[0], scan_pair[1], small_pair[0]):
        for skip in (1, 0):
            ref, st_r = oracle.voxelize(cloud, 0.3, skip)
            got, st_g = handle.voxelize(cloud, 0.3, skip)
            if len(ref) > handle.cfg.max_voxel_points:
                assert st_g == 3  # QB200_CAPACITY_EXCEEDED is reported, not silently truncated
                continue
            assert st_g == st_r == 0
            assert same_bits(got, ref)  # centroids bit for bit, same order


def test_voxelize_edge_cases(handle, oracle):
    pts = P4([[0.1, 0.1, 0.1], [np.nan, 0, 0], [0.2, 0.1, 0.1], [5, 5, 5], [-0.1, 0, 0], [np.inf, 1, 1]])
    pts[3, 3] = -1.0
    for skip in (0, 1):
        ref, _ = oracle.voxelize(pts, 0.3, skip)
        got, st = handle.voxelize(pts, 0.3, skip)
        assert st == 0 and same_bits(got, ref)
    got, st = handle.voxelize(P4(np.zeros((0, 3))), 0.3, 1)
    assert len(got) == 0 and st == 0
    got, st = handle.voxelize(P4([[np.nan, 0, 0]]), 0.3, 1)
    assert len(got) == 0
    # leaf so small that dx*dy*dz overflows int32: PCL returns the input unfiltered
    big = P4([[0, 0, 0], [3000, 3000, 300]])
    ref, st_r = oracle.voxelize(big, 0.001, 0)
    got, st_g = handle.voxelize(big, 0.001, 0)
    assert st_r == st_g == -5 and np.array_equal(got, ref)


# ---- K2-K5 normals + FPFH ------------------------------------------------------------------------------
def test_fpfh_bit_exact(handle, oracle, scan_pair, small_pair):
    for raw, cell in ((scan_pair[0], 0.3), (small_pair[1], 0.3), (scan_pair[1], DEFAULT_CELL), (small_pair[0], DEFAULT_CELL)):
        vox, _ = oracle.voxelize(raw, 0.3, 1)
        n_ref, d_ref = oracle.compute_fpfh(vox, 0.5, 0.75, cell)
        n_got, d_got = handle.compute_fpfh(vox, 0.5, 0.75, cell)
        same_n = (n_got.view(np.uint32) == n_ref.view(np.uint32)) | (np.isnan(n_got) & np.isnan(n_ref))
        assert same_n.all(), f"{(~same_n).any(1).sum()} of {len(vox)} normals differ"
        same_d = d_got.view(np.uint32) == d_ref.view(np.uint32)
        assert same_d.all(), f"{(~same_d).any(1).sum()} of {len(vox)} descriptors differ, max abs {np.abs(d_got - d_ref).max()}"


def test_fpfh_other_lattice_and_unsorted_input(handle, oracle):
    rng = np.random.default_rng(5)
    g = np.arange(-4, 4.01, 0.25)
    xx, yy = np.meshgrid(g, g)
    pts = np.concatenate([np.stack([xx.ravel(), yy.ravel(), np.full(xx.size, -1.7)], 1),
                          np.stack([np.full(xx.size, 5.0), xx.ravel(), yy.ravel()], 1),
                          rng.uniform(-4, 4, (500, 3))])
    pts = pts[rng.permutation(len(pts))] + rng.normal(0, 0.01, (len(pts), 3))
    for cell in (0.3, 0.5, 0.2, DEFAULT_CELL):
        n_ref, d_ref = oracle.compute_fpfh(P4(pts), 0.5, 0.75, cell)
        n_got, d_got = handle.compute_fpfh(P4(pts), 0.5, 0.75, cell)
        assert same_bits(d_got, d_ref)
        assert same_bits(n_got, n_ref, nan_equal=True)
    # isolated / too-few-neighbour points: NaN normals, finite descriptors
    iso = P4([[0, 0, 0], [0.1, 0, 0], [10, 10, 10]])
    n_got, d_got = handle.compute_fpfh(iso, 0.5, 0.75, 0.3)
    n_ref, d_ref = oracle.compute_fpfh(iso, 0.5, 0.75, 0.3)
    assert np.isnan(n_got[:, :3]).all() and np.array_equal(d_got, d_ref)


# ---- K6/K7 matching ------------------------------------------------------------------------------------
def test_match_bit_exact(handle, oracle, scan_pair):
    src, tgt, _ = scan_pair
    sv, _ = oracle.voxelize(src, 0.3, 1)
    tv, _ = oracle.voxelize(tgt, 0.3, 1)
    _, sd = oracle.compute_fpfh(sv, 0.5, 0.75, 0.3)
    _, td = oracle.compute_fpfh(tv, 0.5, 0.75, 0.3)
    p = default_params()
    for a, ad, b, bd in ((sv, sd, tv, td), (tv, td, sv, sd)):   # second case: source larger than target (no swap)
        c_ref, nm_ref, _ = oracle.match(a, ad, b, bd, p)
        c_got, nm_got, st = handle.match(a, ad, b, bd, p)
        assert st == 0 and nm_got == nm_ref
        assert np.array_equal(c_got, c_ref)
    p2 = default_params(); p2.use_tuple_test = 0
    c_ref, nm_ref, _ = oracle.match(sv, sd, tv, td, p2)
    c_got, nm_got, _ = handle.match(sv, sd, tv, td, p2)
    assert np.array_equal(c_got, c_ref) and len(c_got) == nm_got
    p3 = default_params(); p3.seed = 12345
    assert np.array_equal(handle.match(sv, sd, tv, td, p3)[0], oracle.match(sv, sd, tv, td, p3)[0])


def test_match_ties_and_small_inputs(handle, oracle):
    pts = P4([[0, 0, 0], [1, 0, 0], [0, 1, 0]])
    d = np.zeros((3, 33), np.float32)
    p = default_params(); p.use_tuple_test = 0
    assert handle.match(pts, d, pts, d, p)[0].tolist() == [[0, 0]]       # lowest-index tie-break both ways
    rng = np.random.default_rng(2)
    for na, nb in ((1, 1), (5, 130), (129, 127), (300, 257)):
        a, b = P4(rng.uniform(-5, 5, (na, 3))), P4(rng.uniform(-5, 5, (nb, 3)))
        ad, bd = rng.uniform(0, 100, (na, 33)).astype(np.float32), rng.uniform(0, 100, (nb, 33)).astype(np.float32)
        bd[: min(na, nb) // 2] = ad[: min(na, nb) // 2]                # exact duplicates -> zero distances
        for prm in (p, default_params()):
            ref = oracle.match(a, ad, b, bd, prm)
            got = handle.match(a, ad, b, bd, prm)
            assert np.array_equal(got[0], ref[0]) and got[1] == ref[1]


def test_match_isolated_points_and_padding(handle, oracle):
    """All-zero descriptors (FPFH of a point without neighbours) are bit-identical to the zero padding of the last
    128-point block: padded rows / columns must never enter the exact evaluation (regression: they once won ties)."""
    rng = np.random.default_rng(21)
    for na, nb in ((300, 290), (129, 257), (640, 513)):
        a, b = P4(rng.uniform(-30, 30, (na, 3))), P4(rng.uniform(-30, 30, (nb, 3)))
        ad, bd = fpfh_like(rng, na), fpfh_like(rng, nb)
        ad[[7, na // 2, na - 1]] = 0.0
        bd[[3, nb - 2]] = 0.0
        ad[na // 3] = ad[5]; bd[nb // 3] = ad[5]                 # a duplicate class that is not the zero vector
        p = default_params(); p.use_tuple_test = 0
        ref = oracle.match(a, ad, b, bd, p)
        got = handle.match(a, ad, b, bd, p)
        assert np.array_equal(got[0], ref[0]) and got[1] == ref[1], (na, nb)


def _tc_rel_error(handle, a, b):
    """worst |d~ - d| / (|a - mu|^2 + |b - mu|^2): the normalisation the kernel's bound uses (mu = FPFH of a plane: 100 in bins 5, 16, 27)"""
    mu = np.zeros(33); mu[[5, 16, 27]] = 100.0
    got = handle.debug_tc_distances(a, b).astype(np.float64)
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    ref = ((a64[:, None, :] - b64[None, :, :]) ** 2).sum(2)
    scale = ((a64 - mu) ** 2).sum(1)[:, None] + ((b64 - mu) ** 2).sum(1)[None, :]
    assert np.isfinite(got).all()
    with np.errstate(divide="ignore", invalid="ignore"):
        rel = np.where(scale > 0, np.abs(got - ref) / scale, 0.0)
    return rel.max(), np.abs(got - ref).max(), ref.max()


def test_tc_filter_error_bound(handle):
    """The tensor-core (wgmma, 3xTF32) approximate distances must stay inside the margin the candidate filter assumes:
    |d~ - d| <= kTcC/2 * (|a'|^2 + |b'|^2) with kTcC = 1.2e-4, a' = a - mu (csrc/tc_match.cu).  Analytic budget: the dropped lo.lo
    term and the TF32 rounding of lo contribute <= 2^-21 (|a'|^2 + |b'|^2); the undocumented part is the fp32 accumulation inside
    the MMA (120 products per entry), measured here on random and adversarial descriptors.  The margin asserted is 3x."""
    rng = np.random.default_rng(11)
    worst = 0.0
    cases = []
    for trial in range(4):
        a, b = fpfh_like(rng, 128), fpfh_like(rng, 100 + trial)
        if trial == 3:
            b[:50] = a[:50]                                    # exact duplicates: d = 0 rows
        cases.append((a, b))
    # adversarial: large dynamic range inside one descriptor, near-cancelling cross terms, tiny and huge norms side by side
    spike = np.zeros((128, 33), np.float32); spike[np.arange(128), rng.integers(0, 33, 128)] = 100.0; spike += rng.uniform(0, 1e-3, spike.shape).astype(np.float32)
    cases.append((spike, spike[::-1].copy()))
    near = fpfh_like(rng, 128); cases.append((near, (near * np.float32(1 + 2e-4)).astype(np.float32)))       # d ~ 1e-8 |a|^2: full cancellation
    mu = np.zeros(33, np.float32); mu[[5, 16, 27]] = 100.0
    tiny = (mu + rng.normal(0, 1e-3, (128, 33))).astype(np.float32); cases.append((tiny, fpfh_like(rng, 128)))  # |a'| ~ 1e-3 next to |b'| ~ 100
    cases.append((np.tile(mu, (128, 1)), np.zeros((128, 33), np.float32)))                                     # planes vs isolated points
    alt = np.zeros((128, 33), np.float32); alt[:, ::2] = 18.75; alt[:, 1::2] = 0.0; cases.append((alt, (alt.max() - alt).astype(np.float32)))
    for a, b in cases:
        rel, abs_err, ref_max = _tc_rel_error(handle, a, b)
        worst = max(worst, rel)
        assert abs_err < 0.05 * np.sqrt(ref_max + 1) + 1e-3, "tensor-core tile is not even approximately the distance matrix"
    assert worst < 2.0e-5, worst     # kTcC / 2 = 6e-5: three times the worst case seen


def test_match_exact_kernel_and_tie_fallback(oracle, scan_pair, monkeypatch):
    """Default K6 = tensor-core filter + in-kernel exact evaluation; thousands of identical descriptors make its stripes abort
    to the exact CUDA-core kernel.  QB200_MATCH_EXACT=1 forces the exact kernel everywhere.  All must equal the oracle."""
    rng = np.random.default_rng(4)
    n = 2600
    a, b = P4(rng.uniform(-30, 30, (n, 3))), P4(rng.uniform(-30, 30, (n - 7, 3)))
    ad, bd = fpfh_like(rng, n), fpfh_like(rng, n - 7)
    ad[:2200] = ad[0]; bd[:2100] = ad[0]                        # massive exact ties -> lowest-index tie-breaks everywhere
    p = default_params(); p.use_tuple_test = 0
    ref = oracle.match(a, ad, b, bd, p)
    with Handle(max_batch_slots=2) as h:
        got = h.match(a, ad, b, bd, p)
        assert np.array_equal(got[0], ref[0]) and got[1] == ref[1]
    monkeypatch.setenv("QB200_MATCH_EXACT", "1")
    with Handle(max_batch_slots=2) as h:
        got = h.match(a, ad, b, bd, p)
        assert np.array_equal(got[0], ref[0])
        src, tgt, _ = scan_pair
        r_ref, _ = oracle.register_pair(src, tgt, default_params())
        r_got, _ = h.register_pair(src, tgt, default_params())
        assert (r_got.n_mutual, r_got.n_corr, r_got.clique_size) == (r_ref.n_mutual, r_ref.n_corr, r_ref.clique_size)


def test_match_and_pack(handle, oracle, small_pair):
    sv, _ = oracle.voxelize(small_pair[0], 0.3, 1)
    tv, _ = oracle.voxelize(small_pair[1], 0.3, 1)
    p = default_params()
    c_ref, sm_ref, tm_ref, _ = oracle.match_and_pack(sv, tv, p)
    c_got, sm_got, tm_got, st = handle.match_and_pack(sv, tv, p)
    assert st == 0 and np.array_equal(c_got, c_ref) and np.array_equal(sm_got, sm_ref) and np.array_equal(tm_got, tm_ref)
    cc, sm2, tm2 = handle.last_correspondences()
    assert np.array_equal(cc, c_ref) and np.array_equal(sm2, sm_ref)
    bad = default_params(); bad.normal_radius = 1.0   # normal_radius > fpfh_radius: the reference throws invalid_argument
    from quatro_b200.capi import QuatroB200Error
    with pytest.raises(QuatroB200Error):
        handle.match_and_pack(sv, tv, bad)


# ---- K8 graph ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L,ratio", [(2, 1.0), (33, 0.5), (200, 0.4), (1000, 0.3), (3000, 0.3), (4096, 0.1)])
def test_graph_bit_exact(handle, oracle, L, ratio):
    a4, b4, T, inl = synth.matched_pairs(100 + L, L, inlier_ratio=ratio, noise=0.05)
    adj_r, deg_r, ne_r = oracle.build_graph(a4, b4, 0.3, 1.0)
    adj_g, deg_g, ne_g = handle.build_graph(a4, b4, 0.3, 1.0)
    assert np.array_equal(adj_g, adj_r)
    assert np.array_equal(deg_g, deg_r) and ne_g == ne_r


def test_graph_boundary_and_duplicates(handle, oracle):
    # pairs sitting exactly on / next to the |db - da| = 0.6 boundary, duplicate points, large coordinates
    rng = np.random.default_rng(0)
    a = rng.uniform(-80, 80, (600, 3))
    b = a.copy()
    d = rng.normal(size=(600, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    b[::2] += d[::2] * 0.6
    b[1::4] += d[1::4] * np.float32(0.6000001)
    a[10] = a[11]; b[20] = b[21]; a[30] = a[31]; b[30] = b[31]
    a4, b4 = P4(a), P4(b)
    for nb in (0.3, 0.25):
        assert np.array_equal(handle.build_graph(a4, b4, nb, 1.0)[0], oracle.build_graph(a4, b4, nb, 1.0)[0])


# ---- K9 k-core + clique ------------------------------------------------------------------------------
def _random_graph(rng, n, p, planted=0):
    R = rng.uniform(size=(n, n)) < p
    R = np.triu(R, 1); R = R | R.T
    if planted:
        m = np.sort(rng.choice(n, planted, replace=False))
        R[np.ix_(m, m)] = True
    np.fill_diagonal(R, False)
    return R


@pytest.mark.parametrize("n,p,planted", [(1, 0, 0), (2, 1.0, 0), (40, 0.3, 0), (150, 0.03, 25), (500, 0.1, 60), (1000, 0.02, 0),
                                         (3000, 0.02, 300), (4096, 0.01, 100), (700, 0.5, 0)])
def test_kcore_and_clique_bit_exact(handle, oracle, n, p, planted):
    R = _random_graph(np.random.default_rng(n + planted), n, p, planted)
    adj = dense_to_adj(R)
    c_ref, k_ref, o_ref, mc_ref = oracle.max_clique(adj, PMC_HEU)
    c_got, k_got, o_got, mc_got = handle.max_clique(adj, PMC_HEU)
    assert mc_got == mc_ref
    assert np.array_equal(k_got, k_ref), "core numbers differ"
    assert np.array_equal(o_got, o_ref), "peel (degeneracy) order differs"
    assert np.array_equal(c_got, c_ref), "clique membership differs"


def test_clique_on_registration_graphs(handle, oracle):
    for L, ratio in ((300, 0.3), (1500, 0.2), (3000, 0.35)):
        a4, b4, _, inl = synth.matched_pairs(7 * L, L, inlier_ratio=ratio, noise=0.05)
        adj, _, _ = oracle.build_graph(a4, b4, 0.3, 1.0)
        ref = oracle.max_clique(adj, PMC_HEU)
        got = handle.max_clique(adj, PMC_HEU)
        assert np.array_equal(got[0], ref[0]) and np.array_equal(got[2], ref[2]) and got[3] == ref[3]
        ref = oracle.max_clique(adj, KCORE_HEU, 0.1)
        got = handle.max_clique(adj, KCORE_HEU, 0.1)
        assert np.array_equal(got[0], ref[0])


def _structured_graphs():
    """graph families that stress the bucket mechanics of the peel: many vertices of equal degree (groups whose members
    already sit inside the target slots -> serial replay), many levels, many improving start vertices in the clique search"""
    out = []
    n = 60; R = np.ones((n, n), bool); np.fill_diagonal(R, False); out.append(("K60", R))
    n = 200; R = np.zeros((n, n), bool)
    for i in range(n):
        for k in (1, 2, 3):
            R[i, (i + k) % n] = R[(i + k) % n, i] = True
    out.append(("ring3", R))
    n = 150; R = np.zeros((n, n), bool); R[0, 1:] = True; R[1:, 0] = True; out.append(("star", R))
    R = np.ones((150, 150), bool)
    for P in (range(0, 40), range(40, 90), range(90, 150)):
        R[np.ix_(list(P), list(P))] = False
    out.append(("multipartite", R))
    R = np.zeros((300, 300), bool)
    for s0 in range(0, 300, 30):
        R[s0:s0 + 30, s0:s0 + 30] = True
    np.fill_diagonal(R, False); out.append(("disjoint cliques", R))
    R = np.zeros((256, 256), bool)
    for i in range(256):
        for b in range(8):
            R[i, i ^ (1 << b)] = True
    out.append(("hypercube8", R))
    # nested cliques of growing size joined by sparse noise: the incumbent improves many times
    rng = np.random.default_rng(5)
    R = rng.uniform(size=(900, 900)) < 0.01; R = np.triu(R, 1); R = R | R.T
    o = 0
    for k in range(3, 40, 3):
        R[o:o + k, o:o + k] = True; o += k
    np.fill_diagonal(R, False); out.append(("growing cliques", R))
    rng = np.random.default_rng(6)
    for n, p_ in ((600, 0.2), (1200, 0.08), (2500, 0.05)):
        R = rng.uniform(size=(n, n)) < p_; R = np.triu(R, 1); R = R | R.T
        out.append((f"G({n},{p_})", R))
    return out


def test_kcore_and_clique_structured_graphs(handle, oracle):
    for name, R in _structured_graphs():
        adj = dense_to_adj(R)
        c_ref, k_ref, o_ref, mc_ref = oracle.max_clique(adj, PMC_HEU)
        c_got, k_got, o_got, mc_got = handle.max_clique(adj, PMC_HEU)
        assert mc_got == mc_ref, name
        assert np.array_equal(k_got, k_ref), f"{name}: core numbers differ"
        assert np.array_equal(o_got, o_ref), f"{name}: peel order differs"
        assert np.array_equal(c_got, c_ref), f"{name}: clique membership differs"


def test_exact_clique_matches_oracle(handle, oracle):
    """PMC_EXACT (src/graph.cc:106-127): same clique as the oracle's canonical branch and bound -- size AND membership -- on graphs
    where the heuristic is already maximum, where the search improves it, and where the node limit cuts it short."""
    from quatro_b200.capi import PMC_EXACT, FLAG_CLIQUE_TRUNCATED
    cases = [(n, p, pl, 0) for n, p, pl in ((2, 1.0, 0), (40, 0.3, 0), (150, 0.03, 25), (500, 0.1, 60), (1000, 0.02, 0), (600, 0.2, 0),
                                             (1200, 0.08, 0), (3000, 0.02, 300), (4096, 0.01, 100))]
    cases += [(300, 0.7, 0, 3000), (700, 0.5, 0, 5000), (90, 0.6, 0, 0)]
    improved = truncated = 0
    for n, p, planted, limit in cases:
        adj = dense_to_adj(_random_graph(np.random.default_rng(n + planted), n, p, planted))
        ref = oracle.max_clique_ex(adj, PMC_EXACT, 0.5, limit)
        got = handle.max_clique_ex(adj, PMC_EXACT, 0.5, limit)
        assert got[3] == ref[3] and got[4] == ref[4], (n, p, got[3:], ref[3:])
        assert np.array_equal(got[1], ref[1]) and np.array_equal(got[2], ref[2])
        assert np.array_equal(got[0], ref[0]), (n, p, planted, limit, got[0], ref[0])
        improved += len(ref[0]) > len(oracle.max_clique(adj, PMC_HEU)[0])
        truncated += bool(ref[4] & FLAG_CLIQUE_TRUNCATED)
    assert improved >= 3 and truncated >= 2
    for name, R in _structured_graphs():
        adj = dense_to_adj(R)
        ref = oracle.max_clique_ex(adj, PMC_EXACT, 0.5, 20000)
        got = handle.max_clique_ex(adj, PMC_EXACT, 0.5, 20000)
        assert np.array_equal(got[0], ref[0]) and got[4] == ref[4], name


def test_exact_mode_pipeline(handle, oracle):
    from quatro_b200.capi import PMC_EXACT
    p = default_params()
    p.inlier_selection_mode = PMC_EXACT
    for seed, L, ratio in ((5, 300, 0.3), (6, 1500, 0.1), (7, 3000, 0.05)):
        a4, b4, T, inl = synth.matched_pairs(seed, L, inlier_ratio=ratio, noise=0.05)
        r_g, st_g = handle.solve_correspondences(a4, b4, p)
        r_o, st_o = oracle.solve_correspondences(a4, b4, p)
        assert st_g == st_o and r_g.clique_size == r_o.clique_size and r_g.flags == r_o.flags
        assert np.array_equal(handle.last_clique(), np.sort(handle.last_clique()))
        assert np.allclose(r_g.matrix(), r_o.matrix(), atol=1e-9)
    # a wave of more than 64 sets: the exact search runs 64 pairs per launch on shared scratch
    with Handle(max_batch_slots=72, max_raw_points=16384, max_voxel_points=2048, max_corr=512) as hb:
        sets = [synth.matched_pairs(100 + i, 150 + 3 * i, inlier_ratio=0.15, noise=0.05)[:2] for i in range(72)]
        out = hb.solve_batch(sets, p)
        for i in (0, 1, 31, 63, 64, 65, 71):
            r_o, st_o = oracle.solve_correspondences(sets[i][0], sets[i][1], p)
            assert out[i]["clique_size"] == r_o.clique_size and out[i]["flags"] == r_o.flags and out[i]["status"] == st_o
            assert np.allclose(np.asarray(out[i]["T"]).reshape(4, 4).T, r_o.matrix(), atol=1e-9)
    # whole pairs through the batch path (several pairs per wave, exact search per pair)
    pairs = [synth.outdoor_pair(40 + i, rings=32, azimuths=900)[:2] for i in range(3)]
    res = handle.register_batch(pairs, p)
    for (src, tgt), r in zip(pairs, res):
        ref, st_ref = oracle.register_pair(src, tgt, p)
        assert r["clique_size"] == ref.clique_size and r["n_corr"] == ref.n_corr and r["flags"] == ref.flags
        assert np.allclose(np.asarray(r["T"]).reshape(4, 4).T, ref.matrix(), atol=1e-9)


def test_graph_and_clique_wide_handle(oracle):
    """max_corr = 8192: 256-word rows (8-warp peel, 64-bit packed group sizes, 8 adjacency words per lane in the descent)."""
    with Handle(max_batch_slots=2, max_corr=8192) as h:
        a4, b4, T, inl = synth.matched_pairs(4321, 6000, inlier_ratio=0.1, noise=0.05)
        adj_r, deg_r, ne_r = oracle.build_graph(a4, b4, 0.3, 1.0)
        adj_g, deg_g, ne_g = h.build_graph(a4, b4, 0.3, 1.0)
        assert np.array_equal(adj_g, adj_r) and np.array_equal(deg_g, deg_r) and ne_g == ne_r
        ref = oracle.max_clique(adj_r, PMC_HEU)
        got = h.max_clique(adj_r, PMC_HEU)
        assert got[3] == ref[3] and np.array_equal(got[1], ref[1]) and np.array_equal(got[2], ref[2]) and np.array_equal(got[0], ref[0])
        p = default_params()
        r_g, st_g = h.solve_correspondences(a4, b4, p)
        r_o, st_o = oracle.solve_correspondences(a4, b4, p)
        assert st_g == st_o and r_g.clique_size == r_o.clique_size and np.allclose(r_g.matrix(), r_o.matrix(), atol=1e-9)
        R = _random_graph(np.random.default_rng(77), 8192, 0.004, 120)
        adj = dense_to_adj(R)
        ref = oracle.max_clique(adj, PMC_HEU)
        got = h.max_clique(adj, PMC_HEU)
        assert got[3] == ref[3] and np.array_equal(got[1], ref[1]) and np.array_equal(got[2], ref[2]) and np.array_equal(got[0], ref[0])


def test_graph_error_band_adversarial(handle, oracle):
    """The fp32 Gram-form filter of K8 must hand every pair it cannot decide to the literal fp64 expression: coincident
    duplicates in both clouds (0/0 in the literal form), tiny triangles (da + db < beta), points far from the origin
    (large |a|^2: wide error band), points on the threshold to 1 ulp, and everything shifted by a large offset."""
    rng = np.random.default_rng(11)
    n = 700
    a = rng.uniform(-2, 2, (n, 3)); b = a + rng.normal(0, 0.05, (n, 3))
    a[5] = a[6]; b[5] = b[6]            # coincident in both clouds
    a[7] = a[8]                         # coincident in one cloud only
    a[100:140] = a[100] + rng.normal(0, 0.05, (40, 3)); b[100:140] = b[100] + rng.normal(0, 0.05, (40, 3))   # tiny triangles
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    b[200:300] = a[200:300] + d[200:300] * 0.6
    for shift, scale in ((0.0, 1.0), (75.0, 1.0), (0.0, 40.0), (400.0, 1.0)):
        a4, b4 = P4(a * scale + shift), P4(b * scale + shift)
        for nb in (0.3, 0.05):
            g, dg, ng = handle.build_graph(a4, b4, nb, 1.0)
            r, dr, nr = oracle.build_graph(a4, b4, nb, 1.0)
            assert np.array_equal(g, r), (shift, scale, nb, int((g != r).sum()))
            assert np.array_equal(dg, dr) and ng == nr
    z = np.zeros((70, 3)); z4 = P4(z)   # every point identical
    assert np.array_equal(handle.build_graph(z4, z4, 0.3, 1.0)[0], oracle.build_graph(z4, z4, 0.3, 1.0)[0])


def test_small_capacity_handles(oracle, small_pair):
    """Configurations the default tests never touch (ADVICE r1): one slot, V = 128 / 256, max_raw_points < max_voxel_points,
    max_raw_points = 200 (the voxel sort's 256 histogram words per tile exceed R)."""
    src, tgt, _ = small_pair
    p = default_params()
    sv, _ = oracle.voxelize(src, 0.3, 1); tv, _ = oracle.voxelize(tgt, 0.3, 1)
    for kw in (dict(max_batch_slots=1, max_voxel_points=16384, max_raw_points=4096),
               dict(max_batch_slots=1, max_voxel_points=128, max_raw_points=200), dict(max_batch_slots=1, max_voxel_points=128),
               dict(max_batch_slots=1, max_voxel_points=256), dict(max_batch_slots=1)):
        with Handle(**kw) as h:
            V = h.cfg.max_voxel_points
            raw = src[:min(len(src), h.cfg.max_raw_points)]
            for skip in (0, 1):
                ref, st_r = oracle.voxelize(raw, 0.3, skip)
                got, st_g = h.voxelize(raw, 0.3, skip)
                if len(ref) > V:   # QB200_CAPACITY_EXCEEDED, the first V voxels still computed
                    assert st_g == 3 and len(got) == V, (kw, skip)
                    ref = ref[:V]
                else:
                    assert st_g == st_r == 0, (kw, skip)
                assert same_bits(got, ref), (kw, skip)
            a, b = sv[:min(len(sv), V, h.cfg.max_raw_points)], tv[:min(len(tv), V, h.cfg.max_raw_points)]
            n_g, d_g = h.compute_fpfh(a, 0.5, 0.75, DEFAULT_CELL)
            n_r, d_r = oracle.compute_fpfh(a, 0.5, 0.75, DEFAULT_CELL)
            assert same_bits(d_g, d_r), kw
            _, d_b = oracle.compute_fpfh(b, 0.5, 0.75, DEFAULT_CELL)
            c_g = h.match(a, d_r, b, d_b, p)[0]
            c_r = oracle.match(a, d_r, b, d_b, p)[0]
            assert np.array_equal(c_g, c_r), kw


# ---- K10/K11 pose --------------------------------------------------------------------------------------
def test_solve_pose_matches_oracle(handle, oracle):
    for seed, L, ratio in ((1, 300, 0.3), (2, 2000, 0.25), (3, 64, 0.9)):
        a4, b4, T, inl = synth.matched_pairs(seed, L, inlier_ratio=ratio, noise=0.04)
        adj, _, _ = oracle.build_graph(a4, b4, 0.3, 1.0)
        clique = oracle.max_clique(adj, PMC_HEU)[0]
        for mode in (0, COTE_WEIGHTED_MEAN):
            p = default_params(); p.cote_mode = mode
            r_ref, rm_ref, tm_ref, st_r = oracle.solve_pose(a4, b4, clique, p)
            r_got, rm_got, tm_got, st_g = handle.solve_pose(a4, b4, clique, p)
            assert st_g == st_r == 0 and r_got.valid == 1
            assert np.allclose(r_got.matrix(), r_ref.matrix(), atol=1e-9, rtol=0)
            assert r_got.gnc_iters == r_ref.gnc_iters
            assert np.array_equal(rm_got, rm_ref) and np.array_equal(tm_got, tm_ref)
            assert (r_got.n_rot_inliers, r_got.n_final_inliers) == (r_ref.n_rot_inliers, r_ref.n_final_inliers)
            assert r_got.cost == r_ref.cost or abs(r_got.cost - r_ref.cost) < 1e-9 * max(1.0, abs(r_ref.cost))
    p = default_params(); p.using_rot_inliers_when_estimating_cote = 1
    r_ref, _, tm_ref, _ = oracle.solve_pose(a4, b4, clique, p)
    r_got, _, tm_got, _ = handle.solve_pose(a4, b4, clique, p)
    assert np.allclose(r_got.matrix(), r_ref.matrix(), atol=1e-9) and r_got.n_final_inliers == r_ref.n_final_inliers


def test_solve_pose_with_ryrx_prior(handle, oracle):
    a4, b4, T, inl = synth.matched_pairs(5, 400, inlier_ratio=0.4, noise=0.03)
    adj, _, _ = oracle.build_graph(a4, b4, 0.3, 1.0)
    clique = oracle.max_clique(adj, PMC_HEU)[0]
    p = default_params(); p.use_pre_estimated_RyRx = 1
    ang = np.deg2rad(0.5)
    Ry = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]])
    for i, v in enumerate(Ry.ravel()):
        p.RyRx[i] = v
    r_ref, *_ = oracle.solve_pose(a4, b4, clique, p)
    r_got, *_ = handle.solve_pose(a4, b4, clique, p)
    assert np.allclose(r_got.matrix(), r_ref.matrix(), atol=1e-9)


def test_solve_correspondences_and_degenerate(handle, oracle):
    for seed, L in ((21, 500), (22, 3000)):
        a4, b4, T, inl = synth.matched_pairs(seed, L, inlier_ratio=0.3, noise=0.04)
        p = default_params()
        r_ref, st_r, c_ref, f_ref = oracle.solve_correspondences(a4, b4, p, want_sets=True)
        r_got, st_g = handle.solve_correspondences(a4, b4, p)
        assert st_g == st_r == 0
        assert np.array_equal(handle.last_clique(), c_ref)                       # max-clique membership bit-exact
        assert np.array_equal(handle.last_final_inliers(), f_ref)
        assert (r_got.n_edges, r_got.max_core, r_got.clique_size) == (r_ref.n_edges, r_ref.max_core, r_ref.clique_size)
        assert np.allclose(r_got.matrix(), r_ref.matrix(), atol=1e-9)
        rot, tr = synth.pose_error(r_got.matrix(), T)
        assert rot < 0.5 and tr < 0.1
    a = P4([[0, 0, 0], [10, 0, 0], [0, 10, 0]]); b = P4([[0, 0, 0], [50, 0, 0], [0, 90, 0]])
    r, st = handle.solve_correspondences(a, b, default_params())
    assert st == 1 and r.valid == 0 and np.array_equal(r.matrix(), np.eye(4))
    r, st = handle.solve_correspondences(a[:1], b[:1], default_params())
    assert st == 2 and r.valid == 0
    pn = default_params(); pn.inlier_selection_mode = INLIER_NONE
    a4, b4, T, _ = synth.matched_pairs(30, 200, inlier_ratio=0.9, noise=0.02)
    r_got, _ = handle.solve_correspondences(a4, b4, pn)
    r_ref, _ = oracle.solve_correspondences(a4, b4, pn)
    assert np.allclose(r_got.matrix(), r_ref.matrix(), atol=1e-9)


def test_solve_batch_matches_single_and_oracle(handle, oracle):
    """qb200_solve_batch = computeTransformation per correspondence set; 11 sets > 8 slots (two waves), ragged sizes."""
    p = default_params()
    sets = []
    for i, L in enumerate((40, 3, 160, 700, 0, 1, 33, 320, 1500, 64, 2)):
        a4, b4, _, _ = synth.matched_pairs(300 + i, max(L, 1), inlier_ratio=0.3, noise=0.03)
        sets.append((a4[:L], b4[:L]))
    out = handle.solve_batch(sets, p)
    assert len(out) == len(sets)
    for (a4, b4), g in zip(sets, out):
        if len(a4) == 0:
            assert g["valid"] == 0
            continue
        r_ref, st_ref = oracle.solve_correspondences(a4, b4, p)
        r_one, st_one = handle.solve_correspondences(a4, b4, p)
        for k in ("valid", "status", "n_corr", "n_edges", "max_core", "clique_size", "gnc_iters", "n_rot_inliers", "n_final_inliers"):
            assert g[k] == getattr(r_ref, k) == getattr(r_one, k), (k, len(a4))
        assert np.allclose(np.asarray(g["T"]).reshape(4, 4).T, r_ref.matrix(), atol=1e-9)
    import torch
    dev = [(torch.from_numpy(np.ascontiguousarray(a)).cuda(), torch.from_numpy(np.ascontiguousarray(b)).cuda()) for a, b in sets]
    torch.cuda.synchronize()
    out_d = handle.solve_batch([(a.data_ptr() if len(a) else 0, b.data_ptr() if len(b) else 0, len(a)) for a, b in dev], p, kind=1)
    assert out_d.tobytes() == out.tobytes()


# ---- end to end ----------------------------------------------------------------------------------------
def test_register_pair_end_to_end(handle, oracle, scan_pair):
    src, tgt, T = scan_pair
    p = default_params()
    r_ref, st_r = oracle.register_pair(src, tgt, p)
    r_got, st_g = handle.register_pair(src, tgt, p)
    assert st_g == st_r == 0
    assert_same_record(r_got, r_ref)
    rot, tr = synth.pose_error(r_got.matrix(), T)
    assert rot < 2.0 and tr < 0.5        # vs ground truth (the z offset of a yaw-only model stays in the budget)
    rot, tr = synth.pose_error(r_got.matrix(), r_ref.matrix())
    assert rot < 1e-6 and tr < 1e-6      # vs the CPU reference path: north_star asks for 2 deg / 0.3 m


def test_register_batch_matches_single_and_oracle(handle, oracle, monkeypatch):
    p = default_params()
    pairs = [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(10, 21)]   # 11 pairs > 8 slots: two waves
    out = handle.register_batch(pairs, p)
    assert out.dtype == RESULT_DTYPE and len(out) == len(pairs)
    for (src, tgt), g in zip(pairs, out):
        r_ref, _ = oracle.register_pair(src, tgt, p)
        assert_same_record(g, r_ref)
    # order / batch composition must not change any pair's result
    out2 = handle.register_batch(pairs[::-1], p)
    assert out2[::-1].tobytes() == out.tobytes()
    # three waves alternating between the two lanes, and the single-lane path (QB200_LANES=1): same records
    with Handle(max_batch_slots=4) as h4:
        assert h4.register_batch(pairs, p).tobytes() == out.tobytes()
        assert h4.register_batch(pairs, p).tobytes() == out.tobytes()      # lanes are reusable
    monkeypatch.setenv("QB200_LANES", "1")
    with Handle(max_batch_slots=4) as h1:
        assert h1.register_batch(pairs, p).tobytes() == out.tobytes()


def test_register_batch_enqueue_flush_pipelined(oracle):
    """qb200_register_batch_enqueue / _flush: three batches in flight over reused lanes give the records of the blocking call,
    and an entry point called in between flushes implicitly."""
    import ctypes as C
    from quatro_b200.capi import Handle, Pair, MEM_HOST
    p = default_params()
    batches = [[synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(b, b + n)] for b, n in ((200, 11), (220, 5), (240, 9))]
    with Handle(max_batch_slots=4) as h:
        ref = [h.register_batch(b, p) for b in batches]
        arrs, outs, keep = [], [], []
        for b in batches:
            arr = (Pair * len(b))()
            for i, (s, t) in enumerate(b):
                s, t = np.ascontiguousarray(s, np.float32), np.ascontiguousarray(t, np.float32)
                keep.append((s, t))
                arr[i].src, arr[i].n_src, arr[i].tgt, arr[i].n_tgt = s.ctypes.data, len(s), t.ctypes.data, len(t)
            arrs.append(arr)
            outs.append(np.zeros(len(b), RESULT_DTYPE))
        for arr, out in zip(arrs, outs):
            h.register_batch_enqueue_raw(arr, len(out), p, MEM_HOST, out)
        h.register_batch_flush()
        for out, r in zip(outs, ref):
            assert out.tobytes() == r.tobytes()
        # implicit flush: a blocking call right after an enqueue completes the queued batch first
        outs[0][:] = 0
        h.register_batch_enqueue_raw(arrs[0], len(outs[0]), p, MEM_HOST, outs[0])
        again = h.register_batch(batches[1], p)
        assert outs[0].tobytes() == ref[0].tobytes() and again.tobytes() == ref[1].tobytes()
        h.register_batch_flush()   # nothing in flight: a no-op
        # solve_correspondences and set_stream flush as well: the queued record is the blocking call's, the solve's its own
        import torch
        one = h.register_batch(batches[0][:1], p)
        a4, b4 = synth.matched_pairs(250, 500, inlier_ratio=0.3, noise=0.04)[:2]
        solo, _ = h.solve_correspondences(a4, b4, p)
        out1 = np.zeros(1, RESULT_DTYPE)
        h.register_batch_enqueue_raw(arrs[0], 1, p, MEM_HOST, out1)
        got, _ = h.solve_correspondences(a4, b4, p)
        h.register_batch_flush()
        assert out1.tobytes() == one.tobytes() and bytes(got) == bytes(solo)
        side = torch.cuda.Stream()
        out1[:] = 0
        h.solve_correspondences(a4, b4, p)   # leaves the solve's record where the batch's will be copied from
        h.register_batch_enqueue_raw(arrs[0], 1, p, MEM_HOST, out1)
        h.set_stream(side.cuda_stream)
        h.register_batch_flush()
        h.set_stream(0)
        assert out1.tobytes() == one.tobytes()
    r_ref, _ = oracle.register_pair(batches[0][0][0], batches[0][0][1], p)
    assert_same_record(ref[0][0], r_ref)


def test_register_batch_device_resident_inputs(handle, oracle):
    import torch
    p = default_params()
    host = [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in (31, 32, 33)]
    dev = [(torch.from_numpy(s).cuda(), torch.from_numpy(t).cuda()) for s, t in host]
    ptrs = [(a.data_ptr(), a.shape[0], b.data_ptr(), b.shape[0]) for a, b in dev]
    torch.cuda.synchronize()
    out_d = handle.register_batch(ptrs, p, kind=1)
    out_h = handle.register_batch(host, p)
    assert out_d.tobytes() == out_h.tobytes()


def test_empty_and_degenerate_clouds_in_batch(handle):
    p = default_params()
    good = synth.outdoor_pair(40, rings=32, azimuths=900)[:2]
    empty = np.zeros((0, 4), np.float32)
    ground_only = good[0][good[0][:, 3] < 0]
    out = handle.register_batch([good, (empty, good[1]), (ground_only, good[1]), good], p)
    assert out["valid"].tolist() == [1, 0, 0, 1]
    assert out["status"][1] == 2 and out["status"][2] == 2
    assert np.array_equal(out["T"][1], np.eye(4).ravel())
    assert out[0].tobytes() == out[3].tobytes()


def test_launch_counter_and_stage_times(handle):
    p = default_params()
    before = handle.launch_count()
    handle.register_batch([synth.outdoor_pair(50, rings=16, azimuths=450)[:2]], p)
    assert handle.launch_count() - before >= 25
    ms = handle.stage_ms()
    assert (ms >= 0).all() and ms[1:7].sum() > 0


# ---- scan cache (descriptor reuse: odometry chains, loop-closure sweeps) ----------------------------------------------------
def test_scan_cache_matches_uncached_pipeline(oracle):
    """qb200_cache_scans + qb200_register_cached must give the records of qb200_register_batch byte for byte, whichever slots the
    scans sit in and however often a scan is reused; the cached descriptors are the ones of the stage entry points."""
    p = default_params()
    scans = []
    for seed in (21, 22, 23):
        s, t, _ = synth.outdoor_pair(seed, rings=32, azimuths=900)
        scans += [s, t]
    pairs_idx = [(0, 1), (2, 3), (4, 5), (0, 3), (1, 0), (5, 5)]     # three ordinary pairs, a cross pair, a reversed pair, a scan with itself
    with Handle(max_batch_slots=4) as h:
        ref = h.register_batch([(scans[a], scans[b]) for a, b in pairs_idx], p)
        h.cache_reserve(9)
        slots = [7, 0, 3, 8, 1, 5]                                    # arbitrary slot placement
        h.cache_scans(scans, slots, p)
        got = h.register_cached([(slots[a], slots[b]) for a, b in pairs_idx], p)
        assert got.tobytes() == ref.tobytes()
        # odometry chain: swapTgt2Src = copy the target's slot over the source's
        h.cache_copy(slots[1], 2)
        again = h.register_cached([(2, slots[3])], p)
        direct = h.register_batch([(scans[1], scans[3])], p)
        assert again.tobytes() == direct.tobytes()
        # getSceneDescriptor / getTgtNormals: what the cache holds is what the stage entry points compute
        vox, nrm, desc = h.cache_read(slots[2])
        v_ref, _ = oracle.voxelize(scans[2], p.voxel_size, 1)
        n_ref, d_ref = oracle.compute_fpfh(v_ref, p.normal_radius, p.fpfh_radius, DEFAULT_CELL)
        assert same_bits(vox, v_ref)
        assert same_bits(desc, d_ref)
        assert same_bits(nrm, n_ref, nan_equal=True)
        # parameters other than the cached ones are refused
        q = default_params(); q.voxel_size = 0.25
        from quatro_b200.capi import QuatroB200Error
        with pytest.raises(QuatroB200Error):
            h.register_cached([(slots[0], slots[1])], q)


def test_tc_verify_whole_batch(monkeypatch):
    """QB200_TC_VERIFY=1: every nearest-neighbour table entry of a batch is recomputed by the exact CUDA-core kernel and compared
    with the tensor-core path's result: zero mismatches (the filter's error bound held for every entry)."""
    monkeypatch.setenv("QB200_TC_VERIFY", "1")
    p = default_params()
    pairs = [synth.outdoor_pair(80 + i)[:2] for i in range(4)]
    with Handle(max_batch_slots=4) as h:
        a = h.register_batch(pairs, p)
        v = h.debug_match_verify()
    assert v["compared"] > 4 * 10000 and v["mismatches"] == 0, v
    assert int(a["valid"].sum()) == 4


def test_dense_indoor_pair_50k_voxels(oracle):
    """BASELINE configs[4]: ~500 k points per scan, 0.05 m voxel -> ~34-53 k voxel points per cloud (max_voxel_points = 65536): the
    tensor-core matcher over 2.3e9 descriptor pairs, every stage counter and the pose identical to the CPU oracle."""
    src, tgt, T = synth.indoor_pair(0)
    p = default_params()
    p.voxel_size, p.normal_radius, p.fpfh_radius, p.noise_bound, p.cote_noise_bound, p.skip_flagged = 0.05, 0.10, 0.15, 0.05, 0.05, 0
    ref, st_ref = oracle.register_pair(src, tgt, p)
    with Handle(max_batch_slots=1, max_raw_points=524288, max_voxel_points=65536) as h:
        got, st = h.register_pair(src, tgt, p)
        stats = h.debug_match_stats()
    assert st == st_ref == 0 and got.valid == 1
    assert got.n_src_vox > 50000 and got.n_tgt_vox > 35000
    assert (got.n_src_vox, got.n_tgt_vox, got.n_mutual, got.n_corr, got.n_edges, got.max_core, got.clique_size) == \
           (ref.n_src_vox, ref.n_tgt_vox, ref.n_mutual, ref.n_corr, ref.n_edges, ref.max_core, ref.clique_size)
    assert np.allclose(got.matrix(), ref.matrix(), atol=1e-9)
    rot, tr = synth.pose_error(got.matrix(), T)
    assert rot < 2.0 and tr < 0.3
    assert stats["tiles"] > 0      # the tensor-core path ran (indoor planes produce near-tie stripes that fall back to the exact kernel: stats["aborted_stripes"])
