"""K8 (tim_graph_kernel, graph.cu) decides most pair tests in fp32 Gram form and sends a test to the literal fp64 expression only when
|t_c| <= q, when the column's smallest s' is near -beta^2, or when its M is beyond 2^62 (DESIGN 5.2).  The CPU tests run a host
restatement of the kernel (tests/fixtures/graph_band.cpp) on adversarial sets and check every fp32 decision against t and s' in
__float128 and against the literal expression, how close the sets come to the band, and that the sets really reach it.  The GPU tests
compare qb200_build_graph with the oracle on the same sets placed at the kernel's work-item edges, and whole solver waves that mix
noise bounds from 1e-6 to 1e9, INLIER_NONE pairs and pairs without work items."""
import subprocess

import numpy as np
import pytest

from support import P4, ROOT

REC = np.dtype([("set", "<i4"), ("i", "<i4"), ("j", "<i4"), ("dec32", "u1"), ("to64", "u1"), ("lit", "u1"), ("exact", "u1"),
                ("ratio", "<f8")])
TO64_BAND, TO64_NET, TO64_BIG = 1, 2, 4

BETAS = (1e-6, 0.05, 0.6, 10.0, 1e3)
OFFSETS = {"0": (0.0, 0.0, 0.0), "400 m": (400.0, -300.0, 20.0), "30 km": (3e4, -1e4, 5.0), "UTM": (5e5, 4.4e6, 30.0),
           "1e8 m": (1e8, 0.0, 0.0)}
DISTANCES = (1e-3, 1e-2, 0.1, 1.0, 10.0, 100.0, 1e3, 1e4)
KS = range(-8, 9)


# ---- the host restatement ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def band_exe(tmp_path_factory):
    exe = tmp_path_factory.mktemp("graph_band") / "graph_band"
    subprocess.run(["/usr/bin/g++", "-O2", "-ffp-contract=off", "-std=c++17", "-o", str(exe), str(ROOT / "tests" / "fixtures" / "graph_band.cpp")],
                   check=True)
    return exe


def restate(exe, sets, fix=True):
    """Every pair test tim_graph_kernel makes on `sets` (a list of (a4, b4, beta)), as REC records."""
    d = exe.parent
    with open(d / "in.bin", "wb") as f:
        f.write(np.int32(len(sets)).tobytes())
        for a4, b4, beta in sets:
            f.write(np.array([len(a4), 0], np.int32).tobytes() + np.array([beta / 2, 1.0], np.float64).tobytes())
            f.write(np.ascontiguousarray(a4, np.float32).tobytes() + np.ascontiguousarray(b4, np.float32).tobytes())
    subprocess.run([str(exe), str(d / "in.bin"), str(d / "out.bin")] + ([] if fix else ["nofix"]), check=True)
    return np.fromfile(d / "out.bin", REC)


def kernel_decision(r):
    return np.where(r["to64"] != 0, r["lit"], r["dec32"]).astype(bool)


# ---- adversarial sets: lists of (a4, b4, beta) with noise_bound = beta / 2, cbar2 = 1 ------------------------------------------------
def _unit(rng, n):
    u = rng.normal(size=(n, 3))
    return u / np.linalg.norm(u, axis=1, keepdims=True)


def _threshold_set(rng, beta, offset, d, jitter=None, step=2.0 ** -24):
    """34 point pairs (2m, 2m + 1) at distance d in a and d_b = d_a +- beta (1 + k step), k = -8 ... 8, near `offset`; d_a is taken
    from the rounded float32 points, so only the rounding of b_j moves a pair off its target.  step = 2^-24 puts the pairs inside the
    error band (relative width ~1e-4), step = 2^-12 just outside it."""
    n = 2 * len(KS)
    jit = min(d, 50.0) if jitter is None else jitter
    ai = P4(np.asarray(offset) + rng.uniform(-jit, jit, (n, 3)))[:, :3].astype(np.float64)
    aj = P4(ai + d * _unit(rng, n))[:, :3].astype(np.float64)
    bi = P4(ai + np.array([0.31, -0.17, 0.05]))[:, :3].astype(np.float64)
    da = np.linalg.norm(aj - ai, axis=1)
    sgn = np.repeat([1.0, -1.0], len(KS))
    k = np.tile(np.array(list(KS), np.float64), 2)
    db = np.abs(da + sgn * beta * (1 + k * step))
    bj = bi + db[:, None] * _unit(rng, n)
    a = np.empty((2 * n, 3)); b = np.empty((2 * n, 3))
    a[0::2], a[1::2], b[0::2], b[1::2] = ai, aj, bi, bj
    return P4(a), P4(b)


def threshold_sets(seed=1, step=2.0 ** -24):
    rng = np.random.default_rng(seed)
    out = []
    for beta in BETAS:
        for off in OFFSETS.values():
            for d in DISTANCES:
                a4, b4 = _threshold_set(rng, beta, off, d, step=step)
                out.append((a4, b4, beta))
    return out


def tight_block_sets(seed=2):
    """32-row blocks whose rows and columns all have the same norm R (M smallest against the pair), and one block where a single row of
    norm 1000 R widens M for the other 31."""
    rng = np.random.default_rng(seed)
    out = []
    for R, d, beta in ((1.0, 0.3, 0.05), (50.0, 2.0, 0.6), (100.0, 30.0, 0.6), (3e4, 10.0, 0.6), (3e4, 500.0, 10.0), (5e5, 1e3, 10.0),
                       (1e3, 100.0, 1e-6)):
        for huge in (False, True):
            n = 32
            sgn = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
            k = (np.arange(n) % 17) - 8
            da, db = np.full(n, d), np.abs(d + sgn * beta * (1 + k * 2.0 ** -24))
            pts = []
            for dist in (da, db):
                v = _unit(rng, n)
                w = np.cross(v, _unit(rng, n)); w /= np.linalg.norm(w, axis=1, keepdims=True)
                th = 2 * np.arcsin(np.clip(dist / (2 * R), 0, 1))
                p0, p1 = R * v, R * (np.cos(th)[:, None] * v + np.sin(th)[:, None] * w)
                x = np.empty((2 * n, 3)); x[0::2], x[1::2] = p0, p1
                pts.append(x)
            a, b = pts
            if huge:
                a[5] *= 1000.0; b[5] *= 1000.0
            out.append((P4(a), P4(b), beta))
    return out


def smin_net_sets():
    """Both distances ~0: coincident points in both clouds and in one, 1 ulp apart, subnormal coordinates and differences, +-0.0."""
    f = np.float32
    tiny = np.float32(1e-40)
    a = [[0, 0, 0], [0, 0, 0], [-0.0, 0.0, -0.0], [1, 2, 3], [1, 2, 3], [1, 2, np.nextafter(f(3), f(4))], [tiny, 0, 0], [2 * tiny, 0, 0],
         [0, tiny, -tiny], [5, 5, 5], [5, 5, 5], [np.nextafter(f(5), f(6)), 5, 5], [1e-38, 1e-38, 0], [1e-38, np.nextafter(f(1e-38), f(1)), 0],
         [400.0, 400.0, 0.0], [400.0, 400.0, 0.0], [np.nextafter(f(400), f(500)), 400, 0]]
    b = [[0, 0, 0], [0, 0, 0], [0.0, -0.0, 0.0], [1, 2, 3], [1, 2, np.nextafter(f(3), f(4))], [1, 2, 3], [tiny, 0, 0], [tiny, tiny, 0],
         [0, -tiny, tiny], [5, 5, 5], [5.3, 5, 5], [5, 5, 5], [1e-38, 1e-38, 0], [1e-38, 1e-38, 0], [400.0, 400.0, 0.0],
         [np.nextafter(f(400), f(500)), 400.0, 0.0], [400.0, 400.0, 0.0]]
    out = []
    for beta in (1e-6, 0.05, 0.6):
        out.append((P4(a), P4(b), beta))
        out.append((P4(np.array(a) + [75.0, -20.0, 3.0]), P4(np.array(b) + [75.0, -20.0, 3.0]), beta))
    return out


def overflow_sets(beta, X, n=400):
    """The pair (X, 0, 0) -> (-X, 1, 0) in a, (X, 0, 0) -> (-X + o, 1, 0) in b, o = beta (-1.5 + 3 k / n): 2 beta^2 s' overflows."""
    out = []
    for k in range(n):
        off = beta * (-1.5 + 3.0 * k / n)
        a = P4([[X, 0, 0], [-X, 1, 0]])
        b = P4([[X, 0, 0], [-X + off, 1, 0]])
        out.append((a, b, beta))
    return out


def float_range_sets(seed=3):
    """beta up to 1e9, coordinates up to 1e19 and FLT_MAX (M overflows), NaN and +-inf in one coordinate of one cloud and of both."""
    rng = np.random.default_rng(seed)
    fmax = float(np.finfo(np.float32).max)
    out = []
    for beta, X in ((1e6, 1e13), (1e9, 1e10), (1e9, 1e9), (1e9, 1e12), (10.0, 1e17), (10.0, 1e19), (1e3, fmax), (0.6, 1e19), (0.6, 1e18)):
        a, b = _threshold_set(rng, beta, (X, -0.5 * X, 0.25 * X), min(max(4 * beta, 1.0), 1e12), jitter=0.0)
        out.append((a, b, beta))
        a = P4(rng.uniform(-1, 1, (40, 3)) * min(X, fmax / 2)); b = a.copy(); b[::3, 1] *= -1
        out.append((a, b, beta))
    base_a = P4(rng.uniform(-3, 3, (48, 3))); base_b = base_a + np.float32(0.2) * P4(rng.normal(size=(48, 3)), 0.0)
    for val in (np.nan, np.inf, -np.inf):
        for where in ("a", "b", "both"):
            for idx, col in ((0, 0), (7, 2), (31, 1), (32, 0), (47, 2)):
                a, b = base_a.copy(), base_b.copy()
                if where in ("a", "both"):
                    a[idx, col] = val
                if where in ("b", "both"):
                    b[idx, col] = val
                out.append((a, b, 0.6))
    return out


def _max_ratio(recs):
    r = recs[recs["to64"] == 0]["ratio"]
    r = r[np.isfinite(r)]
    return float(r.max()) if len(r) else 0.0


def hill_climb(exe, seed=4, gens=30, cands=8):
    """From threshold pairs just outside the band as two-point sets, move b_j and a_j by 1 ... 4 ulps and keep a move when it raises
    the largest |t_c - t| / q among the set's fp32-decided tests."""
    rng = np.random.default_rng(seed)
    start = []
    for beta in BETAS:
        for off in list(OFFSETS.values())[:3]:     # further out the smin net takes every test
            for d in (0.1, 1.0, 10.0, 100.0):
                a4, b4 = _threshold_set(rng, beta, off, d, step=2.0 ** -8)
                for m in (0, 8, 17, 25):
                    start.append([a4[2 * m:2 * m + 2].copy(), b4[2 * m:2 * m + 2].copy(), beta])
    recs = restate(exe, [tuple(s) for s in start])
    best = np.array([_max_ratio(recs[recs["set"] == i]) for i in range(len(start))])
    for _ in range(gens):
        trial = []
        for s in start:
            for _ in range(cands):
                a4, b4 = s[0].copy(), s[1].copy()
                for x in (a4, b4):
                    c = rng.integers(0, 3)
                    steps = int(rng.integers(1, 5)) * (1 if rng.uniform() < 0.5 else -1)
                    v = x[1, c]
                    for _ in range(abs(steps)):
                        v = np.nextafter(v, np.float32(np.inf) if steps > 0 else np.float32(-np.inf))
                    x[1, c] = v
                trial.append((a4, b4, s[2]))
        recs = restate(exe, trial)
        order = np.argsort(recs["set"], kind="stable")
        bounds = np.searchsorted(recs["set"][order], np.arange(len(trial) + 1))
        for n, s in enumerate(start):
            for c in range(cands):
                t = n * cands + c
                r = recs[order[bounds[t]:bounds[t + 1]]]
                v = _max_ratio(r)
                if v > best[n]:
                    best[n] = v
                    s[0], s[1] = trial[t][0], trial[t][1]
    return [tuple(s) for s in start], best


# ---- CPU: the restatement against exact arithmetic ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def climbed(band_exe):
    return hill_climb(band_exe)


def _check_decisions(recs, label):
    """Every fp32-decided test equals the exact sign and the literal fp64 expression, |t_c - t| < q on every one of them, and the
    kernel's decision equals the literal expression on every test.  Returns the largest |t_c - t| / q."""
    f32 = recs[recs["to64"] == 0]
    bad = f32[(f32["dec32"] != f32["exact"]) | (f32["dec32"] != f32["lit"])]
    assert len(bad) == 0, (label, len(bad), bad[:5])
    wrong = recs[kernel_decision(recs) != recs["lit"].astype(bool)]
    assert len(wrong) == 0, (label, len(wrong), wrong[:5])
    r = f32["ratio"][np.isfinite(f32["ratio"])]
    assert len(r) == 0 or r.max() < 1.0, (label, r.max())
    return _max_ratio(recs)


def _to64_share(recs, n_sets, groups):
    """Share of the pair tests the kernel sends to fp64, per group name (groups[s]: the name of set s)."""
    per_set = np.bincount(recs["set"], minlength=n_sets)
    to64 = np.bincount(recs["set"], weights=recs["to64"] != 0, minlength=n_sets)
    names = np.array(groups)
    return {g: float(to64[names == g].sum() / per_set[names == g].sum()) for g in dict.fromkeys(groups)}


@pytest.mark.parametrize("step,reached", [(2.0 ** -24, 0.160), (2.0 ** -12, 0.181)])
def test_threshold_pairs_decide_exactly(band_exe, step, reached):
    sets = threshold_sets(step=step)
    recs = restate(band_exe, sets)
    worst = _check_decisions(recs, "threshold")
    assert (recs["to64"] & TO64_BAND).any() and ((recs["to64"] == 0) & (recs["dec32"] == 1)).any()
    # the generator comes close to the band: `reached` is what it reaches on this seed; a blunted generator fails here
    assert worst >= reached / 2, worst
    # the share of tests the kernel sends to fp64, per offset (counted, DESIGN 5.2): far out, the smin net takes all of them
    share = _to64_share(recs, len(sets), [name for _ in BETAS for name in OFFSETS for _ in DISTANCES])
    assert share["0"] < 0.3 and share["30 km"] > 0.8 and share["UTM"] == 1.0 and share["1e8 m"] == 1.0, share


def test_tight_blocks_and_hill_climb_stay_inside_the_bound(band_exe, climbed):
    worst_tight = _check_decisions(restate(band_exe, tight_block_sets()), "tight blocks")
    sets, best = climbed
    worst_climb = _check_decisions(restate(band_exe, sets), "hill climb")
    assert np.isclose(worst_climb, best.max())
    # reached on these seeds: 0.191 on the tight blocks, 0.174 after the climb (from 0 on most of its starting pairs)
    assert worst_tight >= 0.191 / 2, worst_tight
    assert worst_climb >= 0.174 / 2, worst_climb


def test_smin_net_and_float_range_ends(band_exe):
    for label, sets in (("smin net", smin_net_sets()), ("float range", float_range_sets())):
        recs = restate(band_exe, sets)
        _check_decisions(recs, label)
        assert (recs["to64"] & (TO64_NET if label == "smin net" else TO64_BIG)).any(), label


@pytest.mark.parametrize("beta,X,count", [(1e9, 1e10, 133), (1e6, 1e13, 261)])
def test_overflowing_pair_tests_go_to_fp64(band_exe, beta, X, count):
    """2 beta^2 s' overflows, t = -inf and |t| - q = +inf: without the M guard the fp32 path calls every such pair an edge."""
    sets = overflow_sets(beta, X)
    recs = restate(band_exe, sets)
    assert (kernel_decision(recs) == recs["lit"].astype(bool)).all()
    assert (recs["to64"] & TO64_BIG).all()
    old = restate(band_exe, sets, fix=False)
    wrong = kernel_decision(old) != old["lit"].astype(bool)
    # two tests per set (both orders on the diagonal block), each wrong for every non-edge
    assert wrong.sum() == 2 * count and (~old["lit"].astype(bool)).sum() == 2 * count


def test_restatement_equals_the_oracle(band_exe, oracle):
    """The adjacency the restated kernel produces, both halves, equals the oracle's on every kind of set."""
    sets = threshold_sets()[::7] + tight_block_sets() + smin_net_sets() + float_range_sets() + overflow_sets(1e9, 1e10, 8)
    recs = restate(band_exe, sets)
    dec = kernel_decision(recs)
    for s, (a4, b4, beta) in enumerate(sets):
        L = len(a4)
        m = recs["set"] == s
        got = np.zeros((L, L), bool)
        got[recs["j"][m], recs["i"][m]] = dec[m]    # the column's word holds the bit of (row i, column j) at row j
        off = m & (recs["j"] // 32 != recs["i"] // 32)
        got[recs["i"][off], recs["j"][off]] = dec[off]
        adj, _, _ = oracle.build_graph(a4, b4, beta / 2, 1.0)
        want = np.unpackbits(adj.view(np.uint8), axis=1, bitorder="little")[:, :L].astype(bool)
        assert np.array_equal(got, want), (s, int((got != want).sum()))


# ---- GPU: qb200_build_graph and whole solver waves against the oracle ----------------------------------------------------------------
@pytest.fixture(scope="module")
def h8k():
    from quatro_b200.capi import Handle
    with Handle(max_batch_slots=4, max_corr=8192) as h:
        yield h


def _same_graph(h, oracle, a4, b4, beta, label):
    """qb200_build_graph equals the oracle bit for bit (adjacency, degrees, edge count) and the numpy float64 restatement off its
    knife edge."""
    from independent_ref import tim_graph
    g, dg, ng = h.build_graph(a4, b4, beta / 2, 1.0)
    r, dr, nr = oracle.build_graph(a4, b4, beta / 2, 1.0)
    assert np.array_equal(g, r), (label, int((g != r).sum()))
    assert np.array_equal(dg, dr) and ng == nr, label
    L = len(a4)
    if 0 < L <= 1024:
        a, b = a4[:, :3].astype(np.float64), b4[:, :3].astype(np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            e, _ = tim_graph(a, b, beta)
            da = np.linalg.norm(a[:, None] - a[None], axis=2); db = np.linalg.norm(b[:, None] - b[None], axis=2)
            knife = np.abs(np.abs(da - db) - beta) <= 1e-12 * (da + db + beta)   # where two float64 evaluations may differ
        got = np.unpackbits(g.view(np.uint8), axis=1, bitorder="little")[:, :L].astype(bool)
        assert np.array_equal(got[~knife], e[~knife]), (label, int((got[~knife] != e[~knife]).sum()))


def _placed(L, seed):
    """L points whose pairs scatter around |d_a - d_b| = 0.6, with threshold pairs placed on rows 31 / 32, on columns 127 / 128 and
    inside diagonal blocks."""
    rng = np.random.default_rng(seed)
    a = rng.uniform(-20, 20, (L, 3)); b = a + rng.normal(0, 0.35, (L, 3))
    ta, tb = _threshold_set(rng, 0.6, (0.0, 0.0, 0.0), 3.0)
    slots = [(31, 32), (127, 128), (5, 6), (64 + 9, 64 + 10), (31, 128), (0, L - 1), (L - 2, L - 1), (4094, 4095), (4095, 4096)]
    m = 0
    for i, j in slots:
        if 0 <= i < j < L:
            a[i], a[j], b[i], b[j] = ta[2 * m, :3], ta[2 * m + 1, :3], tb[2 * m, :3], tb[2 * m + 1, :3]
            m += 1
    return P4(a), P4(b)


@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 4095, 4096, 4097])
def test_build_graph_at_work_item_edges(h8k, oracle, L):
    _same_graph(h8k, oracle, *_placed(L, 100 + L), 0.6, L)


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["threshold", "outside the band", "tight blocks", "hill climb", "smin net", "float range"])
def test_build_graph_on_adversarial_sets(h8k, oracle, climbed, family):
    sets = {"threshold": lambda: threshold_sets(), "outside the band": lambda: threshold_sets(step=2.0 ** -12),
            "tight blocks": tight_block_sets, "hill climb": lambda: climbed[0], "smin net": smin_net_sets,
            "float range": float_range_sets}[family]()
    for s, (a4, b4, beta) in enumerate(sets):
        _same_graph(h8k, oracle, a4, b4, beta, (family, s))


@pytest.mark.gpu
@pytest.mark.parametrize("beta,X", [(1e9, 1e10), (1e6, 1e13)])
def test_build_graph_where_m_overflows(h8k, oracle, beta, X):
    """The overflow pairs one per two-point set and all 400 in one set of 800 points (cross pairs included)."""
    sets = overflow_sets(beta, X)
    for s in (0, 1, 133, 200, 266, 399):
        _same_graph(h8k, oracle, *sets[s][:2], beta, s)
    a4 = np.concatenate([s[0] for s in sets]); b4 = np.concatenate([s[1] for s in sets])
    _same_graph(h8k, oracle, a4, b4, beta, "800 points")


def _mixed_sets(seed=7):
    """Correspondence sets of 0 ... 700 matched points with noise bounds from 1e-6 to 1e9 (beta = 2 noise_bound), INLIER_NONE pairs,
    and sets of L = 0, 1, 2 first, in the middle and last."""
    from quatro_b200 import synth
    from quatro_b200.capi import INLIER_NONE, PMC_HEU, default_params
    rng = np.random.default_rng(seed)
    sets, params = [], []

    def add(a4, b4, nb, mode=PMC_HEU):
        p = default_params()
        p.noise_bound, p.inlier_selection_mode = nb, mode
        p.rot_noise_bound = nb      # explicit: no pair takes the handle's latched rotation noise bound
        sets.append((a4, b4)); params.append(p)

    def tiny(L):
        a = P4(rng.uniform(-5, 5, (L, 3))); return a, a + P4(rng.normal(0, 0.1, (L, 3)), 0.0)

    for L in (0, 1, 2):
        add(*tiny(L), 0.3)
    for k, nb in enumerate((5e-7, 0.025, 0.3, 5.0, 500.0, 5e5, 5e8)):
        L = (300, 33, 700, 129, 64, 257, 500)[k]
        a4, b4, _, _ = synth.matched_pairs(900 + k, L, inlier_ratio=0.3, noise=0.05)
        if nb >= 5e5:
            a4[:, :3] *= np.float32(1e3); b4[:, :3] *= np.float32(1e3)     # beta of 1e6 / 1e9 against 1e4 m clouds
        add(a4, b4, nb)
        if k == 3:
            for L0 in (2, 0, 1):
                add(*tiny(L0), 0.3)
            add(a4, b4, nb, INLIER_NONE)
    ov = overflow_sets(1e9, 1e10, 40)
    add(np.concatenate([s[0] for s in ov]), np.concatenate([s[1] for s in ov]), 5e8)
    add(*tiny(300), 0.3, INLIER_NONE)
    for L in (1, 0, 2):
        add(*tiny(L), 0.3)
    return sets, params


def _check_wave(oracle, sets, params, recs, lists):
    for s, ((a4, b4), p, r, lst) in enumerate(zip(sets, params, recs, lists)):
        ro, st, clique, _ = oracle.solve_correspondences(a4, b4, p, want_sets=True)
        for k in ("n_corr", "n_edges", "max_core", "clique_size"):
            assert r[k] == getattr(ro, k), (s, k, r[k], getattr(ro, k))
        assert np.array_equal(lst["clique"], clique), s
        if 2 * p.noise_bound <= 10:
            assert r["status"] == st and np.allclose(np.asarray(r["T"]).reshape(4, 4).T, ro.matrix(), atol=1e-9, rtol=0), s


@pytest.mark.gpu
def test_mixed_noise_bounds_in_one_wave_and_in_queued_waves(oracle):
    """Pairs of very different beta share warps through the per-warp constants; pairs without work items sit between them in the
    prefix of item counts.  One qb200_solve_batch_each wave, then two queued waves and one flush."""
    from quatro_b200.capi import Handle, ListBuffers, MEM_HOST, RESULT_DTYPE, SET_LISTS
    sets, params = _mixed_sets()
    n = len(sets)
    with Handle(max_batch_slots=n, max_corr=1024) as h:
        lb = ListBuffers(n, 1024, MEM_HOST, SET_LISTS)
        recs, lists = h.solve_batch_each(sets, params, buffers=lb)
        _check_wave(oracle, sets, params, recs, lists)
        half = n // 2
        parts = [(sets[:half], params[:half]), (sets[half:][::-1], params[half:][::-1])]
        keep, outs, bufs = [], [], []
        for ss, ps in parts:
            arr, k = h._set_array(ss, MEM_HOST)
            pa = h.params_array(ps)
            out = np.zeros(len(ss), RESULT_DTYPE)
            b = ListBuffers(len(ss), 1024, MEM_HOST, SET_LISTS)
            keep.append((arr, k, pa)); outs.append(out); bufs.append(b)
            h.solve_batch_enqueue_each_raw(arr, len(ss), pa, MEM_HOST, out, b)
        h.register_batch_flush()
        for (ss, ps), out, b in zip(parts, outs, bufs):
            _check_wave(oracle, ss, ps, out, b.trimmed(out))


@pytest.mark.gpu
def test_full_prefix_of_2048_slots(oracle):
    """A wave of 2048 sets fills the kernel's prefix of per-pair item counts (kGraphMaxPairs + 1 entries)."""
    from quatro_b200.capi import Handle, ListBuffers, MEM_HOST, SET_LISTS, default_params
    rng = np.random.default_rng(9)
    sets, params = [], []
    for s in range(2048):
        L = int(rng.integers(0, 65))
        a = P4(rng.uniform(-10, 10, (L, 3))); b = a + P4(rng.normal(0, 0.3, (L, 3)), 0.0)
        if s % 97 == 0 and L >= 2:
            a[0, :3] = [1e10, 0, 0]; a[1, :3] = [-1e10, 1, 0]; b[0, :3] = [1e10, 0, 0]; b[1, :3] = [-1e10 + 3e8, 1, 0]
        p = default_params()
        p.noise_bound = 5e8 if s % 97 == 0 else float(rng.choice([0.05, 0.3, 0.6]))
        sets.append((a, b)); params.append(p)
    with Handle(max_batch_slots=2048, max_corr=64, max_raw_points=256, max_voxel_points=128) as h:
        recs, lists = h.solve_batch_each(sets, params, buffers=ListBuffers(2048, 64, MEM_HOST, SET_LISTS))
    for s in list(range(0, 2048, 7)) + [2047] + list(range(0, 2048, 97)):
        a4, b4 = sets[s]
        ro, st, clique, _ = oracle.solve_correspondences(a4, b4, params[s], want_sets=True)
        assert (recs["n_edges"][s], recs["max_core"][s], recs["clique_size"][s]) == (ro.n_edges, ro.max_core, ro.clique_size), s
        assert np.array_equal(lists[s]["clique"], clique), s
