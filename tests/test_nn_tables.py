"""Both nearest-neighbour tables of the matcher (K6), entry for entry, against the oracle on adversarial descriptors.

The correspondence list only shows mutual pairs, and most wrong row or column bests cannot change it.  These tests read the
whole tables: `qb200_debug_nn_tables` (the GPU's `rowbest` / `colbest` after any exact redo) against `qo_nn_tables` (the
oracle's fp32 fma chain, lowest-index ties, NaN never wins), bit for bit, on the tensor-core path and on a handle created
with QB200_MATCH_EXACT=1.  The families aim at the parts of tc_nn_kernel (csrc/tc_match.cu) that approximate and then
correct: the filter margin, the tile skipping (norm-gap bound, the 256-tile window, the column-max cache), duplicate classes,
the abort to the exact kernel, and non-finite or overflowing descriptors.

The CPU tests pin the oracle itself: float64 argmins, mutual pairs, and exact power-of-two scale invariance."""
import numpy as np
import pytest

from quatro_b200.capi import default_params
from support import P4, fpfh_like

NONE = np.uint64(0xFFFFFFFFFFFFFFFF)
MU = np.zeros(33, np.float32)
MU[[5, 16, 27]] = 100.0     # the centring vector of tc_match.cu (FPFH of a plane)


# ---- descriptor families ----------------------------------------------------------------------------------------------
def _norm_chain(x):
    """|x - mu|^2 by the fp32 chain of norm_key_kernel / split_desc_kernel (fma emulated in float64, exact for a square)."""
    xc = (x.astype(np.float32) - MU).astype(np.float32)
    acc = np.zeros(len(x), np.float32)
    for d in range(33):
        acc = (xc[:, d].astype(np.float64) ** 2 + acc.astype(np.float64)).astype(np.float32)
    return acc


def _unit(rng, n):
    u = rng.standard_normal((n, 33))
    return u / np.linalg.norm(u, axis=1, keepdims=True)


def fam_scaled(rng, k, na=1500, nb=2100):
    """FPFH-like descriptors scaled by 2^k: small k collapses every centred norm onto |mu|, large k stresses the margins."""
    s = np.float32(2.0 ** k)
    return (fpfh_like(rng, na) * s).astype(np.float32), (fpfh_like(rng, nb) * s).astype(np.float32)


def fam_clustered(rng, n=8192, k=16):
    """k clusters at well-separated norms, spread inside each cluster, plus near-duplicates: heavy skipping."""
    def cloud(m):
        c = rng.integers(0, k, m)
        centre = MU + (60.0 * (c + 1))[:, None] * _unit(np.random.default_rng(77), k)[c]
        x = centre + rng.normal(0, 4.0, (m, 33))
        dup = rng.random(m) < 0.15
        src = rng.integers(0, m, m)
        x[dup] = x[src[dup]] + rng.normal(0, 1e-3, (dup.sum(), 33))
        return x.astype(np.float32)
    return cloud(n), cloud(n)


def fam_shell(rng, na=2048, nb=4096, r=100.0):
    """Every descriptor at the same centred norm: no tile can be skipped, the walk must reach every tile."""
    return (MU + r * _unit(rng, na)).astype(np.float32), (MU + r * _unit(rng, nb)).astype(np.float32)


def fam_collinear(rng, scale, n_sel=1024, m=6144):
    """Collinear near-ties.  Row a = mu + R u, its true neighbour b = mu + (R + g) u (distance g^2, norm gap g), a decoy
    c = a + g (1 + 1e-4) v (v orthogonal to u) in the row's nearest-norm tiles, and a twin row of b that settles b's column
    early.  Of m candidate directions the n_sel are kept whose fp32 norm chains put a LOW and b HIGH, so the computed gap between
    the a stripes and the b tiles exceeds the true one as far as rounding allows: a bound without enough slack skips b."""
    R, g = 128.0 * scale, scale / 64.0
    u = _unit(rng, m)
    w = rng.standard_normal((m, 33))
    v = w - (w * u).sum(1, keepdims=True) * u
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    a = (MU + R * u).astype(np.float32)
    b = (MU + (R + g) * u).astype(np.float32)
    na, nb = np.sqrt(_norm_chain(a)), np.sqrt(_norm_chain(b))
    score = (nb.astype(np.float64) - nb.mean()) - (na.astype(np.float64) - na.mean())
    sel = np.argsort(-score, kind="stable")[:n_sel]
    a, b, u, v = a[sel], b[sel], u[sel], v[sel]
    c = (MU + R * u + g * (1 + 1e-4) * v).astype(np.float32)
    twin = (b + 1e-2 * g * _unit(rng, n_sel)).astype(np.float32)
    A, B = np.concatenate([a, twin]), np.concatenate([c, b])
    return A[rng.permutation(len(A))], B[rng.permutation(len(B))]


def fam_wide(rng, nb, na=2048, n_low=512):
    """nb columns, the true neighbours of most rows among the highest norms (column tiles >= 256 once nb > 16384)."""
    B = fpfh_like(rng, nb)
    hi = (MU + rng.uniform(400, 900, (na - n_low, 1)) * _unit(rng, na - n_low)).astype(np.float32)
    B[nb - len(hi):] = (hi + rng.normal(0, 0.5, hi.shape)).astype(np.float32)
    # 64 isolated columns above every other norm (tile 256 alone at nb = 16448): their own column bound keeps them from
    # being skipped, the bound of any other tile would not
    B[:64] = (MU + 3000.0 * _unit(rng, 64)).astype(np.float32)
    A = np.concatenate([hi, (B[rng.integers(0, nb - len(hi), n_low)] + rng.normal(0, 0.3, (n_low, 33))).astype(np.float32)])
    return A[rng.permutation(na)], B[rng.permutation(nb)]


def fam_equal_keys(rng, n_base=48, per=6, n_rows=1500):
    """Bin permutations of a descriptor whose fp32 norm chain gives the same bits (different descriptors, equal sort keys),
    interleaved with bit-identical copies in index order P, Q, P, R, P, ...: dedup_kernel may only merge bit-identical runs."""
    free = np.array([d for d in range(33) if MU[d] == 0])
    cols = []
    for base in fpfh_like(rng, n_base):
        key = _norm_chain(base[None])[0]
        perms = []
        for _ in range(400):
            q = base.copy()
            q[free] = base[rng.permutation(free)]
            if _norm_chain(q[None])[0] == key and not np.array_equal(q, base) and not any(np.array_equal(q, p) for p in perms):
                perms.append(q)
            if len(perms) == per:
                break
        for q in perms:
            cols += [base, q]
        cols.append(base)
    cols.append(MU)        # the plane signature on both sides: its lower bound is exactly 0 = its exact distance
    B = np.array(cols, np.float32)
    A = np.concatenate([B[rng.integers(0, len(B), n_rows // 2)], fpfh_like(rng, n_rows - n_rows // 2)])
    A[::3] = (A[::3] + rng.normal(0, 0.05, A[::3].shape)).astype(np.float32)
    A[1] = MU
    return A.astype(np.float32), B


def fam_ulp(rng, na=1100, nb=1300):
    """1-ulp perturbations of one descriptor in random bins (none bit-identical): every entry is a near-tie."""
    base = fpfh_like(rng, 1)[0] + np.float32(1.0)
    def cloud(n):
        x = np.tile(base, (n, 1))
        up = rng.random((n, 33)) < 0.3
        x[up] = np.nextafter(x[up], np.float32(np.inf))
        return x
    return cloud(na), cloud(nb)


def fam_nonfinite(rng, na=300, nb=400):
    """NaN / +-inf in one bin of a few rows and columns, and finite descriptors whose centred squared norm overflows."""
    A, B = fpfh_like(rng, na), fpfh_like(rng, nb)
    A[3, 4] = np.nan; A[10, 7] = np.inf; A[11, 7] = -np.inf; A[12, 20] = np.inf
    B[5, 7] = np.inf; B[6, 0] = np.nan; B[8, 20] = -np.inf
    A[20] = 0; A[20, :2] = 2e19; B[30] = A[20]; B[30, 10] = 1.0           # exact distance 1, |x'|^2 = 8e38 overflows
    A[21] = 0; A[21, 2] = 5e18; B[31] = A[21]; B[31, 12] = 2.0            # finite norm 2.5e37, above the tensor-core range
    return A, B


# ---- helpers ------------------------------------------------------------------------------------------------------------
def _dist(packed):
    return (packed >> np.uint64(32)).astype(np.uint32).view(np.float32)


def _idx(packed):
    return np.where(packed == NONE, -1, (packed & np.uint64(0xFFFFFFFF)).astype(np.int64))


def _mutual_from_tables(rb, cb):
    """match()'s mutual pairs from the tables: ascending index of the larger cloud (the source on ties)."""
    swapped = len(cb) > len(rb)
    first, second = (cb, rb) if swapped else (rb, cb)
    out = []
    for i, p in enumerate(first):
        j = _idx(p)
        if j >= 0 and _idx(second[j]) == i:
            out.append((i, j))
    return np.array(out, np.int32).reshape(-1, 2)


def _table_diff(name, got, ref):
    bad = np.flatnonzero(got != ref)
    if len(bad) == 0:
        return ""
    show = ", ".join(f"{i}: got ({_dist(got[i:i + 1])[0]!r}, {_idx(got[i:i + 1])[0]}) want ({_dist(ref[i:i + 1])[0]!r}, "
                     f"{_idx(ref[i:i + 1])[0]})" for i in bad[:4])
    return f"{name}: {len(bad)} of {len(ref)} entries differ ({show})"


# ---- CPU: the oracle against float64 -------------------------------------------------------------------------------------
def _small_families(rng):
    yield "fpfh-16", fam_scaled(rng, -16, 200, 260)
    yield "fpfh+32", fam_scaled(rng, 32, 200, 260)
    yield "clustered", fam_clustered(rng, 400, 6)
    yield "shell", fam_shell(rng, 150, 230)
    yield "collinear", fam_collinear(rng, 256.0, 128, 512)
    yield "wide", fam_wide(rng, 700, 200, 50)
    yield "equal-keys", fam_equal_keys(rng, 8, 4, 150)
    yield "ulp", fam_ulp(rng, 120, 140)
    yield "nonfinite", fam_nonfinite(rng, 60, 70)


def _check_against_float64(A, B, best, axis_rows, rng, block=64):
    """Each oracle index is the float64 argmin of its row (NaN ignored) or ties with it within 1e-5 relative; a distance the
    fp32 chain overflowed to +inf must be one float64 puts above FLT_MAX."""
    rows = np.unique(np.concatenate([np.arange(min(block, len(A))), rng.integers(0, len(A), block)]))
    a64, b64 = A[rows].astype(np.float64), B.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        D = ((a64[:, None, :] - b64[None, :, :]) ** 2).sum(2)
    for r, i in enumerate(rows):
        row = D[r]
        ok = ~np.isnan(row)
        j = _idx(best[i:i + 1])[0]
        if not ok.any():
            assert j == -1, (axis_rows, i)
            continue
        m = row[ok].min()
        assert j >= 0 and ok[j], (axis_rows, i, j)
        dj = float(_dist(best[i:i + 1])[0])
        if np.isinf(dj):
            assert row[j] > np.finfo(np.float32).max and m > np.finfo(np.float32).max * 0.5, (axis_rows, i, row[j], m)
        else:
            assert row[j] <= m * (1 + 1e-5) + 1e-30, (axis_rows, i, j, row[j], m)
            assert abs(dj - row[j]) <= 1e-5 * row[j] + 1e-30, (axis_rows, i, dj, row[j])


def test_oracle_tables_against_float64(oracle):
    rng = np.random.default_rng(7)
    p = default_params()
    p.use_tuple_test = 0
    for name, (A, B) in _small_families(rng):
        rb, cb = oracle.nn_tables(A, B)
        assert len(rb) == len(A) and len(cb) == len(B)
        _check_against_float64(A, B, rb, name + " rows", rng)
        _check_against_float64(B, A, cb, name + " cols", rng)
        # the mutual pairs derived from the tables are the ones match() lists
        _, nm, _, mutual = oracle.match(P4(rng.uniform(-30, 30, (len(A), 3))), A, P4(rng.uniform(-30, 30, (len(B), 3))), B, p,
                                        want_mutual=True)
        got = _mutual_from_tables(rb, cb)
        assert nm == len(got) and np.array_equal(got, mutual), name


def test_oracle_tables_nonfinite_semantics(oracle):
    """NaN never wins; inf is a valid candidate; the overflowing pair keeps its finite distance."""
    A, B = fam_nonfinite(np.random.default_rng(3), 60, 70)
    rb, cb = oracle.nn_tables(A, B)
    assert rb[3] == NONE                                           # a NaN bin makes every distance of row 3 NaN
    assert cb[6] == NONE
    assert np.isinf(_dist(rb[10:11])[0]) and _idx(rb[10:11])[0] == 0  # inf row: every finite column ties at +inf -> lowest index
    assert _idx(rb[20:21])[0] == 30 and _dist(rb[20:21])[0] == 1.0 and _idx(cb[30:31])[0] == 20
    assert _idx(rb[21:22])[0] == 31 and _dist(rb[21:22])[0] == 4.0 and _idx(cb[31:32])[0] == 21


def test_oracle_tables_power_of_two_invariance(oracle):
    """Scaling both sets by 2^k commutes with every fp32 rounding while all values stay normal: indices unchanged, distances
    times exactly 4^k.  Values are multiples of 2^-10 in [2^-10, 2^7), so every nonzero difference is >= 2^-42 at k = -32
    and every square and sum stays below 2^120 at k = 48."""
    rng = np.random.default_rng(19)
    def quant(x):
        q = np.round(x.astype(np.float64) * 1024.0) / 1024.0
        return np.where(q < 2.0 ** -10, 0.0, q).astype(np.float32)
    A, B = quant(fpfh_like(rng, 300)), quant(fpfh_like(rng, 340))
    B[:40] = A[:40]
    B[40:80] = quant(A[40:80] + rng.normal(0, 0.01, (40, 33)))
    rb0, cb0 = oracle.nn_tables(A, B)
    d_rb0, d_cb0 = _dist(rb0).astype(np.float64), _dist(cb0).astype(np.float64)
    for k in range(-32, 49):
        s = np.float32(2.0 ** k)
        rb, cb = oracle.nn_tables(A * s, B * s)
        assert np.array_equal(_idx(rb), _idx(rb0)) and np.array_equal(_idx(cb), _idx(cb0)), k
        assert np.array_equal(_dist(rb).astype(np.float64), d_rb0 * 4.0 ** k), k
        assert np.array_equal(_dist(cb).astype(np.float64), d_cb0 * 4.0 ** k), k


# ---- GPU: both tables bit for bit, tensor-core path and exact kernel ------------------------------------------------------
@pytest.fixture(scope="module")
def handles():
    from quatro_b200.capi import Handle
    tc = Handle(max_batch_slots=2)
    with pytest.MonkeyPatch.context() as mp:       # a module fixture has no monkeypatch of its own
        mp.setenv("QB200_MATCH_EXACT", "1")
        ex = Handle(max_batch_slots=2)
    yield tc, ex
    tc.close()
    ex.close()


def _run_case(h, A, B, a4, b4, p, ref, want, label):
    """qb200_match on h: both tables and the correspondence list against the oracle's; returns the matcher counters."""
    h.debug_match_stats(reset=True)
    got = h.match(a4, A, b4, B, p)
    stats = h.debug_match_stats(reset=True)
    rb, cb = h.debug_nn_tables(len(A), len(B))
    msg = "; ".join(m for m in (_table_diff("rowbest", rb, ref[0]), _table_diff("colbest", cb, ref[1])) if m)
    assert not msg, f"{label}: {msg} (matcher counters {stats})"
    assert np.array_equal(got[0], want[0]) and got[1] == want[1], f"{label}: correspondence list differs"
    return stats


def _both_paths(handles, oracle, A, B, label):
    rng = np.random.default_rng(len(A) * 7919 + len(B))
    a4, b4 = P4(rng.uniform(-30, 30, (len(A), 3))), P4(rng.uniform(-30, 30, (len(B), 3)))
    p = default_params()
    p.use_tuple_test = 0
    ref, want = oracle.nn_tables(A, B), oracle.match(a4, A, b4, B, p)
    tc, ex = handles
    st_tc = _run_case(tc, A, B, a4, b4, p, ref, want, label + " (tensor cores)")
    st_ex = _run_case(ex, A, B, a4, b4, p, ref, want, label + " (QB200_MATCH_EXACT=1)")
    assert st_ex["tiles"] == 0 and st_ex["aborted_stripes"] == 0, st_ex     # the exact kernel only
    assert st_tc["tiles"] > 0, st_tc                                        # the tensor-core kernel ran
    return st_tc


def _stripes(n):
    return (n + 127) // 128


def _tiles(n):
    return (n + 63) // 64


@pytest.mark.gpu
@pytest.mark.parametrize("k", [-32, -16, 0, 8, 16, 32, 48])
def test_nn_tables_fpfh_scaled(handles, oracle, k):
    A, B = fam_scaled(np.random.default_rng(100 + k), k)
    st = _both_paths(handles, oracle, A, B, f"fpfh x 2^{k}")
    if k <= -16:   # every centred norm collapses onto |mu|: the filter passes everything and the stripes hand the pair back
        assert st["aborted_stripes"] > 0, st


@pytest.mark.gpu
def test_nn_tables_clustered(handles, oracle):
    A, B = fam_clustered(np.random.default_rng(200))
    st = _both_paths(handles, oracle, A, B, "clustered")
    assert st["aborted_stripes"] > 0 or st["tiles"] < _stripes(len(A)) * _tiles(len(B)) // 2, st   # skipping happened


@pytest.mark.gpu
def test_nn_tables_norm_shell(handles, oracle):
    A, B = fam_shell(np.random.default_rng(300))
    st = _both_paths(handles, oracle, A, B, "norm shell")
    assert st["aborted_stripes"] == 0, st
    assert st["tiles"] == _stripes(len(A)) * _tiles(len(B)), st            # nothing skippable: every tile of every stripe


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [1.0, 256.0, 65536.0])
def test_nn_tables_collinear_near_ties(handles, oracle, scale):
    A, B = fam_collinear(np.random.default_rng(400 + int(np.log2(scale))), scale)
    _both_paths(handles, oracle, A, B, f"collinear x {scale:g}")


@pytest.mark.gpu
def test_nn_tables_wide_column_counts(oracle, monkeypatch):
    """Column counts around the scheduler's 256-tile shared-memory window (16384 columns) and far beyond it."""
    from quatro_b200.capi import Handle
    hs = []
    try:
        hs.append(Handle(max_batch_slots=2, max_voxel_points=40064))
        monkeypatch.setenv("QB200_MATCH_EXACT", "1")
        hs.append(Handle(max_batch_slots=2, max_voxel_points=40064))
        for nb in (16384 - 64, 16384, 16384 + 64, 20000, 40000):
            A, B = fam_wide(np.random.default_rng(500 + nb), nb)
            _both_paths(hs, oracle, A, B, f"{len(A)} x {nb}")
    finally:
        for h in hs:
            h.close()


@pytest.mark.gpu
def test_nn_tables_equal_norm_keys(handles, oracle):
    A, B = fam_equal_keys(np.random.default_rng(600))
    keys = _norm_chain(B)
    _, first = np.unique(keys, return_index=True)
    assert len(first) < len(np.unique(B, axis=0)), "no two different descriptors share a norm key"
    _both_paths(handles, oracle, A, B, "equal norm keys")


@pytest.mark.gpu
def test_nn_tables_ulp_perturbations(handles, oracle):
    A, B = fam_ulp(np.random.default_rng(700))
    assert len(np.unique(B, axis=0)) == len(B)
    st = _both_paths(handles, oracle, A, B, "1-ulp perturbations")
    assert st["aborted_stripes"] > 0, st       # massive near-ties: the stripes hand the pair to the exact kernel


@pytest.mark.gpu
def test_nn_tables_nonfinite_and_overflow(handles, oracle):
    A, B = fam_nonfinite(np.random.default_rng(800))
    _both_paths(handles, oracle, A, B, "NaN / inf / overflow")
    # the pair whose squared norms overflow fp32 is a mutual match at distance 1
    rb, cb = handles[0].debug_nn_tables(len(A), len(B))
    assert _idx(rb[20:21])[0] == 30 and _dist(rb[20:21])[0] == 1.0 and _idx(cb[30:31])[0] == 20
