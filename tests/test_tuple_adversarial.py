"""The matcher's back half (K7: match_mutual_kernel's list, cloud_mean_kernel, tuple_test_kernel, scatter_partner_kernel,
pack_corr_kernel) against tests/independent_ref.py's float32 restatement of feature_matcher.cc:18-76 and :187-264, on scenes built
to sit on the tuple test's edges.

Every scene comes as caller keypoints and descriptors: each matched pair shares one fpfh_like row in both clouds, and unmatched
points, which live in one cloud of a scene only, have rows of their own.  The mutual list is then exactly the twins, so the
coordinates are free to put every trial where it is wanted:

- ratio ties: dyadic triangles with exact means under the dyadic scales 0.5 / 0.75 / 0.875, one side at lj = li*scale and
  lj = li/scale exactly and one ulp either side of each, the other sides comfortably inside;
- odd scales: 0.95 on congruent copies (everything survives), 1, 1.5, -0.5, NaN, +inf, FLT_MIN, a subnormal, 1e-30 on a cloud whose
  li/scale overflows, +-0 (the test off), and a subnormal scale whose decision changes if it were flushed to zero;
- one, two and three pairs, and coincident keypoints (zero-length sides, 0 < 0);
- n_src one below, equal to and one above n_tgt (the larger cloud is fi, the source on ties; the list is in ascending fi order);
- clouds whose mean sits 5e5 and 5e6 m out while the matched points sit near the origin: centring rounds, and the list changes if
  the mean is summed in any order but the reference's (a coordinate within a factor two of its mean centres exactly, so a cloud
  that is far out as a whole does not depend on the mean's bits);
- a NaN and an inf keypoint with a finite descriptor (the call accepts them; the mean is not finite and nothing survives);
- mutual lists of 4095 / 4096 / 4097 pairs around the tuple kernel's shared-memory staging, about 40 000, and 262 000 pairs in
  clouds at the 262 144-point limit, which also leaves more survivors than max_corr (the clip and QB200_CAPACITY_EXCEEDED);
- 0, 1, 7 and 100 trials per correspondence on 37 pairs, so no trial count is a multiple of 32.

On the CPU the constructions are shown to hit their edges (exact margins of 0 and +-1 ulp), the Philox restatement equals the
Random123 known answers and oracle.philox (counters up to 2^64 - 1), and oracle.match equals the restatement on every scene small
enough for its O(n^2) search.  On the GPU qb200_match and qb200_match_features_each equal the restatement bit for bit on every scene,
one mixed wave of every scene equals the single calls through one lane and four, and qb200_register_features_each gives the
restated correspondence count and the oracle's solver record.  Every device call runs at most 26.2 M trials; counters at and above
2^32 would need 4 G trials in one call and cannot be restated in numpy, so they are checked on the CPU only, through Philox."""
import functools
from dataclasses import dataclass, field

import numpy as np
import pytest

from independent_ref import cloud_mean, philox4x32_10, philox4x32_10_words, tuple_decide, tuple_match
from quatro_b200.capi import MATCH_LISTS, MEM_HOST, ListBuffers, default_params
from support import fpfh_like, make_handle

F32 = np.float32
FLT_MIN = float(np.finfo(np.float32).tiny)
SUBNORMAL = float(np.nextafter(F32(FLT_MIN), F32(0)))        # the largest subnormal
V_MAX, CORR_MAX = 262144, 32768                              # the device handle: QB200_MAX_VOXEL_POINTS, QB200_MAX_CORR
CAPACITY_EXCEEDED = 3
ORACLE_MAX = 5000                                            # clouds the oracle's O(n^2) search handles in a second


@dataclass
class Scene:
    name: str
    src: np.ndarray            # n_src x 4 keypoints (w random: the matched copies of a feature wave keep it)
    sdesc: np.ndarray
    tgt: np.ndarray
    tdesc: np.ndarray
    twins: np.ndarray          # the mutual pairs by construction: (source index, target index)
    prm: dict = field(default_factory=dict)

    def params(self):
        p = default_params()
        p.use_tuple_test, p.tuple_scale = self.prm.get("use", 1), self.prm.get("scale", 0.95)
        p.tuple_trials_per_corr, p.seed = self.prm.get("trials", 100), self.prm.get("seed", 0x5EED)
        p.rot_noise_bound = 2 * p.noise_bound
        return p

    @property
    def small(self):
        return max(len(self.src), len(self.tgt)) <= ORACLE_MAX


def make_scene(name, A, B, xs=(), xt=(), rs=0, permute=True, **prm):
    """Matched coordinates A[q] <-> B[q] (twin q) and unmatched points xs (source) or xt (target), both clouds shuffled unless
    permute=False (the twins first).  prm: use, scale, trials, seed of the tuple test."""
    rng = np.random.default_rng(rs)
    A, B = np.asarray(A, F32).reshape(-1, 3), np.asarray(B, F32).reshape(-1, 3)
    xs, xt = np.asarray(xs, F32).reshape(-1, 3), np.asarray(xt, F32).reshape(-1, 3)
    assert len(A) == len(B) and (len(xs) == 0 or len(xt) == 0)
    m = len(A)
    rows = fpfh_like(rng, m + len(xs) + len(xt))

    def cloud(P, X, xrows):
        pts, desc = np.concatenate([P, X]), np.concatenate([rows[:m], xrows])
        perm = rng.permutation(len(pts)) if permute else np.arange(len(pts))
        where = np.empty(len(pts), np.int64)
        where[perm] = np.arange(len(pts))
        out = np.empty((len(pts), 4), F32)
        out[:, :3] = pts[perm]
        out[:, 3] = rng.uniform(-1, 1, len(pts)).astype(F32)
        return out, np.ascontiguousarray(desc[perm]), where[:m]

    src, sdesc, ws = cloud(A, xs, rows[m:m + len(xs)])
    tgt, tdesc, wt = cloud(B, xt, rows[m + len(xs):])
    return Scene(name, src, sdesc, tgt, tdesc, np.stack([ws, wt], 1), prm)


def _line(xs):
    return np.stack([np.asarray(xs, F32), np.zeros(len(xs), F32), np.zeros(len(xs), F32)], 1)


TIE_SCALES = (0.5, 0.75, 0.875)


def _tie_scene(scale, kind, off):
    """Three pairs, (0, 0), (l, 0) and (-l, 48) in both clouds (every sum exact, the mean exactly (0, 16)): side l is on the edge,
    the two sides of about 50 comfortably inside.  The target's l sits at li*scale (kind "lo") or li/scale ("hi"), both exact,
    moved by `off` ulps."""
    s = F32(scale)
    li0 = F32(8) if kind == "lo" else F32(8 * s)
    edge = F32(li0 * s) if kind == "lo" else F32(li0 / s)
    assert (float(edge) == float(li0) * float(s)) if kind == "lo" else (float(edge) * float(s) == float(li0))
    lj0 = edge if off == 0 else np.nextafter(edge, F32(np.inf if off > 0 else -np.inf))
    A, B = _line([0, li0, -li0]), _line([0, lj0, -lj0])
    A[2, 1] = B[2, 1] = 48
    return make_scene(f"tie_{scale}_{kind}_{off:+d}", A, B, rs=7, scale=scale)


def _noisy(m, seed, outliers=0.3):
    """m pairs: a rotated, moved copy with 5 cm noise, `outliers` of the target points re-drawn anywhere (their triangles pass by
    chance, so which of them survive depends on the draws)."""
    rng = np.random.default_rng(seed)
    A = rng.uniform(-30, 30, (m, 3))
    c, s = np.cos(0.7), np.sin(0.7)
    B = A @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T + [5.0, -3.0, 0.5] + rng.normal(0, 0.05, (m, 3))
    out = rng.random(m) < outliers
    B[out] = rng.uniform(-30, 30, (out.sum(), 3))
    return A, B, rng


def _congruent(m, seed, mag=20.0):
    rng = np.random.default_rng(seed)
    A = rng.uniform(-mag, mag, (m, 3)).astype(F32)
    return A, np.stack([-A[:, 1], A[:, 0], A[:, 2]], 1)      # a quarter turn: exact, the same sides


MEAN_VARIANTS = {"reversed": lambda p: cloud_mean(np.asarray(p)[::-1]),
                 "pairwise": lambda p: np.array([np.ascontiguousarray(np.asarray(p, F32)[:, k]).sum(dtype=F32) for k in range(3)]) / F32(len(p)),
                 "float64": lambda p: (np.asarray(p, F32)[:, :3].astype(np.float64).sum(0) / len(p)).astype(F32)}


def _side0(P, mean):
    c = (P[:2, :3] - mean).astype(F32)
    d = c[1] - c[0]
    return F32(np.sqrt(F32(F32(d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])))


def _far_scene(far):
    """A bulk of 2000 unmatched source points `far` m out on x and a matched triangle near the origin whose first two vertices sit
    on half-way ties of the mean's ulp, an even and an odd number of ulps apart: their centred difference depends on the parity of
    the mean's last bit.  The bulk is the first whose reversed, pairwise and float64 means all have the other parity, and the
    target's first side sits between the two possible source sides, so the triangle passes with the reference's mean only."""
    g = float(np.spacing(F32(far)))
    P = np.array([[0.5 * g, 0, 0], [31.5 * g, 0, 0], [0, 8, 0]], F32)
    for rs in range(400):
        rng = np.random.default_rng(rs)
        bulk = np.zeros((2000, 3), F32)
        bulk[:, 0] = (far + rng.uniform(-100, 100, 2000)).astype(F32)
        cloud = np.concatenate([P, bulk])
        true = _side0(P, cloud_mean(cloud))
        alt = {k: _side0(P, fn(cloud)) for k, fn in MEAN_VARIANTS.items()}
        if all(v != true for v in alt.values()):
            break
    else:
        raise AssertionError("no mean-sensitive bulk")
    alt = alt["reversed"]
    lj0 = F32(alt * F32(0.5)) if alt > true else F32(alt * F32(2))   # scale 0.5 passes li/2 < lj < 2 li
    B = _line([0, lj0, -lj0])
    B[2, 1] = 12                                             # the mean (0, 4, 0) is exact
    return make_scene(f"far_{far:g}", P, B, xs=bulk, rs=rs, permute=False, scale=0.5, seed=3)


@functools.lru_cache(maxsize=None)
def scenes():
    out = [_tie_scene(s, kind, off) for s in TIE_SCALES for kind in ("lo", "hi") for off in (-1, 0, 1)]
    A, B = _congruent(64, 1)
    for name, sc in (("0.95", 0.95), ("1", 1.0), ("1.5", 1.5), ("-0.5", -0.5), ("nan", float("nan")), ("inf", float("inf")),
                     ("flt_min", FLT_MIN), ("subnormal", 1e-40), ("1e-30", 1e-30), ("+0", 0.0), ("-0", -0.0)):
        out.append(make_scene(f"scale_{name}", A, B, rs=11, scale=sc, seed=21))
    A, B = _congruent(64, 2, mag=2e9)                        # sides ~1e9: li / 1e-30 overflows to inf
    out.append(make_scene("scale_1e-30_overflow", A, B, rs=12, scale=1e-30))
    # x86 keeps the subnormal scale: side 0 fails (li*s > lj) and nothing survives; flushed to zero, every side would pass
    out.append(make_scene("scale_subnormal_kept", _line([0, 1.7e19, 1.71e19]), _line([0, 1.5e-19, 2.7e-19]), rs=13, scale=SUBNORMAL))
    for m in (1, 2, 3):
        A, B = _congruent(m, 30 + m)
        out.append(make_scene(f"ncorr_{m}", A, B, rs=30 + m))
    A, B = _congruent(12, 40)
    A[:6], B[:6] = A[0], B[0]
    out.append(make_scene("coincident_half", A, B, rs=41))
    out.append(make_scene("coincident_all", np.repeat(A[:1], 12, 0), np.repeat(B[:1], 12, 0), rs=42))
    A, B, rng = _noisy(300, 50)
    extra = rng.uniform(-30, 30, (1, 3))
    out.append(make_scene("swap_src_below", A, B, xt=extra, rs=51, seed=5))
    out.append(make_scene("swap_equal", A, B, rs=52, seed=5))
    out.append(make_scene("swap_src_above", A, B, xs=extra, rs=53, seed=5))
    out += [_far_scene(5e5), _far_scene(5e6)]
    A, B = _congruent(40, 60)
    out.append(make_scene("nan_keypoint", A, B, xs=[[np.nan, 0, 0]], rs=61))
    out.append(make_scene("inf_keypoint", A, B, xs=[[0, np.inf, 0]], rs=62))
    for m in (4095, 4096, 4097, 40000):
        A, B, _ = _noisy(m, m)
        out.append(make_scene(f"size_{m}", A, B, rs=m, seed=m))
    A, B, rng = _noisy(262000, 70)
    out.append(make_scene("size_262000", A, B, xs=rng.uniform(-30, 30, (V_MAX - 262000, 3)), rs=71, trials=10, seed=9))
    A, B, _ = _noisy(37, 80)
    for t in (0, 1, 7, 100):
        out.append(make_scene(f"trials_{t}", A, B, rs=81, trials=t, seed=t))
    return {sc.name: sc for sc in out}


NAMES = list(scenes())
SMALL = [n for n in NAMES if scenes()[n].small]


@functools.lru_cache(maxsize=None)
def restated(name, margins=None):
    sc = scenes()[name]
    p = sc.params()
    margins = sc.small and len(sc.twins) <= 64 if margins is None else margins
    return tuple_match(sc.src, sc.tgt, sc.twins, p.use_tuple_test, p.tuple_scale, p.tuple_trials_per_corr, p.seed, margins=margins)


def _expected(name, max_corr):
    """What the device leaves for a scene: the restated list clipped to max_corr, its count and the pair's status."""
    corr = restated(name)["corr"]
    return corr[:max_corr], min(len(corr), max_corr), CAPACITY_EXCEEDED if len(corr) > max_corr else 0


# ---- CPU: the restatement ------------------------------------------------------------------------------------------------------
def test_philox_restatement_equals_known_answers_and_the_oracle(oracle):
    # Random123 kat_vectors, philox4x32 10 (counter words 2 and 3 in use: the general form), then D1's form (ctr lo, ctr hi, 0, 0)
    kat = [((0, 0, 0, 0, 0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 6, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344, 0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for words, want in kat:
        assert tuple(int(w) for w in philox4x32_10_words(*words)) == want
    assert [int(w) for w in philox4x32_10(0, 0)[:, 0]] == list(kat[0][1])
    ctrs = [0, 1, 2, 31, 32, 33, (1 << 31) - 1, 1 << 31, (1 << 32) - 1, 1 << 32, (1 << 32) + 1, (1 << 40) + 3, (1 << 63), (1 << 64) - 1]
    for seed in (0, 1, 0x5EED, 21, (1 << 32) - 1, 1 << 32, (1 << 32) + 5, (1 << 64) - 1):
        got = philox4x32_10(seed, np.array(ctrs, np.uint64))
        for k, c in enumerate(ctrs):
            assert np.array_equal(got[:, k], oracle.philox(seed, c)), (seed, c)
    big = np.arange((1 << 32) - 2048, (1 << 32) + 2048, dtype=np.uint64)    # the vectorised form across the word boundary
    ref = np.stack([oracle.philox(77, int(c)) for c in big[::97]], 1)
    assert np.array_equal(philox4x32_10(77, big)[:, ::97], ref)


def test_restatement_is_fast_on_twenty_million_trials():
    import time
    sc = scenes()["size_40000"]
    t = time.perf_counter()
    out = tuple_match(sc.src, sc.tgt, sc.twins, 1, 0.95, 500, 1)
    assert time.perf_counter() - t < 60 and 0 < len(out["corr"]) < 40000


def test_mean_is_the_running_sum():
    rng = np.random.default_rng(5)
    p = (5e5 + rng.uniform(-100, 100, (3001, 4))).astype(F32)
    acc = np.zeros(3, F32)
    for q in p[:, :3]:
        acc = (acc + q).astype(F32)
    assert np.array_equal(cloud_mean(p), acc / F32(len(p)))


@pytest.mark.parametrize("scale", TIE_SCALES)
def test_ties_sit_on_their_edges(scale):
    """In every trial with three distinct draws exactly one side sits on the tested edge, at an exact margin of 0 or +-1 ulp of lj;
    every other comparison is comfortably true.  Only lj = li*scale + 1 ulp and lj = li/scale - 1 ulp survive."""
    for kind in ("lo", "hi"):
        for off in (-1, 0, 1):
            name = f"tie_{scale}_{kind}_{off:+d}"
            r = restated(name)
            li, m = r["sides"][:, :3], r["margins"]
            distinct = (li > 0).all(1)
            assert distinct.sum() > 10, name
            edge, other = (m[distinct][:, 0::2], m[distinct][:, 1::2]) if kind == "lo" else (m[distinct][:, 1::2], m[distinct][:, 0::2])
            on_edge = edge == (off if kind == "lo" else -off)
            assert (on_edge.sum(1) == 1).all() and (edge[~on_edge] > 1000).all(), (name, np.unique(edge))
            assert (other > 1000).all(), name
            survives = (kind == "lo" and off == 1) or (kind == "hi" and off == -1)
            assert len(r["corr"]) == (3 if survives else 0), name
            # the degenerate draws (r0 == r1 and the like) have a zero side: 0*scale < 0 is false
            assert (r["sides"][~distinct] == 0).any(1).all() and (~distinct).sum() > 0, name


def test_odd_scales_decide_as_float32_does():
    S = {n: restated(n) for n in NAMES if n.startswith("scale_")}
    assert len(S["scale_0.95"]["corr"]) == 64                  # congruent copies: everything survives
    for n in ("1", "1.5", "-0.5", "nan", "inf"):               # li*s < lj < li/s is empty; NaN passes != 0 and fails every test
        assert "mark" in S[f"scale_{n}"] and len(S[f"scale_{n}"]["corr"]) == 0, n
    for n in ("flt_min", "subnormal", "1e-30", "1e-30_overflow"):
        assert len(S[f"scale_{n}"]["corr"]) == 64, n
    for n in ("+0", "-0"):                                     # tuple_scale == 0: the test is off
        assert "mark" not in S[f"scale_{n}"] and len(S[f"scale_{n}"]["corr"]) == 64, n
    li = S["scale_1e-30_overflow"]["sides"][:, :3]
    with np.errstate(over="ignore"):
        assert np.isinf(li[li > 0] / F32(1e-30)).mean() > 0.9  # li / scale overflows to +inf, and lj < inf holds
    assert np.isfinite(S["scale_1e-30"]["sides"][:, :3] / F32(1e-30)).all()
    # the largest subnormal scale: side 0 fails on x86 (li*s = 2.0e-19 > lj = 1.5e-19); flushed to zero, every side would pass
    r = restated("scale_subnormal_kept")
    assert len(r["corr"]) == 0
    L = r["sides"][(r["sides"][:, :3] > 0).all(1)]
    assert len(L) > 0 and (np.asarray(tuple_decide(L[:, :3], L[:, 3:], 0.0)).all())
    assert not np.asarray(tuple_decide(L[:, :3], L[:, 3:], SUBNORMAL)).all(0).all(1).any()
    assert np.isfinite(L).all() and (L[:, 3:] ** 2 >= FLT_MIN).all()     # the target's squares are normal: no underflow involved


def test_small_lists_and_coincident_points():
    for m in (1, 2):                                           # every trial repeats a draw: a zero side, nothing survives
        assert len(restated(f"ncorr_{m}")["corr"]) == 0
    assert len(restated("ncorr_3")["corr"]) == 3
    r = restated("coincident_half")
    assert (r["sides"][:, :3] == 0).any() and len(r["corr"]) == 12
    assert len(restated("coincident_all")["corr"]) == 0


def test_swaps_far_clouds_nonfinite_points_sizes_and_trials_reach_their_cases():
    assert [restated(n)["swapped"] for n in ("swap_src_below", "swap_equal", "swap_src_above")] == [True, False, False]
    for n in ("swap_src_below", "swap_equal", "swap_src_above"):
        assert 0.5 * 300 < len(restated(n)["corr"]) < 300, n   # some pairs survive and others do not: the draws decide
    for n in ("nan_keypoint", "inf_keypoint"):
        assert "mark" in restated(n) and len(restated(n)["corr"]) == 0, n
    assert [restated(f"size_{m}")["n_mutual"] for m in (4095, 4096, 4097, 40000, 262000)] == [4095, 4096, 4097, 40000, 262000]
    assert len(scenes()["size_262000"].src) == V_MAX
    assert len(restated("size_262000")["corr"]) > CORR_MAX and len(restated("size_40000")["corr"]) > CORR_MAX    # the clip
    assert len(restated("size_4097")["corr"]) < CORR_MAX
    for t in (1, 7, 100):
        assert (37 * t) % 32 != 0
    counts = [len(restated(f"trials_{t}")["corr"]) for t in (0, 1, 7, 100)]
    assert counts[0] == 0 and 0 < counts[1] < counts[2] <= counts[3] < 37, counts


@pytest.mark.parametrize("far", ["far_500000", "far_5e+06"])
def test_far_cloud_lists_depend_on_the_summation_order(far):
    sc = scenes()[far]
    p = sc.params()
    assert len(restated(far)["corr"]) == 3 and abs(cloud_mean(sc.src)[0]) > 0.99 * float(far[4:])
    for k, fn in MEAN_VARIANTS.items():
        assert not np.array_equal(fn(sc.src), cloud_mean(sc.src)), k
        other = tuple_match(sc.src, sc.tgt, sc.twins, 1, p.tuple_scale, p.tuple_trials_per_corr, p.seed, mean=fn)
        assert len(other["corr"]) == 0, k


# ---- CPU: the oracle against the restatement -------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SMALL)
def test_oracle_equals_restatement(oracle, name):
    sc = scenes()[name]
    r = restated(name)
    p = sc.params()
    corr, nm, st, mutual = oracle.match(sc.src, sc.sdesc, sc.tgt, sc.tdesc, p, cap=max(1, len(sc.twins)), want_mutual=True)
    assert st == 0 and nm == r["n_mutual"] == len(sc.twins)
    assert np.array_equal(mutual, r["mutual"]), "mutual list (larger cloud first, ascending) or the swap differs"
    assert np.array_equal(corr, r["corr"]), (len(corr), len(r["corr"]))
    p.use_tuple_test = 0                                        # the mutual list is exactly the twins
    corr, nm, st = oracle.match(sc.src, sc.sdesc, sc.tgt, sc.tdesc, p, cap=max(1, len(sc.twins)))
    assert np.array_equal(corr, sc.twins[np.lexsort((sc.twins[:, 1], sc.twins[:, 0]))])


def test_oracle_clips_at_its_capacity(oracle):
    sc = scenes()["swap_equal"]
    corr, nm, st = oracle.match(sc.src, sc.sdesc, sc.tgt, sc.tdesc, sc.params(), cap=64)
    assert st == CAPACITY_EXCEEDED and np.array_equal(corr, restated("swap_equal")["corr"][:64])


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def h1():
    h = make_handle(1, max_batch_slots=4, max_voxel_points=V_MAX, max_corr=CORR_MAX)
    yield h
    h.close()


def _feature_call(h, names, fn="match_features_each"):
    lb = ListBuffers(len(names), CORR_MAX, MEM_HOST, MATCH_LISTS)
    feats = [(scenes()[n].src, scenes()[n].sdesc, scenes()[n].tgt, scenes()[n].tdesc) for n in names]
    recs, lists = getattr(h, fn)(feats, [scenes()[n].params() for n in names], buffers=lb)
    return recs, lists


@pytest.fixture(scope="module")
def singles(h1):
    """every scene through qb200_match_features_each on its own"""
    return {n: _feature_call(h1, [n]) for n in NAMES}


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_device_matchers_equal_restatement(h1, singles, name):
    sc = scenes()[name]
    corr, n_corr, status = _expected(name, CORR_MAX)
    got, nm, st = h1.match(sc.src, sc.sdesc, sc.tgt, sc.tdesc, sc.params(), cap=CORR_MAX)
    assert (st, nm) == (status, len(sc.twins)) and np.array_equal(got, corr), (st, nm, len(got), len(corr))
    recs, lists = singles[name]
    rec, lst = recs[0], lists[0]
    assert (rec["status"], rec["n_mutual"], rec["n_corr"]) == (status, len(sc.twins), n_corr)
    if status == CAPACITY_EXCEEDED:                            # the single-pair call hands out the clipped list, a batch call none
        corr = corr[:0]
    assert np.array_equal(lst["corr"], corr)
    assert lst["src_matched4"].tobytes() == sc.src[corr[:, 0]].tobytes()          # keypoints verbatim, w kept
    assert lst["tgt_matched4"].tobytes() == sc.tgt[corr[:, 1]].tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 4])
def test_mixed_wave_equals_single_calls(h1, singles, lanes):
    h = h1 if lanes == 1 else make_handle(4, max_batch_slots=4, max_voxel_points=V_MAX, max_corr=CORR_MAX)
    try:
        order = NAMES[::-1] if lanes == 4 else NAMES
        recs, lists = _feature_call(h, order)
    finally:
        if h is not h1:
            h.close()
    for k, n in enumerate(order):
        srec, slist = singles[n]
        assert recs[k].tobytes() == srec[0].tobytes(), n
        for key in MATCH_LISTS:
            assert np.asarray(lists[k][key]).tobytes() == np.asarray(slist[0][key]).tobytes(), (n, key)


@pytest.mark.gpu
def test_register_features_gives_restated_count_and_oracle_record(h1, oracle):
    names = ["scale_0.95", "tie_0.75_lo_+1", "ncorr_3", "swap_src_below", "swap_src_above", "trials_7", "far_500000", "nan_keypoint"]
    recs, lists = _feature_call(h1, names, "register_features_each")
    for k, n in enumerate(names):
        sc = scenes()[n]
        corr = restated(n)["corr"]
        assert recs[k]["n_corr"] == len(corr) and recs[k]["n_mutual"] == len(sc.twins), n
        assert np.array_equal(lists[k]["corr"], corr), n
        ref, st = oracle.solve_correspondences(sc.src[corr[:, 0]], sc.tgt[corr[:, 1]], sc.params())
        for key in ("valid", "status", "n_corr", "n_edges", "max_core", "clique_size", "gnc_iters", "n_rot_inliers", "n_final_inliers"):
            assert recs[k][key] == getattr(ref, key), (n, key, recs[k][key], getattr(ref, key))
        assert np.allclose(np.asarray(recs[k]["T"]).reshape(4, 4).T, ref.matrix(), atol=1e-9, rtol=0), n
