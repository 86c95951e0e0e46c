"""Normals, SPFH and FPFH-33 against a float32 restatement of PCL 1.8.1's NormalEstimation and FPFHEstimation over FLANN's radius search
(tests/independent_ref.py, written from the PCL and FLANN texts, not from the oracle or the kernels), on neighbourhoods built to sit on
the stage's float decisions: neighbours at d2 = r2 and one ulp either side, points whose d2 falls on different sides of r2 under the
other association, a neighbour on the normal radius inside the FPFH radius, normal_radius == fpfh_radius, a query on lattice cell
faces with a cell of r / 2 and r / 5, |c0| at FLT_EPSILON and one ulp either side, planar patches of thickness 0 ... 1e-3, isotropic
sets that reach the a_over_3 and q clamps, tight patches 1 ... 40 km out whose single-pass covariance is not PSD (roots[0] <= 0),
collinear sets, covariances below FLT_MIN, planes through the viewpoint (cos_theta = 0), facing planes (f1 near +-pi), k = 1, 2, 3,
coincident duplicates, d2 = FLT_MIN and a subnormal d2 whose weight is infinite, a descriptor whose thirds sum to 0, and 80 / 81
neighbours on either side of the neighbour list.  The Darboux edges that need exact operands (|a1| == |a2|, equal acos of different
|a|, dp parallel to n1, NaN normals, f1 = +-pi, every bin edge +-1 ulp) are checked pair by pair.

With D7's polynomials the restatement must equal the oracle bit for bit (neighbour sets and order, normals with their NaN pattern,
SPFH rows, descriptors); the device must equal both.  With float64 transcendentals (the plain reading of PCL) every discrete output must
agree wherever each decision's margin clears the error a 3-ulp change in a transcendental can cause, and in both readings the normal
must lie within 128 u ||C|| / (l1 - l0) of the exact eigenvector of the float32 covariance that was formed."""
import ctypes as C
import functools

import numpy as np
import pytest

import independent_ref as R
from independent_ref import F32, F64, FLT_EPSILON, FLT_MIN, radius_sq
from quatro_b200.capi import _ptr
from support import P4, make_handle, make_params, same_bits


# ---- constructions ------------------------------------------------------------------------------------------------------------------
def _flann_d2(c, cand):
    d = (np.asarray(c, F32) - np.asarray(cand, F32)).astype(F32)
    return ((F32(0) + d[..., 0] * d[..., 0]) + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _sphere(rng, n):
    u = rng.normal(size=(n, 3))
    return u / np.linalg.norm(u, axis=1, keepdims=True)


def rim_points(c, r, rng, n_try=200000):
    """Points whose flann d2 from c is exactly r2 - 1 ulp, r2, r2 + 1 ulp and float(r * r) of the double radius (one ulp below r2 for
    r = 0.1 and 1/3), and two points whose d2 lies on different sides of r2 under ((dx2 + dy2) + dz2) and (dx2 + (dy2 + dz2))."""
    c = np.asarray(c, F32)
    r2 = radius_sq(F32(r))
    targets = [np.nextafter(r2, F32(0)), r2, np.nextafter(r2, F32(1)), F32(float(r) * float(r))]
    out = []
    for t in targets:
        cand = (c.astype(F64) + np.sqrt(F64(t)) * _sphere(rng, n_try)).astype(F32)
        hit = np.flatnonzero(_flann_d2(c, cand) == t)
        out.append(cand[hit[0]])
    cand = (c.astype(F64) + np.sqrt(F64(r2)) * _sphere(rng, n_try)).astype(F32)
    d = (c - cand).astype(F32)
    sq = d * d
    left, right = (sq[:, 0] + sq[:, 1]) + sq[:, 2], sq[:, 0] + (sq[:, 1] + sq[:, 2])
    out.append(cand[np.flatnonzero((left < r2) & (right >= r2))[0]])
    out.append(cand[np.flatnonzero((right < r2) & (left >= r2))[0]])
    return np.array(out, F32)


def on_faces(c, cell):
    """c moved to the nearest point whose coordinates times (1 / cell) are exact integers: the query sits on three cell faces."""
    inv = F32(1) / F32(cell)
    out = []
    for x in np.asarray(c, F32):
        k = F32(np.round(x * inv))
        v = F32(k / inv)
        for _ in range(64):
            if F32(v * inv) == k:
                break
            v = np.nextafter(v, F32(np.inf))
        assert F32(v * inv) == k
        out.append(v)
    return np.array(out, F32)


def rim_cloud(r_n, r_f, seed, centre=(1.5, -0.75, 0.25), k_f=None, cell=None):
    """A query with a few inner neighbours (or exactly k_f FPFH neighbours) and rim points on both radii; with a cell, the query sits
    on cell faces and two axis neighbours just inside r_f lie on the far cell faces of the reach."""
    rng = np.random.default_rng(seed)
    c = np.asarray(centre, F32) if cell is None else on_faces(centre, cell)
    inner = (c.astype(F64) + _sphere(rng, 6) * rng.uniform(0.1, 0.5, (6, 1)) * r_n).astype(F32)
    rims = [rim_points(c, r_f, rng)] + ([rim_points(c, r_n, rng)] if r_n != r_f else [])
    pts = [c[None], inner] + rims
    if cell is not None:
        r2 = radius_sq(F32(r_f))
        for sgn in (1, -1):
            x = F32(c[0] + F32(sgn * r_f))
            while _flann_d2(c, [x, c[1], c[2]]) >= r2:
                x = np.nextafter(x, c[0])
            pts.append(np.array([[x, c[1], c[2]]], F32))
    pts = np.concatenate(pts)
    if k_f is not None:                                  # fill the inside until the query has exactly k_f FPFH neighbours
        have = int((_flann_d2(c, pts) < radius_sq(F32(r_f))).sum())
        fill = (c.astype(F64) + _sphere(rng, k_f - have) * rng.uniform(0.2, 0.9, (k_f - have, 1)) * r_f).astype(F32)
        pts = np.concatenate([pts, fill])
    return P4(pts)


def plane_patch(t, seed, n=40, centre=(3.0, 2.0, 1.0)):
    """n points in a 0.45 m disc of a tilted plane, displaced along its normal by t * N(0, 1)."""
    rng = np.random.default_rng(seed)
    nrm = np.array([0.3, -0.2, 1.0]) / np.linalg.norm([0.3, -0.2, 1.0])
    a = np.cross(nrm, [1.0, 0.0, 0.0])
    a /= np.linalg.norm(a)
    b = np.cross(nrm, a)
    uv = rng.uniform(-0.3, 0.3, (n, 2))
    return P4(np.asarray(centre) + uv[:, :1] * a + uv[:, 1:] * b + t * rng.normal(size=(n, 1)) * nrm)


def c0_cloud(step):
    """Seven points {0, +-0.25 e_x, +-b e_y, +-z e_z} (b <= 0.25): the covariance is exactly diagonal with m00 = 1 after scaling, so
    c0 = m11 * m22; b and z are chosen so that c0 = FLT_EPSILON moved by `step` ulps.  Every point sees all seven, so every normal takes
    the same branch."""
    want = F32(FLT_EPSILON)
    for _ in range(abs(step)):
        want = np.nextafter(want, F32(np.inf) if step > 0 else F32(0))
    for b in np.arange(32, 16, -1) / 128:
        z0 = F32(0.25 * np.sqrt(float(FLT_EPSILON)) * 0.25 / b)
        for z in (z0.view(np.int32) + np.arange(-60, 60)).astype(np.int32).view(F32):
            pts = P4([[0, 0, 0], [0.25, 0, 0], [-0.25, 0, 0], [0, b, 0], [0, -b, 0], [0, 0, z], [0, 0, -z]])
            _, rec = R.normal_pcl32(pts[:, :3], pts[0, :3], R.D7_MATH)
            if rec["c0"] == want:
                return pts
    raise AssertionError(f"no (b, z) gives c0 = {want}")


def icosahedron(s):
    g = (1 + 5 ** 0.5) / 2
    v = [(0, a, b * g) for a in (-1, 1) for b in (-1, 1)]
    v = v + [(a, b * g, 0) for a in (-1, 1) for b in (-1, 1)] + [(b * g, 0, a) for a in (-1, 1) for b in (-1, 1)]
    return np.array([[0, 0, 0]] + v) * s


def isotropic(kind, shift=(0.0, 0.0, 0.0)):
    if kind == "cube":
        p = np.array([[0, 0, 0]] + [[a, b, c] for a in (-1, 1) for b in (-1, 1) for c in (-1, 1)]) * 0.2
    elif kind == "octahedron":
        p = np.array([[0, 0, 0]] + [list(s * e) for e in np.eye(3) for s in (-1, 1)]) * 0.25
    else:
        p = icosahedron(0.12)
    return P4(p + np.asarray(shift))


def clamp_cloud():
    """An octahedron whose arms differ by a few 2^-22: the exact a_over_3 is a hair below 0, the float32 one rounds above it (both
    clamps of computeRoots then fire: q = half_b^2 > 0)."""
    for i in range(1, 40):
        for j in range(0, 40):
            a, b = 0.25 * (1 + i * 2.0 ** -22), 0.25 * (1 + j * 2.0 ** -22)
            pts = P4([[0, 0, 0], [0.25, 0, 0], [-0.25, 0, 0], [0, a, 0], [0, -a, 0], [0, 0, b], [0, 0, -b]])
            _, rec = R.normal_pcl32(pts[:, :3], pts[0, :3], R.D7_MATH)
            if rec.get("a_over_3", -1) > 0 and rec.get("q", -1) > 0:
                return pts
    raise AssertionError("no octahedron reaches the a_over_3 clamp")


def far_patch(offset, seed, n=30):
    """A tight patch (0.15 m, 1 cm thick) far from the origin: the single-pass covariance is dominated by |p|^2 / n rounding."""
    rng = np.random.default_rng(seed)
    return P4(np.asarray(offset) + rng.uniform(-0.15, 0.15, (n, 3)) * [1.0, 1.0, 0.07])


def flip_planes(seed):
    """Planes through the viewpoint (the origin): z = 0 exactly (normal (0, 0, +-1), cos_theta = +-0.0) and tilted planes
    z = a x + b y with dyadic slopes, whose cos_theta is a rounding residue of either sign."""
    rng = np.random.default_rng(seed)
    out = []
    for a, b, x0, y0 in ((0.0, 0.0, 2.0, 0.5), (0.0, 0.0, -2.0, -4.0), (0.0, 0.0, 6.0, -6.0), (0.0, 0.0, -6.0, 6.0),
                         (0.5, 0.25, 4.0, 3.0), (-0.375, 0.125, -3.0, 2.0), (0.25, -0.75, 8.0, 0.0), (1.25, 0.5, -8.0, -1.0)):
        xy = np.round(rng.uniform(-0.25, 0.25, (12, 2)) * 64) / 64 + [x0, y0]
        out.append(np.column_stack([xy, a * xy[:, 0] + b * xy[:, 1]]))
    return P4(np.concatenate(out))


def tiny_cloud():
    """Coordinates 1e-20 apart around the origin: covariance entries far below FLT_MIN (subnormal or 0, scale reset to 1), d2 subnormal
    and 1 / d2 = inf."""
    k = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [2, 1, 1], [-1, 2, 0]], F64)
    return P4(k * 1e-20)


def flt_min_cloud():
    """d2 = FLT_MIN exactly (offsets of 2^-63 along one axis), a subnormal d2 (2^-70: 1 / d2 = inf), and a plain neighbour."""
    h, s = 2.0 ** -63, 2.0 ** -70
    return P4([[0, 0, 0], [h, 0, 0], [0, h, 0], [0, 0, s], [h, h, 0], [0.1, 0.0, 0.05]])


def small_k_cloud():
    """k = 1 (an isolated point), k = 2 (a pair) and k = 3 (a triple), far apart; a plane patch with three coincident copies of one
    point; three coincident points alone (every pair skipped: zero SPFH rows, descriptor thirds summing to 0)."""
    iso = [[10.0, 10.0, 0.0]]
    pair = [[-10.0, 10.0, 0.0], [-10.0, 10.25, 0.0]]
    triple = [[10.0, -10.0, 0.0], [10.25, -10.0, 0.0], [10.0, -10.25, 0.125]]
    patch = plane_patch(0.01, 5, n=20, centre=(-10.0, -10.0, 0.5))[:, :3]
    dup = np.concatenate([patch, patch[[3, 3, 3]]])
    alone = [[0.0, 20.0, 1.0]] * 3
    return P4(np.concatenate([iso, pair, triple, dup, alone]))


def facing_planes():
    """Two parallel patches 0.375 m apart on either side of z = 0, seen from the origin: their normals point at each other,
    so the cross pairs have n2 = -n1 (f1 near +-pi); normal_radius 0.25 keeps each normal on its own patch."""
    g = np.array([[x, y] for x in np.arange(-2, 3) * 0.0625 for y in np.arange(-2, 3) * 0.0625]) + [2.0, 2.0]
    lo = np.column_stack([g, np.full(len(g), -0.1875)])
    hi = np.column_stack([g, np.full(len(g), 0.1875)])
    return P4(np.concatenate([lo, hi]))


@functools.lru_cache(maxsize=1)
def constructions():
    """(name, points, normal_radius, fpfh_radius, grid_cell or 0 for the default (1 + 2^-9) * fpfh_radius)."""
    C = []
    for r in (0.5, 0.3, 0.1, 1 / 3):
        C.append((f"rim_{r:.3g}", rim_cloud(F32(r) * F32(2 / 3), r, 10 + len(C)), float(F32(r) * F32(2 / 3)), r, 0.0))
    C.append(("rim_0.75_equal_radii", rim_cloud(0.75, 0.75, 20), 0.75, 0.75, 0.0))
    C.append(("rim_0.3_cell_r/2_faces", rim_cloud(0.2, 0.3, 21, cell=0.15), 0.2, 0.3, 0.15))
    C.append(("rim_0.5_cell_r/5_faces", rim_cloud(0.5, 0.5, 22, cell=0.1), 0.5, 0.5, 0.1))
    for k in (80, 81):
        C.append((f"rim_0.3_k{k}", rim_cloud(0.2, 0.3, 23, k_f=k), 0.2, 0.3, 0.0))
    for t in (0.0, 1e-7, 1e-5, 1e-3):
        C.append((f"plane_t{t:g}", plane_patch(t, 30), 0.5, 0.75, 0.0))
    for step in (-1, 0, 1):
        C.append((f"c0_eps{step:+d}", c0_cloud(step), 0.75, 0.75, 0.0))
    for kind in ("cube", "octahedron", "icosahedron"):
        C.append((f"iso_{kind}", isotropic(kind), 0.5, 0.75, 0.0))
        C.append((f"iso_{kind}_shifted", isotropic(kind, (3.0, -2.0, 1.0)), 0.5, 0.75, 0.0))
    C.append(("iso_clamps", clamp_cloud(), 0.5, 0.75, 0.0))
    for off in ((1000.0, 0.0, 0.0), (5000.0, 3000.0, 10.0), (40000.0, 0.0, 0.0), (0.0, 28000.0, 300.0)):
        C.append((f"far_{off[0]:g}_{off[1]:g}", far_patch(off, int(off[0] + off[1])), 0.5, 0.75, 0.0))
    C.append(("collinear", P4(np.column_stack([np.arange(12) * 0.05 + 2.0, np.full(12, 1.0), np.full(12, 0.5)])), 0.5, 0.75, 0.0))
    C.append(("collinear_diagonal", P4(np.arange(10)[:, None] * np.array([0.04, 0.03, 0.02]) + [1.0, -1.0, 0.25]), 0.5, 0.75, 0.0))
    C.append(("below_flt_min", tiny_cloud(), 0.5, 0.75, 0.0))
    C.append(("d2_flt_min_and_subnormal", flt_min_cloud(), 0.5, 0.75, 0.0))
    C.append(("planes_through_viewpoint", flip_planes(40), 0.5, 0.75, 0.0))
    C.append(("small_k_and_duplicates", small_k_cloud(), 0.5, 0.75, 0.0))
    C.append(("facing_planes", facing_planes(), 0.25, 0.75, 0.0))
    return C


def resolved_cell(rn, rf, cell):
    return float(cell) if cell > 0 else float(F32(rf) * R.CELL_FACTOR)


@pytest.fixture(scope="module")
def cons():
    return constructions()


@pytest.fixture(scope="module")
def restated(cons):
    """per construction: (D7 reading, float64 reading)"""
    return {name: (R.fpfh_pcl32(p, rn, rf, cell or None, R.D7_MATH), R.fpfh_pcl32(p, rn, rf, cell or None, R.F64_MATH))
            for name, p, rn, rf, cell in cons}


# ---- pair constructions: exact operands for the Darboux decisions --------------------------------------------------------------------
def _edges(lo, hi, n_bins, scale):
    """float32 values nearest to each inner bin edge of [lo, hi] and one ulp either side"""
    out = []
    for k in range(1, n_bins):
        e = F32(lo + (hi - lo) * k / n_bins)
        out += [np.nextafter(e, F32(-np.inf)), e, np.nextafter(e, F32(np.inf))]
    return out


def pair_cases():
    """(label, p1, n1, p2, n2) float32 4-tuples of 3-vectors."""
    cases = []
    dp = np.array([1, 0, 0], F32)
    z = np.zeros(3, F32)
    h = F32(np.sqrt(F32(0.75)))
    n1 = np.array([0.5, 0, h], F32)                                        # a1 = 0.5 exactly, the frame below is exact
    cases.append(("|a1| == |a2|", z, n1, dp, np.array([-0.5, 0.6, 0.6], F32)))
    cases.append(("|a1| == |a2| swapped roles", z, np.array([-0.5, 0.6, 0.6], F32), dp, n1))
    cases.append(("equal acos of different |a|", z, np.array([1e-9, 0, 1], F32), dp, np.array([2e-9, 1, 0], F32)))
    cases.append(("equal acos, other order", z, np.array([2e-9, 1, 0], F32), dp, np.array([1e-9, 0, 1], F32)))
    cases.append(("dp parallel to n1", z, np.array([1, 0, 0], F32), dp, np.array([0, 1, 0], F32)))
    cases.append(("dp parallel to n2 (swapped)", z, np.array([0, 1, 0], F32), dp, np.array([-1, 0, 0], F32)))
    cases.append(("coincident", z, n1, z, n1))
    cases.append(("NaN n1", z, np.array([np.nan, 0, 1], F32), dp, np.array([0, 1, 0], F32)))
    cases.append(("NaN n2", z, n1, dp, np.array([0, np.nan, 1], F32)))
    # w = (h, 0, -0.5): w . n2 = h (x + 0.25) is a tiny positive / negative, n1 . n2 = -0.5, |a2| = |x| < |a1| (no swap)
    cases.append(("f1 = +pi", z, n1, dp, np.array([F32(-0.25) + F32(2.0 ** -25), 0.8, -h * F32(0.5)], F32)))
    cases.append(("f1 = -pi", z, n1, dp, np.array([F32(-0.25) - F32(2.0 ** -25), 0.8, -h * F32(0.5)], F32)))
    cases.append(("f1 = pi from +0", z, n1, dp, -n1))
    # f3 = a1 = t exactly (no swap: a2 = 0), f2 = t exactly with n1 = e_z, n2 = (0, -t, sqrt(1 - t^2)) (a1 = a2 = 0, no swap)
    for t in [F32(-1), F32(1)] + _edges(-1.0, 1.0, 11, 1):
        s = F32(np.sqrt(max(0.0, 1 - float(t) ** 2)))
        cases.append((f"f3 = {t!r}", z, np.array([t, s, 0], F32), dp, np.array([0, 0, 1], F32)))
        cases.append((f"f2 = {t!r}", z, np.array([0, 0, 1], F32), dp, np.array([0, -t, s], F32)))
    # f1 at the inner edges of [-pi, pi] +-1 ulp: search n2 in the exact frame of n1 = (0.5, 0, h), dp = e_x
    rng = np.random.default_rng(5)
    d_pi = R.D_PI
    for k in range(1, 11):
        ang = -np.pi + 2 * np.pi * k / 11
        cand = np.zeros((400000, 3), F32)
        jit = rng.uniform(-3e-6, 3e-6, (400000, 2))
        w = np.array([h, 0, -0.5], F64)
        u = np.array([0.5, 0, h], F64)
        rho = 0.3 + jit[:, 1:] * 1e4                              # |a2| <= rho < |a1| = 0.5: no swap; f1 ignores the e_y part
        cand[:] = (rho * (np.cos(ang + jit[:, :1]) * u + np.sin(ang + jit[:, :1]) * w) + np.sqrt(1 - rho ** 2) * np.array([0, 1, 0])).astype(F32)
        cand = cand[np.abs(cand[:, 0]) < 0.45]
        pf = R.pair_features_pcl32(np.zeros_like(cand), np.broadcast_to(n1, cand.shape), np.broadcast_to(dp, cand.shape), cand, R.D7_MATH)
        sc = 11 * ((pf["f1"].astype(F64) + np.pi) * F64(d_pi))
        sel = pf["ok"] & ~pf["swap"]
        f1 = pf["f1"]
        below = f1[sel & (sc < k)].max()                           # f1 values: the last below the edge, the first at or above, the next
        at = f1[sel & (sc >= k)].min()
        above = f1[sel & (f1 > at)].min()
        for side, val in ((-1, below), (0, at), (1, above)):
            i = np.flatnonzero(sel & (f1 == val))[0]
            cases.append((f"f1 edge {k} {side:+d}", z, n1, dp, cand[i]))
    return cases


def _pair_arrays(cases):
    return [np.array([c[i] for c in cases], F32) for i in (1, 2, 3, 4)]


@pytest.fixture(scope="module")
def oracle_bins(oracle):
    L = oracle.lib
    L.qo_test_feature_bins.argtypes = [C.c_float, C.c_float, C.c_float, C.c_void_p]

    def bins(f1, f2, f3):
        b = np.zeros(3, np.int32)
        L.qo_test_feature_bins(float(f1), float(f2), float(f3), _ptr(b))
        return b
    return bins


# ---- CPU: every construction reaches its edge ------------------------------------------------------------------------------------------
def test_constructions_hit_their_edges(cons, restated):
    ref = {name: restated[name][0] for name, *_ in cons}
    pts = {name: p for name, p, *_ in cons}
    radii = {name: (rn, rf, cell) for name, _, rn, rf, cell in cons}
    # radius boundary: the query (point 0) sees r2 - 1 ulp and the split-association point, not r2, r2 + 1 ulp or the other split point
    for name in [n for n in ref if n.startswith("rim_") and "_k8" not in n]:
        rn, rf, cell = radii[name]
        p = pts[name][:, :3]
        d2 = _flann_d2(p[0], p)
        for r, nb in ((rf, ref[name]["nbr_f"][0]), (rn, ref[name]["nbr_n"][0])):
            r2 = radius_sq(F32(r))
            assert (d2 == np.nextafter(r2, F32(0))).any() and (d2 == r2).any() and (d2 == np.nextafter(r2, F32(1))).any(), (name, r)
            inside = set(nb.tolist())
            assert all((i in inside) == (d2[i] < r2) for i in range(len(p))), name
        assert len(ref[name]["nbr_n"][0]) < len(ref[name]["nbr_f"][0]) or rn == rf
    for r in (0.1, 1 / 3):                                                 # D19: the double radius's float square is one ulp below
        assert radius_sq(r) == np.nextafter(radius_sq(F32(r)), F32(0))
    for name in ("rim_0.3_cell_r/2_faces", "rim_0.5_cell_r/5_faces"):
        rn, rf, cell = radii[name]
        c = pts[name][0, :3] * (F32(1) / F32(cell))
        assert (c == np.floor(c)).all(), name                                # the query sits on three cell faces
        assert int(np.ceil(F32(rf) * (F32(1) / F32(cell)) + F32(1e-3))) >= 2
    for k in (80, 81):
        assert len(ref[f"rim_0.3_k{k}"]["nbr_f"][0]) == k
    # eigen33: the c0 knife edge on both sides, both clamps, roots[0] <= 0, the scale reset, ties among l1 l2 l3
    for step, branch in ((-1, "roots2"), (0, "cubic"), (1, "cubic")):
        recs = ref[f"c0_eps{step:+d}"]["nrec"]
        assert all(r["branch"] == branch for r in recs), step
    assert ref["c0_eps+0"]["nrec"][0]["c0"] == FLT_EPSILON
    recs = [r for v in ref.values() for r in v["nrec"]]
    assert any(r.get("a_over_3", -1) > 0 for r in recs)
    assert any(r.get("q", -1) > 0 for r in recs)
    assert any(r.get("roots0_nonpositive") for r in recs)
    assert any(r.get("scale_reset") for r in recs if r["k"] >= 3)
    assert any(r["branch"] != "few" and len(set(float(x) for x in r["l"])) < 3 for r in recs)
    far = [r for n, v in ref.items() if n.startswith("far_") for r in v["nrec"] if "cov" in r]
    assert any((np.diag(r["cov"]) < 0).any() for r in far)                   # single-pass cancellation: a negative variance
    assert any(np.linalg.eigvalsh(r["cov"].astype(F64))[0] < 0 for r in far)
    for t in ("plane_t0", "plane_t1e-07", "plane_t1e-05", "plane_t0.001"):
        assert np.isfinite(ref[t]["normals"][:, :3]).all(), t
    # an axis-parallel line: the covariance is exactly rank one, so c0 = c1 = 0, computeRoots2 gives roots (0, 0, c2), every row cross
    # product of the shifted matrix is 0 and the normal is 0 / 0
    col = [r for r in ref["collinear"]["nrec"] if r["k"] >= 3]
    assert col and all(r["c0"] == 0 and r["c1"] == 0 and r["branch"] == "roots2" and r["roots"][0] == 0 and r["roots"][1] == 0 and
                       r["roots"][2] > 0 for r in col)
    rows = [i for i, r in enumerate(ref["collinear"]["nrec"]) if r["k"] >= 3]
    assert np.isnan(ref["collinear"]["normals"][rows, :3]).all() and (ref["collinear"]["normals"][rows, 3] == 0).all()
    # the flip on its knife edge: cos_theta = 0 exactly (the plane z = 0), and rounding residues of both signs (tilted planes)
    cos = np.array([r["cos_theta"] for r in ref["planes_through_viewpoint"]["nrec"] + ref["c0_eps+0"]["nrec"] if "cos_theta" in r], F32)
    assert (cos == 0).sum() >= 40
    tiny = cos[(cos != 0) & (np.abs(cos) < 2e-3)]
    assert (tiny > 0).any() and (tiny < 0).any()
    # SPFH / FPFH: k = 1, 2, 3, duplicates counted in k but skipped, zero rows, zero-sum thirds, d2 = FLT_MIN, infinite weights
    sk = ref["small_k_and_duplicates"]
    ks = {len(nb) for nb in sk["nbr_f"]}
    assert {1, 2, 3} <= ks
    zero_rows = np.flatnonzero((sk["spfh"] == 0).all(1) & np.array([len(nb) >= 2 for nb in sk["nbr_f"]]))
    assert len(zero_rows) >= 3 and (sk["desc"][zero_rows] == 0).all()
    d2 = np.concatenate(ref["d2_flt_min_and_subnormal"]["d2_f"])
    with np.errstate(over="ignore"):
        assert (d2 == FLT_MIN).any() and ((d2 > 0) & (d2 < FLT_MIN) & (F32(1) / np.where(d2 > 0, d2, 1) == np.inf)).any()
    assert np.isnan(ref["d2_flt_min_and_subnormal"]["desc"]).any()
    fp = ref["facing_planes"]
    f1 = np.concatenate([pf["f1"][pf["ok"]] for pf in fp["pairs"]])
    assert (np.abs(np.abs(f1) - np.pi) < 1e-3).any()


def test_double_radius_deviation(cons, restated):
    """D19: PCL given the double radius 0.1 or 1/3 squares it in double, one ulp of r2 below the float radius's square; the library
    takes a float32 radius.  With the double radius the query of the rim cloud loses exactly its neighbours at d2 = float(r * r)."""
    for name, r in (("rim_0.1", 0.1), ("rim_0.333", 1 / 3)):
        p, rn, rf, cell = next(c[1:] for c in cons if c[0] == name)
        ref = restated[name][0]
        rank, inl = R.lattice_rank(p[:, :3], ref["cell"])
        lib, _ = R.canonical_neighbours(p[:, :3], 0, F32(r), rank, inl)
        pcl, _ = R.canonical_neighbours(p[:, :3], 0, r, rank, inl)
        assert np.array_equal(lib, ref["nbr_f"][0])
        lost = np.setdiff1d(lib, pcl)
        d2 = _flann_d2(p[0, :3], p[lib, :3])
        assert set(pcl) < set(lib) and np.array_equal(lost, np.sort(lib[d2 == radius_sq(r)]))


def test_pair_cases_hit_their_edges():
    cases = pair_cases()
    pf = R.pair_features_pcl32(*_pair_arrays(cases), R.D7_MATH)
    lab = {c[0]: i for i, c in enumerate(cases)}
    i = lab["|a1| == |a2|"]
    assert abs(pf["a1"][i]) == abs(pf["a2"][i]) and not pf["swap"][i]
    i = lab["equal acos of different |a|"]
    assert abs(pf["a1"][i]) != abs(pf["a2"][i]) and R.D7_MATH.acos(abs(pf["a1"][i])) == R.D7_MATH.acos(abs(pf["a2"][i]))
    assert not pf["swap"][i] and not pf["swap"][lab["equal acos, other order"]]
    assert not pf["ok"][lab["dp parallel to n1"]] and not pf["ok"][lab["dp parallel to n2 (swapped)"]] and not pf["ok"][lab["coincident"]]
    assert pf["swap"][lab["dp parallel to n2 (swapped)"]]
    assert np.isnan(pf["f1"][lab["NaN n1"]]) and np.isnan(pf["f2"][lab["NaN n2"]]) and not np.isnan(pf["f3"][lab["NaN n2"]])
    assert pf["f1"][lab["f1 = +pi"]] == R.PI_F and pf["f1"][lab["f1 = -pi"]] == -R.PI_F and pf["f1"][lab["f1 = pi from +0"]] == R.PI_F
    for name in ("f2", "f3"):
        vals = [pf[name][i] for c, i in lab.items() if c.startswith(name + " =")]
        assert F32(-1) in vals and F32(1) in vals
        sc = np.array([pf["scaled"][i, 1 if name == "f2" else 2] for c, i in lab.items() if c.startswith(name + " =")])
        for k in range(1, 11):                                         # each inner edge has values below it and at or above it
            near = sc[np.abs(sc - k) < 1e-5]
            assert (near < k).any() and (near >= k).any(), (name, k)
    for k in range(1, 11):
        below = pf["scaled"][lab[f"f1 edge {k} -1"], 0]
        at = pf["scaled"][lab[f"f1 edge {k} +0"], 0]
        above = pf["scaled"][lab[f"f1 edge {k} +1"], 0]
        assert below < k <= at < above and at - below < 1e-5, (k, below, at, above)
        assert pf["f1"][lab[f"f1 edge {k} +0"]] == np.nextafter(pf["f1"][lab[f"f1 edge {k} -1"]], F32(np.inf))


# ---- CPU: the D7 reading equals the oracle bit for bit ------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [c[0] for c in constructions()])
def test_restatement_matches_oracle(cons, restated, oracle, name):
    p, rn, rf, cell = next(c[1:] for c in cons if c[0] == name)
    ref = restated[name][0]
    cellv = resolved_cell(rn, rf, cell)
    for q in range(len(p)):
        for r, want in ((rf, ref["nbr_f"][q]), (rn, ref["nbr_n"][q])):
            idx, d2 = oracle.neighbors(p, cellv, q, r)
            assert np.array_equal(idx, want), (name, q, r, idx, want)
    n, d, s = oracle.compute_fpfh(p, rn, rf, cellv, want_spfh=True)
    assert same_bits(ref["normals"], n, nan_equal=True), name
    assert same_bits(ref["spfh"], s, nan_equal=True), name
    assert same_bits(ref["desc"], d, nan_equal=True), name


def test_pair_cases_match_oracle(oracle, oracle_bins):
    cases = pair_cases()
    pf = R.pair_features_pcl32(*_pair_arrays(cases), R.D7_MATH)
    bad = []
    for i, (label, p1, n1, p2, n2) in enumerate(cases):
        ok, f = oracle.pair_features(p1, n1, p2, n2)
        if ok != bool(pf["ok"][i]):
            bad.append(f"{label}: skipped {not ok} vs {not pf['ok'][i]}")
            continue
        if ok:
            mine = np.array([pf["f1"][i], pf["f2"][i], pf["f3"][i]], F32)
            if not same_bits(mine, f, nan_equal=True) or not np.array_equal(oracle_bins(*f), pf["bins"][i]):
                bad.append(f"{label}: {mine} {pf['bins'][i]} vs {f} {oracle_bins(*f)}")
    assert not bad, "\n".join(bad)


# ---- CPU: the float64 reading agrees where every margin clears ---------------------------------------------------------------------
# The normal lies within EIG_C * u * ||C|| / (l1 - l0) of the exact eigenvector of the float32 covariance it was computed from; the angle
# is atan2(|n x v|, |n . v|) in float64 (arccos(|n . v|) would read the float32 normalisation error of n, ~u, as ~sqrt(2u) rad).
EIG_C = 128.0


def normal_angle(n, v):
    n, v = np.asarray(n, F64), np.asarray(v, F64)
    return float(np.arctan2(np.linalg.norm(np.cross(n, v)), abs(np.dot(n, v))))


@pytest.mark.parametrize("name", [c[0] for c in constructions()])
def test_float64_reading_agrees_where_margins_clear(cons, restated, oracle, name):
    d7, f64 = restated[name]
    # the neighbour sets and the covariance do not depend on the transcendentals
    assert all(np.array_equal(a, b) for a, b in zip(d7["nbr_f"], f64["nbr_f"]))
    for q, (ra, rb) in enumerate(zip(d7["nrec"], f64["nrec"])):
        if "cov" in ra:
            assert same_bits(ra["cov"], rb["cov"]) and ra["branch"] == rb["branch"], (name, q)   # c0 precedes every transcendental
        if ra["branch"] == "roots2" and rb["branch"] == "roots2":  # no transcendental on this path: identical normals
            assert same_bits(d7["normals"][q], f64["normals"][q], nan_equal=True), (name, q)
    # normals within the eigengap bound of the exact eigenvector of the float32 covariance, on well-separated spectra
    for q, rec in enumerate(f64["nrec"]):
        if "cov" not in rec or not np.isfinite(f64["normals"][q]).all():
            continue
        w, v, k = R.eig_reference(rec["cov"])
        if w[0] < 0 or (w[1] - w[0]) < 1e-3 * np.abs(w).max() or rec["scale_reset"]:
            continue
        for reading in (d7, f64):
            ang = normal_angle(reading["normals"][q, :3], v)
            assert ang <= EIG_C * k, (name, q, ang, ang / k)
    # discrete outputs: per pair (skip, swap, bins) where the pair's margins and both normals clear; rows and descriptors where stable
    for q, (pa, pb) in enumerate(zip(d7["pairs"], f64["pairs"])):
        if not (f64["normal_stable"][q]):
            continue
        mg = pb["margins"]
        clear = (mg["swap"] > 1) & (mg["skip"] > 1) & (mg["bins"] > 1).all(1) & f64["normal_stable"][pb["other"]]
        assert np.array_equal(pa["ok"][clear], pb["ok"][clear]) and np.array_equal(pa["swap"][clear], pb["swap"][clear]), (name, q)
        both = clear & pa["ok"]
        assert np.array_equal(pa["bins"][both], pb["bins"][both]), (name, q)
    st = f64["spfh_stable"]
    assert same_bits(d7["spfh"][st], f64["spfh"][st], nan_equal=True), name
    st = f64["stable"]
    assert same_bits(d7["desc"][st], f64["desc"][st], nan_equal=True), name


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_matches_restatement(cons, restated, oracle):
    bad = []
    with make_handle(None, max_batch_slots=2) as h:
        for name, p, rn, rf, cell in cons:
            ref = restated[name][0]
            n_got, d_got = h.compute_fpfh(p, rn, rf, resolved_cell(rn, rf, cell))
            n_ref, d_ref = oracle.compute_fpfh(p, rn, rf, resolved_cell(rn, rf, cell))
            if not (same_bits(n_got, ref["normals"], nan_equal=True) and same_bits(d_got, ref["desc"], nan_equal=True)
                    and same_bits(n_got, n_ref, nan_equal=True) and same_bits(d_got, d_ref, nan_equal=True)):
                rows = np.flatnonzero(~((n_got.view(np.uint32) == ref["normals"].view(np.uint32)) | np.isnan(n_got) & np.isnan(ref["normals"])).all(1)
                                      | ~((d_got.view(np.uint32) == ref["desc"].view(np.uint32)) | np.isnan(d_got) & np.isnan(ref["desc"])).all(1))
                bad.append(f"{name}: rows {rows[:8]}")
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 4])
def test_mixed_wave_equals_single_calls(cons, restated, lanes):
    """Every construction in one describe_points_each call, each with its own radii and cell, shuffled: each cloud equals its single
    qb200_compute_fpfh call and the restatement."""
    order = np.random.default_rng(lanes).permutation(len(cons))
    sel = [cons[i] for i in order]
    params = [make_params(normal_radius=rn, fpfh_radius=rf, grid_cell=cell) for _, _, rn, rf, cell in sel]
    with make_handle(lanes, max_batch_slots=2) as h:
        per_cloud, counts, status = h.describe_points_each([p for _, p, *_ in sel], params)
        bad = []
        for (name, p, rn, rf, cell), (nrm, desc), cnt, st in zip(sel, per_cloud, counts, status):
            n1, d1 = h.compute_fpfh(p, rn, rf, resolved_cell(rn, rf, cell))
            ref = restated[name][0]
            if not (st == 0 and cnt == len(p) and nrm.tobytes() == n1.tobytes() and desc.tobytes() == d1.tobytes()
                    and same_bits(desc, ref["desc"], nan_equal=True) and same_bits(nrm, ref["normals"], nan_equal=True)):
                bad.append(f"{name}: status {st}, count {cnt}")
    assert not bad, "\n".join(bad)
