"""Ground removal (Patchwork, patchwork.hpp:264-455) and range-image segmentation (imageProjection.hpp:273-579) on scans built to hit
the places where pw_patch_kernel and the ip_* kernels can go wrong: zone / ring / sector edges, z ties and signed zeros, patch sizes
at num_min_pts and at the 16 384 points of shared memory, seed and threshold edges, degenerate ground sets, every branch of the
likelihood test; pixel collisions, the 0.1 m range cut, the first and last rows, the column wrap, long union-find chains, the two
cross / 4-neighbour patterns and segments exactly at their feasibility limits.

CPU: the oracle agrees exactly -- same points in the same order -- with float64 restatements written from the reference text.  Both
restatements return per-patch / per-segment detail, so that a disagreement can be traced to one step, and every construction asserts
that it hits the edge it is built for.  GPU (-m gpu): qb200_patchwork, qb200_segment_cloud and qb200_preprocess_batch are
byte-identical to the oracle on every case, alone and as one mixed batch through 1 and 4 lanes."""
import math

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import MEM_DEVICE, default_patchwork_params, default_segment_params
from support import same_bits

CAPACITY_EXCEEDED = 3
MAX_PATCH = 16384
F32 = np.float32


# ==== Patchwork: float64 restatement ==========================================================================================
def _d17_normal(cov):
    """Smallest-eigenvalue eigenvector of a symmetric PSD 3x3 (LAPACK), oriented n_z >= 0 (D13).  When that eigenvalue has
    multiplicity >= 2 the reference's JacobiSVD returns a basis vector that depends on rounding; D17 fixes it: (0,0,1) when it lies
    in the eigenspace, else (u_y, -u_x, 0) normalised for u = the largest row of cov - lambda I, or (1,0,0) when u is vertical."""
    w, V = np.linalg.eigh(cov)
    top = max(abs(w[2]), 1e-300)
    if w[1] - w[0] > 1e-12 * top:
        n = V[:, 0]
        return -n if n[2] < 0 else n
    m = cov - w[0] * np.eye(3)
    m[np.abs(m) < 1e-12 * top] = 0.0
    if not m[:, 2].any():
        return np.array([0.0, 0.0, 1.0])
    u = m[int(np.argmax((m * m).sum(1)))]
    h = math.hypot(u[0], u[1])
    return np.array([u[1] / h, -u[0] / h, 0.0]) if h > 0 else np.array([1.0, 0.0, 0.0])


def _patch_ids(P, pp):
    """pc2czm (patchwork.hpp:512-543) per point: zone, ring, sector, the unclamped ring / sector quotients, patch id (-1: not binned)."""
    x, y = P[:, 0], P[:, 1]
    with np.errstate(invalid="ignore"):
        r = np.sqrt(x * x + y * y)
        at = np.arctan2(y, x)
    theta = np.where(at > 0, at, at + 2 * np.pi)
    mr = list(pp.min_ranges_each_zone[:4]) + [pp.max_range]
    zone = np.where(r < mr[1], 0, np.where(r < mr[2], 1, np.where(r < mr[3], 2, 3)))
    ring_q, sec_q = np.zeros(len(P)), np.zeros(len(P))
    ring, sec, pid = np.zeros(len(P), int), np.zeros(len(P), int), np.full(len(P), -1)
    base = 0
    for k in range(4):
        nr, ns = pp.num_rings_each_zone[k], pp.num_sectors_each_zone[k]
        sel = zone == k
        rq = (r[sel] - mr[k]) / ((mr[k + 1] - mr[k]) / nr)
        sq = theta[sel] / (2 * np.pi / ns)
        ring_q[sel], sec_q[sel] = rq, sq
        ri = np.minimum(np.where(np.isfinite(rq), rq, 0).astype(np.int64), nr - 1)
        si = np.minimum(np.where(np.isfinite(sq), sq, 0).astype(np.int64), ns - 1)
        ring[sel], sec[sel], pid[sel] = ri, si, base + ri * ns + si
        base += nr * ns
    ok = np.isfinite(P).all(1) & ~(P[:, 2] < -1.8 * pp.sensor_height) & (r <= pp.max_range) & (r > pp.min_range)
    pid[~ok] = -1
    return dict(r=r, theta=theta, zone=zone, ring=ring.astype(int), sector=sec, ring_q=ring_q, sector_q=sec_q, pid=pid)


def _ref_patchwork(pts, pp):
    """PatchWork::estimate_ground in float64 (two-pass covariance, LAPACK eigenvectors).  Returns (ground indices, non-ground indices,
    status, per-point ids, per-patch records) with the outputs in the reference's order: patches zone -> ring -> sector, ascending
    (z, input index) inside (D11), a rejected patch's ground part first."""
    P = pts[:, :3].astype(np.float64)
    ids = _patch_ids(P, pp)
    pid = ids["pid"]
    G, N, patches, status = [], [], [], 0
    low_margin = -0.1 if pp.sensor_height == 0.0 else pp.adaptive_seed_selection_margin * pp.sensor_height
    nthr = pp.num_thresholds
    concentric, p = 0, 0
    for k in range(4):
        for ring in range(pp.num_rings_each_zone[k]):
            for sector in range(pp.num_sectors_each_zone[k]):
                idx = np.nonzero(pid == p)[0]
                p += 1
                m = len(idx)
                if m <= pp.num_min_pts:
                    continue
                if m > MAX_PATCH:
                    status = CAPACITY_EXCEEDED
                    continue
                idx = idx[np.lexsort((idx, P[idx, 2]))]
                Q, z = P[idx], P[idx, 2]
                init = 0
                if k == 0:
                    while init < m and z[init] < low_margin:
                        init += 1
                s, c = 0.0, 0
                for v in z[init:]:
                    if c >= pp.num_lpr:
                        break
                    s += v
                    c += 1
                lpr = s / c if c else 0.0
                g = z < lpr + pp.th_seeds
                seeds = int(g.sum())
                n, mean, surf = np.array([0.0, 0.0, 1.0]), np.zeros(3), 0.0
                for _ in range(pp.num_iter):
                    if g.any():                       # D14: an empty ground set keeps the previous plane
                        mean = Q[g].mean(0)
                        cov = (Q[g] - mean).T @ (Q[g] - mean) / g.sum()
                        n = _d17_normal(cov)
                        ev = np.abs(np.linalg.eigvalsh(cov))
                        surf = ev.min() / ev.sum() if ev.sum() > 0 else 0.0      # D13: 0 for a zero trace
                    th = F32(pp.th_dist - (-(n @ mean)))                         # th_dist_d_ is a float
                    g = Q @ n < th
                ti = min(ring + 2 * k, nthr - 1)
                if abs(n[2]) < pp.uprightness_thr:
                    keep, branch = False, "upright"
                elif concentric < nthr:
                    if mean[2] > pp.elevation_thresholds[ti]:
                        keep, branch = pp.flatness_thresholds[ti] > surf, "flatness"
                    else:
                        keep, branch = True, "low"
                else:
                    keep = not (pp.using_global_elevation and mean[2] > pp.global_elevation_threshold)
                    branch = "global"
                if keep:
                    G += list(idx[g]); N += list(idx[~g])
                else:
                    N += list(idx[g]) + list(idx[~g])
                patches.append(dict(pid=p - 1, zone=k, ring=ring, sector=sector, m=m, init=init, lpr=lpr, seeds=seeds, normal=n,
                                    mean=mean, surf=surf, keep=keep, branch=branch, ground=idx[g], nonground=idx[~g]))
            concentric += 1
    return np.array(G, int), np.array(N, int), status, ids, patches


# ==== Patchwork: constructions ================================================================================================
def _pp(**kw):
    pp = default_patchwork_params()
    for k, v in kw.items():
        setattr(pp, k, v)
    return pp


def _centre(pp, k, ring, sector):
    mr = list(pp.min_ranges_each_zone[:4]) + [pp.max_range]
    rs = (mr[k + 1] - mr[k]) / pp.num_rings_each_zone[k]
    ss = 2 * np.pi / pp.num_sectors_each_zone[k]
    return mr[k] + (ring + 0.5) * rs, (sector + 0.5) * ss, rs, ss


def _carpet(pp, k, ring, sector, n=96, z0=-1.75, dz=0.03, seed=0):
    """n points inside patch (k, ring, sector), away from its edges; z on three levels around z0 (not degenerate)."""
    r0, t0, rs, ss = _centre(pp, k, ring, sector)
    rng = np.random.default_rng(seed + 7919 * k + 131 * ring + sector)
    r = r0 + rng.uniform(-0.3, 0.3, n) * rs
    t = t0 + rng.uniform(-0.3, 0.3, n) * ss
    z = z0 + dz * (np.arange(n) % 3 - 1)
    return np.stack([r * np.cos(t), r * np.sin(t), z], 1)


def _grid(x0, y0, n, step=0.0625, z=-1.75):
    """n points on an exactly representable square grid from (x0, y0) at height z: float sums over them are exact."""
    w = int(math.ceil(math.sqrt(n)))
    i = np.arange(n)
    return np.stack([x0 + step * (i % w), y0 + step * (i // w), np.full(n, z)], 1)


def _p4(*parts, shuffle=None):
    xyz = np.concatenate([np.asarray(p, np.float64).reshape(-1, 3) for p in parts]).astype(F32)
    out = np.ones((len(xyz), 4), F32)
    out[:, :3] = xyz
    if shuffle is not None:
        out = out[np.random.default_rng(shuffle).permutation(len(out))]
    out[:, 3] = np.arange(len(out), dtype=F32)          # the 4th channel carries the input index through the outputs
    return out


def _f32_around(v):
    """The float32 values just below, at (nearest) and just above the double v."""
    f = F32(v)
    return [np.nextafter(f, F32(-np.inf)), f, np.nextafter(f, F32(np.inf))]


def _all_carpets(pp, **kw):
    return [_carpet(pp, k, r, s, **kw) for k in range(4) for r in range(pp.num_rings_each_zone[k])
            for s in range(pp.num_sectors_each_zone[k])]


def _case_edges():
    """Every patch carpeted, plus points on the zone radii, the ring edges, min_range and max_range (on the +-y axis: r = |y|
    exactly), on the sector edges k * 2 pi / ns (theta = pi/4, pi/2, pi, 3 pi/2) and at theta = 0 / 2 pi with +0 and -0."""
    pp = _pp()
    mr = list(pp.min_ranges_each_zone[:4]) + [pp.max_range]
    edge = []
    for k in range(4):
        rs = (mr[k + 1] - mr[k]) / pp.num_rings_each_zone[k]
        for j in range(pp.num_rings_each_zone[k] + 1):
            for r in _f32_around(mr[k] + j * rs if j < pp.num_rings_each_zone[k] else mr[k + 1]):
                edge += [(0.0, r, -1.75), (0.0, -r, -1.75)]
    for r in (5.0, 10.0, 15.0, 30.0, 60.0, 80.0):
        edge += [(r, 0.0, -1.75), (r, -0.0, -1.75), (-r, 0.0, -1.75), (-r, -0.0, -1.75), (r, r * 1e-7, -1.75), (r, -r * 1e-7, -1.75)]
    for v in (3.0, 9.0, 20.0, 50.0):
        edge += [(v, v, -1.75), (-v, v, -1.75), (-v, -v, -1.75), (v, -v, -1.75)]
    return _p4(*_all_carpets(pp), np.array(edge), shuffle=1), pp


def _case_sizes():
    """Patches of num_min_pts (dropped), num_min_pts + 1, 16384 (one full bitonic sort of tied z) and 16385 points (capacity)."""
    pp = _pp()
    rng = np.random.default_rng(2)
    parts = [_carpet(pp, 0, 0, 1, n=80), _carpet(pp, 0, 0, 3, n=81), _carpet(pp, 1, 0, 5, n=81, z0=-1.0)]
    big = _carpet(pp, 2, 1, 7, n=MAX_PATCH)
    big[:, 2] = -1.75 + 0.03125 * rng.integers(-2, 3, MAX_PATCH)              # five z levels: thousands of ties each
    over = _carpet(pp, 3, 2, 9, n=MAX_PATCH + 1)
    return _p4(*parts, big, over, shuffle=2), pp


def _case_ties():
    """Many equal z in one patch (tie order D11), -0.0 and +0.0 mixed in the non-ground part of another."""
    pp = _pp()
    a = _carpet(pp, 0, 1, 4, n=300)
    a[:, 2] = np.where(np.arange(300) % 2 == 0, -1.75, -1.6875)
    b = _carpet(pp, 1, 1, 9, n=200)
    b[:100, 2] = -1.75
    b[100:, 2] = np.where(np.arange(100) % 3 == 0, -0.0, 0.0)                # well above the plane: non-ground, in index order
    b[150:, 2] = -b[150:, 2]
    return _p4(a, b, _carpet(pp, 2, 0, 0), shuffle=3), pp


def _case_low_margin():
    """Zone 0: a patch whose points all lie below adaptive_seed_selection_margin * sensor_height (init_idx == m, the LPR mean is
    taken over nothing), a patch with points at the float32 neighbours of that margin, points at the neighbours of the -1.8 h cut."""
    pp = _pp()
    margin, cut = pp.adaptive_seed_selection_margin * pp.sensor_height, -1.8 * pp.sensor_height
    a = _carpet(pp, 0, 0, 2, n=120)
    a[:, 2] = -2.5 + 0.25 * (np.arange(120) % 3)
    b = _carpet(pp, 0, 1, 6, n=120)
    b[:3, 2] = _f32_around(margin)
    b[3:6, 2] = _f32_around(margin)
    b[6:9, 2] = _f32_around(cut)
    b[9:20, 2] = -1.85
    return _p4(a, b, shuffle=4), pp


def _case_lpr_zero():
    """num_lpr = 0: the LPR height is 0, so a patch below z = th_seeds is all seeds and one above it has none (an empty ground set
    keeps the first plane, D14)."""
    pp = _pp(num_lpr=0)
    return _p4(_carpet(pp, 0, 0, 5, n=100), _carpet(pp, 1, 2, 3, n=100, z0=0.4), shuffle=5), pp


def _case_height_zero():
    """sensor_height = 0: everything below z = 0 is cut, the seed margin is -0.1; the ground sits on +0.0 / -0.0."""
    pp = _pp(sensor_height=0.0)
    a = _carpet(pp, 0, 0, 7, n=120)
    a[:, 2] = np.where(np.arange(120) % 2 == 0, 0.0, -0.0)
    a[::5, 2] = 0.0625
    a[:10, 2] = -1e-3
    b = _carpet(pp, 0, 1, 9, n=100, z0=0.05, dz=0.02)
    return _p4(a, b, shuffle=6), pp


def _case_degenerate():
    """Ground sets whose covariance has a repeated smallest eigenvalue (all points identical, a horizontal line along x, a diagonal
    horizontal line, a short vertical pole) or zero z-variance (an exactly flat patch), with exactly representable coordinates so that
    the float single-pass sums are exact; and a flat patch 70-80 m out, where those sums cancel."""
    pp = _pp()
    same = np.tile([[-10.0, 0.5, -1.75]], (100, 1))                                    # zone 0, ring 1, sector 7
    i = np.arange(128)
    xline = np.stack([9.0 + i / 64, np.full(128, 0.5), np.full(128, -1.75)], 1)        # zone 0, ring 1, sector 0
    diag = np.stack([-6.0 - i / 64, -6.0 - i / 64, np.full(128, -1.75)], 1)            # zone 1, ring 0: a line at 225 degrees
    pole = np.stack([np.full(128, 6.0), np.full(128, -3.0), -1.75 + i / 512], 1)       # zone 0, ring 0 or 1, sector 14
    flat = _grid(-1.0, 4.0, 128)                                                       # zone 0, ring 0, sector 4
    r = 72.0 + 6.0 * (i % 16) / 16
    t = 0.2 + 0.15 * (i // 16) / 8
    far = np.stack([r * np.cos(t), r * np.sin(t), np.full(128, -1.7)], 1)              # zone 3, ring 3
    return _p4(same, xline, diag, pole, flat, far, shuffle=7), pp


def _case_likelihood(global_elevation):
    """Every branch of the likelihood test: uprightness reject (a 63-degree slope), elevation above its threshold with a flat patch
    (flatness keep) and a rough one (flatness reject), elevation below (keep), and beyond the rings of interest the global-elevation
    test with a patch above and one below global_elevation_threshold."""
    pp = _pp(using_global_elevation=global_elevation)
    r0, t0, _, _ = _centre(pp, 0, 0, 1)
    slope = _grid(r0 * np.cos(t0) - 0.5, r0 * np.sin(t0) - 0.5, 144, step=0.08)
    slope[:, 2] = -1.75 + 2.0 * (slope[:, 0] - slope[:, 0].min())
    r0, t0, _, _ = _centre(pp, 0, 0, 9)
    flat_hi = _grid(np.floor(r0 * np.cos(t0)), np.floor(r0 * np.sin(t0)), 128, z=-1.0)
    r0, t0, _, _ = _centre(pp, 0, 0, 12)
    rough = _grid(np.floor(r0 * np.cos(t0)), np.floor(r0 * np.sin(t0)), 144, step=0.125, z=-1.0)
    rough[:, 2] += 0.0625 * np.where((np.arange(144) + np.arange(144) // 12) % 2 == 0, 1, -1)
    parts = [slope, flat_hi, rough, _carpet(pp, 0, 1, 3), _carpet(pp, 1, 1, 20, z0=-0.25),     # last: ring of interest, flatness
             _carpet(pp, 1, 2, 4, z0=-0.25), _carpet(pp, 1, 3, 8, z0=-0.75), _carpet(pp, 2, 0, 11, z0=-0.3)]
    return _p4(*parts, shuffle=8), pp


def _threshold_th_dist(d):
    """A th_dist for which float(th_dist - d) < th_dist - d: a point exactly on the float threshold is above it (not ground) in the
    reference's float comparison, and below it in a double one."""
    for t in np.arange(0.1, 0.2, 0.001):
        if float(F32(t - d)) < t - d:
            return float(t)
    raise AssertionError("no th_dist rounds down")


def _case_threshold():
    """An exactly flat patch at z = -1.75 (plane (0,0,1), d = 1.75 exactly) plus points whose residual is exactly the float
    th_dist_d_; th_seeds keeps them out of the seeds."""
    th = _threshold_th_dist(1.75)
    pp = _pp(th_dist=th, th_seeds=0.05)
    flat = _grid(4.0, 0.5, 128)
    on = _grid(4.5, 0.75, 8, step=0.125, z=float(F32(th - 1.75)))
    above = _grid(4.25, 0.625, 4, step=0.125, z=float(np.nextafter(F32(th - 1.75), F32(1))))
    return _p4(flat, on, above, shuffle=9), pp


def _case_seed_edge():
    """Points exactly at lpr + th_seeds (-1.75 + 0.25): not seeds.  With one iteration they decide the plane: seeds that included them
    would tilt it through both levels and make every point ground."""
    pp = _pp(num_iter=1)
    low = _grid(4.0, 1.0, 64)
    high = _grid(5.0, 1.0, 64, z=-1.5)
    return _p4(low, high, shuffle=10), pp


PW_CASES = {
    "edges": _case_edges, "sizes": _case_sizes, "ties": _case_ties, "low_margin": _case_low_margin, "lpr_zero": _case_lpr_zero,
    "height_zero": _case_height_zero, "degenerate": _case_degenerate, "likelihood": lambda: _case_likelihood(0),
    "likelihood_global": lambda: _case_likelihood(1), "threshold": _case_threshold, "seed_edge": _case_seed_edge,
}
_pw_cache = {}


def _pw_case(name):
    if name not in _pw_cache:
        pts, pp = PW_CASES[name]()
        _pw_cache[name] = (pts, pp, _ref_patchwork(pts, pp))
    return _pw_cache[name]


def _patch_at(patches, pts, point):
    """The record of the patch holding the input point with these coordinates."""
    hit = np.nonzero((pts[:, :3] == np.asarray(point, F32)).all(1))[0]
    for rec in patches:
        if np.isin(hit, np.concatenate([rec["ground"], rec["nonground"]])).any():
            return rec
    raise AssertionError(f"no processed patch holds {point}")


def _check_pw_edges(name, pts, pp, ref):
    G, N, status, ids, patches = ref
    by = {(r["zone"], r["ring"], r["sector"]): r for r in patches}
    if name == "edges":
        pid, rq, sq = ids["pid"], ids["ring_q"], ids["sector_q"]
        nr = np.array(pp.num_rings_each_zone)[ids["zone"]]
        ns = np.array(pp.num_sectors_each_zone)[ids["zone"]]
        binned = pid >= 0
        assert (binned & (ids["r"] == pp.max_range) & (rq == nr)).any()               # r == max_range: ring quotient == nr, clamped
        assert ((ids["r"] > pp.max_range) & (pid < 0)).any()
        assert (binned & (ids["sector_q"] == ns)).any()                                # theta = 2 pi (y = +-0, x > 0): clamped sector
        assert (binned & (sq == np.floor(sq)) & (sq > 0) & (sq < ns)).sum() >= 8       # exactly on inner sector edges
        for k in (1, 2, 3):                                                            # both sides of every zone radius
            b = pp.min_ranges_each_zone[k]
            assert ((ids["r"] < b) & (ids["r"] > b - 1e-5) & (ids["zone"] == k - 1) & binned).any()
            assert ((ids["r"] >= b) & (ids["r"] < b + 1e-5) & (ids["zone"] == k) & binned).any()
        lo = (ids["r"] <= pp.min_range) & (ids["r"] > pp.min_range - 1e-5)
        assert lo.any() and (pid[lo] < 0).all()
        assert ((ids["r"] > pp.min_range) & (ids["r"] < pp.min_range + 1e-5) & binned).any()
        inner = binned & (ids["ring"] > 0) & (np.abs(rq - np.round(rq)) < 1e-6)        # ring edges: neighbours on both sides
        assert inner.sum() >= 10
        assert len(G) > 0.9 * binned.sum()
    elif name == "sizes":
        assert status == CAPACITY_EXCEEDED
        ms = sorted(r["m"] for r in patches)
        assert ms[0] == pp.num_min_pts + 1 and ms[-1] == MAX_PATCH and (0, 0, 1) not in by
        assert (np.bincount(ids["pid"][ids["pid"] >= 0]) == MAX_PATCH + 1).any()
        assert (np.bincount(ids["pid"][ids["pid"] >= 0]) == pp.num_min_pts).any()
    elif name == "ties":
        rec = by[(1, 1, 9)]
        z = pts[rec["nonground"], 2]
        zero = rec["nonground"][z == 0]
        sign = np.signbit(pts[zero, 2]).astype(int)
        assert len(zero) == 100 and (np.diff(zero) > 0).all()                          # ties in input order whatever the sign
        assert (np.diff(sign) > 0).any() and (np.diff(sign) < 0).any()                 # -0.0 and +0.0 interleaved in that order
    elif name == "low_margin":
        rec = by[(0, 0, 2)]
        assert rec["init"] == rec["m"] and rec["lpr"] == 0.0 and rec["seeds"] == rec["m"]
        rec = by[(0, 1, 6)]
        assert rec["init"] == 6                                                        # the three float32 values below the margin
        margin, cut = pp.adaptive_seed_selection_margin * pp.sensor_height, -1.8 * pp.sensor_height
        z = pts[:, 2].astype(np.float64)
        assert ((z < margin) & (z > margin - 1e-6)).any() and ((z > margin) & (z < margin + 1e-6)).any()
        assert ((z < cut) & (z > cut - 1e-6) & (ids["pid"] < 0)).any() and ((z > cut) & (z < cut + 1e-6) & (ids["pid"] >= 0)).any()
    elif name == "lpr_zero":
        assert all(r["lpr"] == 0.0 for r in patches) and by[(0, 0, 5)]["seeds"] == by[(0, 0, 5)]["m"] and by[(1, 2, 3)]["seeds"] == 0
        assert len(by[(1, 2, 3)]["ground"]) == 0 and np.array_equal(by[(1, 2, 3)]["normal"], [0, 0, 1])
    elif name == "height_zero":
        rec = by[(0, 0, 7)]
        z = pts[np.concatenate([rec["ground"], rec["nonground"]]), 2]
        assert rec["m"] == 110 and (z >= 0).all() and np.signbit(z).any() and (z > 0).any()     # z < 0 cut, -0.0 kept
    elif name == "degenerate":
        for point, normal in (((-10, 0.5, -1.75), (0, 0, 1)), ((9, 0.5, -1.75), (0, 0, 1)), ((-6, -6, -1.75), (0, 0, 1)),
                              ((6, -3, -1.75), (1, 0, 0))):
            rec = _patch_at(patches, pts, point)
            assert np.array_equal(rec["normal"], normal), (point, rec["normal"])
        assert _patch_at(patches, pts, (-10, 0.5, -1.75))["keep"] and len(_patch_at(patches, pts, (-10, 0.5, -1.75))["ground"]) == 100
        assert not _patch_at(patches, pts, (6, -3, -1.75))["keep"]
        far = [r for r in patches if r["zone"] == 3]
        assert len(far) == 1 and far[0]["keep"] and len(far[0]["nonground"]) == 0
    elif name.startswith("likelihood"):
        branches = {(r["branch"], r["keep"]) for r in patches}
        assert {("upright", False), ("flatness", True), ("flatness", False), ("low", True)} <= branches
        assert ("global", not pp.using_global_elevation) in branches and ("global", True) in branches
    elif name == "threshold":
        th = F32(pp.th_dist - 1.75)
        assert float(th) < pp.th_dist - 1.75
        rec = patches[0]
        assert len(patches) == 1 and np.array_equal(rec["normal"], [0, 0, 1]) and rec["mean"][2] == -1.75
        on = np.nonzero(pts[:, 2] == th)[0]
        assert len(on) == 8 and np.isin(on, rec["nonground"]).all() and len(rec["ground"]) == 128
    elif name == "seed_edge":
        rec = patches[0]
        assert rec["lpr"] == -1.75 and rec["seeds"] == 64 and len(rec["ground"]) == 64


@pytest.mark.parametrize("name", list(PW_CASES))
def test_patchwork_constructions_hit_their_edges(name):
    pts, pp, ref = _pw_case(name)
    _check_pw_edges(name, pts, pp, ref)


@pytest.mark.parametrize("name", list(PW_CASES))
def test_patchwork_oracle_matches_float64_reference(oracle, name):
    pts, pp, (G, N, status, _, patches) = _pw_case(name)
    g, ng, st = oracle.patchwork(pts, pp)
    assert st == status
    got_g, got_n = g[:, 3].astype(int), ng[:, 3].astype(int)
    for got, want, what in ((got_g, G, "ground"), (got_n, N, "non-ground")):
        if not np.array_equal(got, want):
            pos = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
            i = (want if pos < len(want) else got)[pos]
            rec = next((r for r in patches if i in r["ground"] or i in r["nonground"]), None)
            pytest.fail(f"{what} output differs at {pos} of {len(want)} (oracle has {len(got)}): point {i} {pts[i, :3]}, patch {rec}")
    assert same_bits(g, pts[G]) and same_bits(ng, pts[N])


def test_degenerate_ground_sets_keep_their_ground():
    """The closed-form eigenvector is 0/0 for a covariance of rank <= 1; D17 gives (0,0,1) for identical points and for a horizontal
    line, so both are ground like JacobiSVD makes them, and a vertical pole is rejected with the normal (1,0,0)."""
    from oracle import Oracle
    o = Oracle()
    pp = _pp()
    for pts in (_p4(np.tile([[10.0, 0.5, -1.75]], (100, 1))), _p4(np.stack([9.0 + np.arange(128) / 64, np.full(128, 0.5),
                                                                           np.full(128, -1.75)], 1))):
        g, ng, st = o.patchwork(pts, pp)
        assert st == 0 and len(g) == len(pts) and len(ng) == 0
    pole = _p4(np.stack([np.full(128, 6.0), np.full(128, -3.0), -1.75 + np.arange(128) / 512], 1))
    g, ng, _ = o.patchwork(pole, pp)
    assert len(g) == 0 and same_bits(ng, pole)


# ==== range image: float64 restatement ========================================================================================
def _seg_params(kind, mode):
    sp = default_segment_params()
    if kind == "vlp16":
        sp.n_scan, sp.horizon_scan, sp.ang_res_x, sp.ang_res_y, sp.ang_bottom = 16, 1800, 0.2, 2.0, 15.1
    elif kind == "tiny":
        sp.n_scan, sp.horizon_scan, sp.ang_res_x, sp.ang_res_y, sp.ang_bottom = 1, 8, 45.0, 2.0, 1.0
        sp.min_pts_for_subclustering = 8
    sp.neighbor_mode = mode
    return sp


def _project64(pts, sp):
    """imageProjection.hpp:308-352 in float64 from the float32 coordinates: (row, col, fractional row, fractional column offset from
    the column's centre)."""
    x, y, z = (pts[:, i].astype(np.float64) for i in range(3))
    rf = (np.degrees(np.arctan2(z, np.sqrt(x * x + y * y))) + sp.ang_bottom) / sp.ang_res_y
    q = (np.degrees(np.arctan2(x, y)) - 90.0) / float(sp.ang_res_x)
    col = (-np.round(q) + sp.horizon_scan // 2).astype(np.int64)
    col = np.where(col >= sp.horizon_scan, col - sp.horizon_scan, col)
    return np.floor(rf).astype(np.int64), col, rf - np.floor(rf), q - np.round(q)


def _ref_segments(pts, pix, sp):
    """segmentCloud in "Patchwork" mode: pix[i] = the pixel point i was placed in (row * W + col, -1: none).  The last finite point of
    a pixel with float range >= 0.1 wins; segments are the connected components (scipy) of the pixel graph under the angle criterion;
    a segment is valid with >= min_pts_for_subclustering pixels, or >= segment_valid_point_num pixels whose rows OTHER than the
    seed's pixel (the lowest pixel: the seed of the row-major sweep) number >= segment_valid_line_num.  Returns (valid point indices,
    outlier point indices) in row-major pixel order and the per-segment records."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    H, W = sp.n_scan, sp.horizon_scan
    x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
    rng = np.sqrt(x * x + y * y + z * z)                      # float32, the reference's order
    ok = np.isfinite(pts[:, :3]).all(1) & (pix >= 0) & ~(rng < F32(0.1))
    win = np.full(H * W, -1, np.int64)
    for i in np.nonzero(ok)[0]:
        win[pix[i]] = i
    occ = np.nonzero(win >= 0)[0]
    img = np.full(H * W, np.nan)
    img[occ] = rng[win[occ]]
    offs = {0: [(-1, 0), (0, 1), (0, -1), (1, 0)], 1: [(-1, 0), (0, 1), (0, -1), (1, 0), (-1, -1), (-1, 1), (1, 1), (1, -1)],
            2: [(-1, -1), (-1, 1), (1, 1), (1, -1)]}[sp.neighbor_mode]
    alpha = {0: math.radians(float(sp.ang_res_x)), 1: math.radians(float(sp.ang_res_y))}
    src, dst = [], []
    for q in occ:
        i, j = divmod(int(q), W)
        for di, dj in offs:
            ti, tj = i + di, (j + dj) % W
            if not 0 <= ti < H or win[ti * W + tj] < 0:
                continue
            a, b = img[q], img[ti * W + tj]
            al = alpha[0] if di == 0 else alpha[1]
            d1, d2 = max(a, b), min(a, b)
            if math.atan2(d2 * math.sin(al), d1 - d2 * math.cos(al)) > sp.segment_theta:
                src.append(q); dst.append(ti * W + tj)
    _, lab = connected_components(coo_matrix((np.ones(len(src)), (src, dst)), shape=(H * W, H * W)), directed=False)
    segs, feasible = {}, {}
    for q in occ:
        segs.setdefault(lab[q], []).append(int(q))
    recs = []
    for l, px in segs.items():
        rows = {p // W for p in px[1:]}                           # px is ascending: px[0] is the seed
        ok_seg = len(px) >= sp.min_pts_for_subclustering or (len(px) >= sp.segment_valid_point_num and len(rows) >= sp.segment_valid_line_num)
        feasible[l] = ok_seg
        recs.append(dict(seed=px[0], size=len(px), rows=len(rows), rows_with_seed=len(rows | {px[0] // W}), valid=ok_seg,
                         pixels=px))
    valid = [win[q] for q in occ if feasible[lab[q]]]
    outlier = [win[q] for q in occ if not feasible[lab[q]]]
    return np.array(valid, int), np.array(outlier, int), recs


# ==== range image: constructions (points placed at pixel centres) =============================================================
def _pixel_points(sp, rows, cols, ranges):
    rows, cols, ranges = (np.asarray(a, np.float64) for a in (rows, cols, ranges))
    v = np.radians((rows + 0.5) * float(sp.ang_res_y) - float(sp.ang_bottom))
    h = 90.0 - (cols - sp.horizon_scan // 2) * float(sp.ang_res_x)
    h = np.radians(np.where(h > 180.0, h - 360.0, np.where(h <= -180.0, h + 360.0, h)))
    return np.stack([ranges * np.cos(v) * np.sin(h), ranges * np.cos(v) * np.cos(h), ranges * np.sin(v)], 1)


class _Image:
    """A scan built pixel by pixel: every point remembers the pixel it was placed in."""

    def __init__(self, sp):
        self.sp, self.xyz, self.pix = sp, [], []

    def put(self, rows, cols, ranges):
        rows, cols = np.atleast_1d(rows), np.atleast_1d(cols) % self.sp.horizon_scan
        rows, cols = np.broadcast_arrays(rows, cols)
        ranges = np.broadcast_to(np.asarray(ranges, np.float64), rows.shape)
        self.xyz.append(_pixel_points(self.sp, rows.ravel(), cols.ravel(), ranges.ravel()))
        self.pix.append((rows * self.sp.horizon_scan + cols).ravel())
        return self

    def raw(self, xyz, pix=-1):
        self.xyz.append(np.asarray(xyz, np.float64).reshape(-1, 3))
        self.pix.append(np.full(len(self.xyz[-1]), pix))
        return self

    def build(self):
        pts = np.ones((sum(len(a) for a in self.xyz), 4), F32)
        pts[:, :3] = np.concatenate(self.xyz).astype(F32)
        pix = np.concatenate(self.pix).astype(np.int64)
        fin = np.isfinite(pts[:, :3]).all(1) & (pix >= 0)
        row, col, fr, fc = _project64(pts[fin], self.sp)
        # every placed point projects into its pixel with a margin no atan2 rounding can cross
        assert np.array_equal(row * self.sp.horizon_scan + col, pix[fin])
        assert (np.abs(fr - 0.5) < 0.45).all() and (np.abs(fc) < 0.45).all()
        return pts, pix


LEVEL = (10.0, 20.0, 40.0, 80.0, 160.0)     # neighbouring pixels of one level join, of two levels never (ratio >= 2)


def _seg_features(sp):
    """Collisions, the 0.1 m cut, the first and last rows, the column wrap and segments exactly at their feasibility limits
    (4-neighbour shapes), on an image of >= 16 rows."""
    H, W = sp.n_scan, sp.horizon_scan
    im = _Image(sp)
    im.put(2, np.arange(100, 110), 10.0)                           # a row segment the collisions sit next to
    im.put(3, 100, 10.0).put(3, 100, 40.0)                         # two points in one pixel: the last (40 m) wins -> cut off
    im.put(3, 105, 40.0).put(3, 105, 10.0)                         # ... the last (10 m) wins -> joins the segment
    im.put(3, 108, 10.0).raw([[np.nan, 1.0, 1.0]], 3 * W + 108)    # a NaN point never wins
    im.put(3, 109, 10.0).put(3, 109, 0.0999)                       # below 0.1 m: dropped, the 10 m point stays
    im.put(5, 120, 0.1001).put(5, 122, 0.0999)                     # just above / just below the cut, alone
    im.put(0, np.arange(200, 235), 10.0)                           # row 0: 35 pixels
    im.put(H - 1, np.arange(200, 212), 20.0)                       # last row
    im.put(np.arange(H - 5, H), 260, 10.0)                         # a 5-pixel column ending in the last row: 4 rows besides the seed
    im.put(np.arange(H - 3, H), 270, 10.0).put([H - 2, H - 1], 271, 10.0)   # 5 pixels, seed row alone: 2 rows besides the seed
    im.put([6, 6, 7, 8, 7], [W - 1, 0, 0, 0, W - 1], 10.0)        # crosses the wrap: 5 pixels, rows 6, 7, 8 besides the seed (6, 0)
    im.put(8, np.arange(300, 330), 20.0)                           # exactly min_pts_for_subclustering
    im.put(10, np.arange(300, 329), 20.0)                          # one short, one row
    im.put([12, 13, 13, 14, 14], [300, 300, 301, 300, 301], 10.0)  # 5 pixels, 3 rows, seed row alone -> 2 rows without it
    im.put([12, 12, 13, 14, 14], [310, 311, 310, 310, 311], 10.0)  # 5 pixels, 3 rows, seed row shared -> 3 rows
    im.put(np.arange(9, 13), 340, 10.0)                            # 4 pixels over 4 rows
    im.put(np.arange(9, 14), 350, 20.0)                            # 5 pixels over 5 rows
    return im.build()


def _seg_checker(sp, period):
    """Every pixel occupied, level (i + period * j) mod len: period 1 = checkerboard of two levels (diagonals join: connected only in
    cross mode); (i + 2 j) mod 5 separates every pixel from all eight neighbours."""
    H, W = sp.n_scan, sp.horizon_scan
    i, j = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    lev = (i + j) % 2 if period == 1 else (i + 2 * j) % 5
    return _Image(sp).put(i.ravel(), j.ravel(), np.array(LEVEL)[lev.ravel()]).build()


def _seg_lines(sp):
    """Horizontal and vertical runs: connected only in 4-neighbour mode."""
    H, W = sp.n_scan, sp.horizon_scan
    im = _Image(sp)
    for r in range(0, H, 3):
        im.put(r, np.arange(0, W, 2)[: W // 2] if r % 2 else np.arange(W), 10.0 if r % 2 else 20.0)
    return im.build()


def _seg_whole(sp):
    H, W = sp.n_scan, sp.horizon_scan
    i, j = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    return _Image(sp).put(i.ravel(), j.ravel(), 10.0).build()


def _seg_snake(sp):
    """A boustrophedon over every second row, joined at alternate ends: one path over half the image (the longest union-find
    chains), in reverse input order so that later points sit at lower pixels."""
    H, W = sp.n_scan, sp.horizon_scan
    im = _Image(sp)
    rows, cols = [], []
    for r in range(0, H, 2):
        rows += [r] * W; cols += list(range(W))
        if r + 1 < H:
            rows.append(r + 1); cols.append(W - 1 if (r // 2) % 2 == 0 else 0)
    rows, cols = np.array(rows)[::-1], np.array(cols)[::-1]
    return im.put(rows, cols, 10.0).build()


def _seg_tiny(sp):
    """n_scan = 1, horizon_scan = 8: seven pixels of one level and one collision; the wrap joins columns 7 and 0."""
    im = _Image(sp)
    im.put(0, [7, 0, 1, 2, 3, 4], 10.0).put(0, 5, 10.0).put(0, 5, 80.0).put(0, 6, 80.0).put(0, 6, 10.0)
    return im.build()


def _seg_tiny_split(sp):
    """... and two levels alternating: every pixel alone, except across the wrap."""
    return _Image(sp).put(0, np.arange(8), np.array(LEVEL)[[0, 1, 0, 1, 0, 1, 2, 0]]).build()


SEG_CASES = {
    ("default", "features"): _seg_features, ("default", "checker"): lambda sp: _seg_checker(sp, 1),
    ("default", "isolated"): lambda sp: _seg_checker(sp, 2), ("default", "lines"): _seg_lines, ("default", "whole"): _seg_whole,
    ("default", "snake"): _seg_snake, ("vlp16", "features"): _seg_features, ("vlp16", "checker"): lambda sp: _seg_checker(sp, 1),
    ("vlp16", "snake"): _seg_snake, ("tiny", "row"): _seg_tiny, ("tiny", "split"): _seg_tiny_split,
}
SEG_IDS = [f"{k}-{c}-m{m}" for k, c in SEG_CASES for m in (0, 1, 2)]
_seg_cache = {}


def _seg_case(kind, case, mode):
    key = (kind, case, mode)
    if key not in _seg_cache:
        sp = _seg_params(kind, mode)
        pts, pix = SEG_CASES[(kind, case)](sp)
        _seg_cache[key] = (pts, sp, pix, _ref_segments(pts, pix, sp))
    return _seg_cache[key]


def _seg_keys():
    return [(k, c, m) for k, c in SEG_CASES for m in (0, 1, 2)]


def _check_seg_edges(kind, case, mode, pts, sp, pix, ref):
    valid, outlier, recs = ref
    H, W = sp.n_scan, sp.horizon_scan
    occupied = sum(r["size"] for r in recs)
    if case == "features":
        x = pts[:, :3]
        rng = np.sqrt((x * x).sum(1))
        assert ((rng < F32(0.1)) & (rng > 0.099)).sum() == 2 and ((rng >= F32(0.1)) & (rng < 0.101)).sum() == 1
        assert len(np.unique(pix[pix >= 0])) < (pix >= 0).sum()                       # collisions
        assert 3 * W + 105 in [p for r in recs for p in r["pixels"]]
        if mode == 0:
            size = {r["seed"]: r for r in recs}
            at = lambda row, col: size[row * W + col]
            assert at(0, 200)["size"] == 35 and at(0, 200)["valid"]
            assert at(H - 5, 260)["size"] == 5 and at(H - 5, 260)["rows"] == 4 and at(H - 5, 260)["valid"]
            assert at(H - 3, 270)["rows"] == 2 and at(H - 3, 270)["rows_with_seed"] == 3 and not at(H - 3, 270)["valid"]
            assert at(6, 0)["size"] == 5 and at(6, 0)["rows"] == 3 and at(6, 0)["valid"]          # only through the wrap
            assert at(8, 300)["size"] == sp.min_pts_for_subclustering and at(8, 300)["valid"]
            assert at(10, 300)["size"] == sp.min_pts_for_subclustering - 1 and not at(10, 300)["valid"]
            assert at(12, 300)["rows"] == 2 and at(12, 300)["rows_with_seed"] == 3 and not at(12, 300)["valid"]
            assert at(12, 310)["rows"] == 3 and at(12, 310)["valid"]
            assert at(9, 340)["size"] == 4 and not at(9, 340)["valid"] and at(9, 350)["size"] == 5 and at(9, 350)["valid"]
            assert at(2, 100)["size"] == 13                                           # 10 + the pixels (3, 105), (3, 108), (3, 109)
            assert at(3, 100)["size"] == 1
    elif case == "checker":
        assert occupied == H * W
        if mode == 0:
            assert len(recs) == H * W
        if mode == 2 and H > 1:
            assert len(recs) == 2 and len(valid) == H * W
    elif case == "isolated":
        assert occupied == H * W and len(recs) == H * W and len(valid) == 0
    elif case == "lines":
        big = max(r["size"] for r in recs)
        assert (big == W) if mode != 2 else (big == 1)
    elif case == "whole":
        assert occupied == H * W
        assert len(recs) == (1 if mode != 2 else 2)
    elif case == "snake":
        if mode == 0:
            assert len(recs) == 1 and recs[0]["size"] > 0.45 * H * W
    elif case == "row":
        if mode != 2:
            assert len(recs) == 2 and {r["size"] for r in recs} == {7, 1}          # the 80 m winner of column 5 splits nothing off...
        else:
            assert len(recs) == 8 and len(valid) == 0                              # no diagonal neighbours in one row
    elif case == "split":
        if mode != 2:
            assert sorted(r["size"] for r in recs) == [1] * 6 + [2]                # columns 7 and 0 through the wrap


@pytest.mark.parametrize("key", _seg_keys(), ids=SEG_IDS)
def test_segment_constructions_hit_their_edges(key):
    pts, sp, pix, ref = _seg_case(*key)
    _check_seg_edges(*key, pts, sp, pix, ref)


@pytest.mark.parametrize("key", _seg_keys(), ids=SEG_IDS)
def test_segment_oracle_matches_float64_reference(oracle, key):
    pts, sp, _, (valid, outlier, _) = _seg_case(*key)
    v, o = oracle.segment_cloud(pts, sp)
    want = lambda idx: np.concatenate([pts[idx, :3], np.ones((len(idx), 1), F32)], 1) if len(idx) else np.zeros((0, 4), F32)
    assert same_bits(v, want(valid)), (len(v), len(valid))
    assert same_bits(o, want(outlier)), (len(o), len(outlier))


# ==== GPU =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PW_CASES))
def test_patchwork_gpu_matches_oracle_on_adversarial_scans(handle, oracle, name):
    pts, pp, _ = _pw_case(name)
    g_o, n_o, st_o = oracle.patchwork(pts, pp)
    g_g, n_g, st_g = handle.patchwork(pts, pp)
    assert st_g == st_o
    assert same_bits(g_g, g_o), "ground output differs"
    assert same_bits(n_g, n_o), "non-ground output differs"


@pytest.mark.gpu
@pytest.mark.parametrize("key", _seg_keys(), ids=SEG_IDS)
def test_segment_cloud_gpu_matches_oracle_on_adversarial_images(handle, oracle, key):
    pts, sp, _, _ = _seg_case(*key)
    v_o, o_o = oracle.segment_cloud(pts, sp)
    v_g, o_g = handle.segment_cloud(pts, sp)
    assert same_bits(v_g, v_o), "valid segments differ"
    assert same_bits(o_g, o_o), "outliers differ"


def _pass_through():
    """Patchwork parameters under which every point of a range-image case reaches the segmentation: no range or height cut, every
    patch processed and rejected (uprightness > 1), so the whole scan is the non-ground output."""
    return _pp(min_range=0.0, max_range=1000.0, sensor_height=100.0, num_min_pts=0, uprightness_thr=2.0,
               min_ranges_each_zone=(0.0, 1.0, 2.0, 3.0))


def _oracle_chain(oracle, scan, pp, sp):
    g, ng, st = oracle.patchwork(scan, pp)
    v, o = oracle.segment_cloud(ng, sp)
    return (g, ng, v, o), [len(g), len(ng), len(v), len(o)], st


def _check_batch_against_oracle(h, oracle, scans, pp, sp):
    per, counts, status = h.preprocess_batch(scans, pp, sp)
    for i, sc in enumerate(scans):
        outs, cnt, st = _oracle_chain(oracle, sc, pp, sp)
        assert list(counts[i]) == cnt and status[i] == st, (i, list(counts[i]), cnt, status[i], st)
        for k in range(4):
            assert same_bits(per[i][k], outs[k]), (i, k)
    return per, counts, status


@pytest.mark.gpu
@pytest.mark.parametrize("lanes", ["1", "4"])
def test_mixed_adversarial_batch_matches_oracle(oracle, monkeypatch, lanes):
    """Every Patchwork case under every case's parameters, with the default-image segmentation cases in the same waves; every
    range-image case under its own segment parameters behind pass-through Patchwork parameters; then the valid segments of one
    batch (device outputs) feed qb200_register_batch."""
    import torch
    monkeypatch.setenv("QB200_LANES", lanes)
    pw_scans = [_pw_case(n)[0] for n in PW_CASES]
    seg_default = [_seg_case("default", c, 2)[0] for c in ("features", "snake", "checker")]
    with capi.Handle(max_batch_slots=2) as h:                         # waves of 4 scans
        for name in PW_CASES:
            _check_batch_against_oracle(h, oracle, pw_scans + seg_default, _pw_case(name)[1], default_segment_params())
        for kind in ("default", "vlp16", "tiny"):
            for mode in (0, 1, 2):
                scans = [_seg_case(kind, c, mode)[0] for k, c in SEG_CASES if k == kind]
                _check_batch_against_oracle(h, oracle, scans, _pass_through(), _seg_params(kind, mode))
        if lanes != "4":
            return
        # registration of the device valid segments: two generator scans and an adversarial one
        pp, sp = default_patchwork_params(), default_segment_params()
        src, tgt, _ = synth.outdoor_pair(901)
        scans = [src, tgt, _pw_case("edges")[0]]
        cap = sp.n_scan * sp.horizon_scan
        buf = {"valid4": torch.zeros((len(scans), cap, 4), dtype=torch.float32, device="cuda")}
        _, counts, status = h.preprocess_batch(scans, pp, sp, cap=cap, dest=MEM_DEVICE, arrays=buf)
        assert (status == 0).all()
        valid = [_oracle_chain(oracle, s, pp, sp)[0][2] for s in scans]
        assert all(same_bits(buf["valid4"][i, :int(counts[i, 2])].cpu().numpy(), valid[i]) for i in range(len(scans)))
        pairs = [(0, 1), (2, 1)]
        p = capi.default_params()
        p.skip_flagged = 0
        ptr = lambda i: buf["valid4"][i].data_ptr()
        got = h.register_batch([(ptr(a), int(counts[a, 2]), ptr(b), int(counts[b, 2])) for a, b in pairs], p, kind=MEM_DEVICE)
        ref = h.register_batch([(valid[a], valid[b]) for a, b in pairs], p)
        assert got.tobytes() == ref.tobytes()
        res, st = oracle.register_pair(valid[0], valid[1], p)
        assert got[0]["status"] == st and got[0]["n_corr"] == res.n_corr and got[0]["clique_size"] == res.clique_size
