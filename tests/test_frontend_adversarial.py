"""The front end (K1 voxel sort, K2-K5 lattice / normals / SPFH / FPFH) against the CPU oracle on clouds built to sit on its
structural edges: every digit count of the voxel sort, tile / chunk / index-width boundaries, unstable-sort detectors, cell
boundaries, the `w` flag, clouds far from the origin, every overflow rule of the voxel index, the neighbour-list windows and a
SPFH bin that collects more than 65 535 pairs.  Every cloud is also run through the scan cache in shuffled, mixed waves, so each
cloud's per-wave state (digit count and A/B parity, chunk counts, tiles, raw offset, bbox grid) is checked slot by slot.
Every comparison is bit for bit (uint32 views, NaN pattern included); status codes and counts must be equal."""
import time

import numpy as np
import pytest

from quatro_b200 import synth
from quatro_b200.capi import Handle, default_params
from independent_ref import voxel_grid
from support import P4, same_bits

DEFAULT_CELL = float(np.float32(0.75) * np.float32(1.001953125))
OK, CAPACITY, OVERFLOW = 0, 3, -5
INT_MAX = 2**31 - 1


def grid_of(pts4, leaf, skip):
    """PCL's grid of the kept points, evaluated the way the library does (float32 products, int64 spans), and the refusal rule:
    (status, digits of the voxel key)."""
    p = pts4[np.isfinite(pts4[:, :3]).all(1) & ~((skip != 0) & (pts4[:, 3] < 0))][:, :3]
    if len(p) == 0:
        return OK, 0
    inv = np.float32(1.0) / np.float32(leaf)
    mn, mx = p.min(0), p.max(0)
    with np.errstate(over="ignore", invalid="ignore"):
        lo, hi, s = np.floor(mn * inv), np.floor(mx * inv), (mx - mn) * inv
    if not ((lo >= -2.0**31).all() and (hi < 2.0**31).all() and (s < 2.0**31).all()):
        return OVERFLOW, None
    trunc = [int(v) + 1 for v in s]
    div = [int(h) - int(l) + 1 for h, l in zip(hi, lo)]
    if np.prod(trunc, dtype=object) > INT_MAX or np.prod(div, dtype=object) > INT_MAX:
        return OVERFLOW, None
    span = int(np.prod(div, dtype=object))
    bits = 0
    while bits < 31 and (1 << bits) < span:
        bits += 1
    return OK, (bits + 7) >> 3


# ---- the cloud set --------------------------------------------------------------------------------------------------------------
def span_cloud(dims, rng, n_fill=3000):
    """Leaf 1: corner points in cells (0, 0, 0) and dims - 1, plus fill strictly inside: the key spans dims[0] dims[1] dims[2]."""
    d = np.asarray(dims, np.float64)
    fill = rng.uniform(0.5, d - 0.5, (n_fill, 3))
    pts = np.concatenate([[[0.5, 0.5, 0.5]], fill, [d - 0.5]])
    return P4(pts[rng.permutation(len(pts))])


def street_crop(seed, radius, shift=(0.0, 0.0, 0.0)):
    s, _, _ = synth.outdoor_pair(seed, rings=32, azimuths=900)
    s = s[np.linalg.norm(s[:, :2], axis=1) < radius].copy()
    s[:, :3] += np.asarray(shift, np.float32)
    return s


def boundary_cloud(leaf, rng):
    """Coordinates with p * inv an exact integer, one ulp either side, negative boundaries, +-0.0 and subnormals."""
    inv = np.float32(1.0) / np.float32(leaf)
    vals = []
    for k in range(-12, 13):
        b = np.float32(k) / inv
        for c in rng.permutation(np.arange(-200, 200))[:60]:   # search the float grid for an exact product
            t = np.float32(b + np.float32(c) * np.spacing(np.float32(max(abs(b), 1e-3))))
            if np.float32(t * inv) == np.float32(k):
                b = t
                break
        vals += [b, np.nextafter(b, np.float32(np.inf)), np.nextafter(b, np.float32(-np.inf))]
    vals += [0.0, -0.0, 1e-40, -1e-40, np.float32(1.4e-45), np.float32(-1.4e-45)]
    vals = np.asarray(vals, np.float32)
    pts = np.stack([rng.choice(vals, 3000), rng.choice(vals, 3000), rng.choice(vals, 3000)], 1)
    return P4(pts)


def stability_cloud(rng):
    """One voxel with 4000 points (spread over every tile and chunk of the scan) interleaved with 16 000 points of other voxels;
    random mantissas, so the float centroid depends on the summation order."""
    n = 20000
    pts = rng.uniform(0.0, 8.0, (n, 3)).astype(np.float32)
    hot = np.arange(0, n, 5)
    pts[hot] = rng.uniform(0.0, 1.0, (len(hot), 3)).astype(np.float32) * np.float32(0.999)
    cold = np.setdiff1d(np.arange(n), hot)
    pts[cold[pts[cold].max(1) < 1.0], 0] += 1.0          # only the hot points in voxel (0, 0, 0)
    return P4(pts)


def voxel_clouds():
    """(name, pts4, leaf, skip_flagged).  Built once, deterministic."""
    rng = np.random.default_rng(2024)
    C = []
    # lattice spans at each digit count (leaf 1)
    C.append(("one_voxel", P4(rng.uniform(0.1, 0.9, (500, 3))), 1.0, 1))
    for name, dims in (("span_2^8", (256, 1, 1)), ("span_2^8+1", (257, 1, 1)), ("span_2^16", (256, 256, 1)),
                       ("span_2^16+1", (65537, 1, 1)), ("span_2^24", (4096, 4096, 1)), ("span_2^24+1", (673, 257, 97)),
                       ("span_max_4_digits", (46340, 46340, 1))):
        C.append((name, span_cloud(dims, rng), 1.0, 1))
    # sizes: tiles of 2048 items, 64 chunks, one warp
    for n in (1, 63, 64, 65, 2047, 2048, 2049):
        C.append((f"n_{n}", P4(rng.uniform(-6.0, 6.0, (n, 3))), 1.0, 1))
    # sparse keeps: one kept point among NaN / flagged points, kept points only in the last of the 64 chunks
    n = 131072
    nan = P4(np.full((n, 3), np.nan))
    nan[77777, :3] = (3.2, -1.1, 0.4)
    C.append(("one_kept_among_nan", nan, 1.0, 1))
    flag = P4(rng.uniform(-5, 5, (n, 3)), w=-1.0)
    flag[n - 1, 3] = 1.0
    C.append(("one_kept_among_flagged", flag, 1.0, 1))
    last = P4(np.full((n, 3), np.nan))
    last[n - n // 64 + 5:, :3] = rng.uniform(-5, 5, (n // 64 - 5, 3))
    C.append(("kept_in_last_chunk", last, 1.0, 1))
    C.append(("stable_hot_voxel", stability_cloud(rng), 1.0, 1))
    # cell boundaries
    C.append(("boundaries_leaf_0.25", boundary_cloud(0.25, rng), 0.25, 1))
    C.append(("boundaries_leaf_1", boundary_cloud(1.0, rng), 1.0, 1))
    # the w field: -0.0 and NaN are not "flagged" (w < 0 is false), -1 is
    wf = P4(rng.uniform(-3, 3, (3000, 3)))
    wf[0::4, 3] = -0.0
    wf[1::4, 3] = np.nan
    wf[2::4, 3] = -1.0
    C.append(("w_field_skip1", wf, 1.0, 1))
    C.append(("w_field_skip0", wf, 1.0, 0))
    # far from the origin: accepted by PCL (the index is relative to the cloud's min cell)
    C.append(("x_40km_leaf_0.3", street_crop(5, 30.0, (40000.0, 0.0, 0.0)), 0.3, 1))
    C.append(("z_1.7km_leaf_0.05", street_crop(6, 8.0, (0.0, 0.0, 1700.0)), 0.05, 1))
    C.append(("utm_leaf_0.3", street_crop(7, 30.0, (5.0e5, 5.0e6, 300.0)), 0.3, 1))
    # the overflow rules
    C.append(("trunc_just_accepted_1d", P4([[0.0, 0.5, 0.5], [2147483520.0, 0.5, 0.5], [1.0e9, 0.5, 0.5]]), 1.0, 1))
    C.append(("trunc_2^31", P4([[0.5, 0.5, 0.5], [65535.5, 32767.5, 0.5], [7.5, 7.5, 0.5]]), 1.0, 1))
    C.append(("trunc_ok_floor_over", P4([[0.5, 0.5, 0.5], [1290.4, 1290.4, 1290.4], [1290.3, 0.6, 1290.2]]), 1.0, 1))
    C.append(("floor_above_int32", P4([[3.0e9, 0.5, 0.5], [3.0e9, 0.5, 0.5]]), 1.0, 1))
    C.append(("floor_below_int32", P4([[0.5, -2.5e9, 0.5]]), 1.0, 1))
    return C


# intended edge of each construction: (status, digits); None = not checked
INTENDED = {"one_voxel": (OK, 0), "span_2^8": (OK, 1), "span_2^8+1": (OK, 2), "span_2^16": (OK, 2), "span_2^16+1": (OK, 3),
            "span_2^24": (OK, 3), "span_2^24+1": (OK, 4), "span_max_4_digits": (OK, 4), "trunc_just_accepted_1d": (OK, 4),
            "trunc_2^31": (OVERFLOW, None), "trunc_ok_floor_over": (OVERFLOW, None), "floor_above_int32": (OVERFLOW, None),
            "floor_below_int32": (OVERFLOW, None), "x_40km_leaf_0.3": (OK, None), "z_1.7km_leaf_0.05": (OK, None),
            "utm_leaf_0.3": (OK, None)}


@pytest.fixture(scope="module")
def clouds():
    return voxel_clouds()


@pytest.fixture(scope="module")
def oracle_vox(clouds, oracle):
    return {name: oracle.voxelize(pts, leaf, skip) for name, pts, leaf, skip in clouds}


# ---- CPU: the constructions hit their edges, and the oracle agrees with float64 ---------------------------------------------------
def test_constructions_hit_their_edges(clouds, oracle_vox):
    seen = set()
    for name, pts, leaf, skip in clouds:
        st, digits = grid_of(pts, leaf, skip)
        assert oracle_vox[name][1] == st, name
        if name in INTENDED:
            want_st, want_d = INTENDED[name]
            assert st == want_st and (want_d is None or digits == want_d), (name, st, digits)
        if st == OK:
            seen.add(digits)
    assert seen >= {0, 1, 2, 3, 4}
    # the window between PCL's two span formulas: the truncated product is accepted, the floor-based one is not
    assert 1290 ** 3 <= INT_MAX < 1291 ** 3


def test_stability_cloud_detects_an_unstable_sort(clouds, oracle):
    """Summing the hot voxel in another order changes its centroid bits: a voxel sort that is not stable cannot pass."""
    pts = dict((c[0], c[1]) for c in clouds)["stable_hot_voxel"]
    ref, _ = oracle.voxelize(pts, 1.0, 1)
    hot = np.nonzero((pts[:, :3] < 1.0).all(1))[0]
    assert len(hot) > 2048
    perm = pts.copy()
    perm[hot] = pts[hot[np.random.default_rng(1).permutation(len(hot))]]
    alt, _ = oracle.voxelize(perm, 1.0, 1)
    assert len(alt) == len(ref) and same_bits(alt[1:], ref[1:]) and not same_bits(alt[:1], ref[:1])


@pytest.mark.parametrize("name", ["boundaries_leaf_0.25", "boundaries_leaf_1", "x_40km_leaf_0.3", "z_1.7km_leaf_0.05", "utm_leaf_0.3",
                                  "span_2^24+1", "trunc_just_accepted_1d"])
def test_oracle_voxels_match_float64(clouds, oracle_vox, name):
    pts, leaf, skip = next((c[1], c[2], c[3]) for c in clouds if c[0] == name)
    ref, st = oracle_vox[name]
    assert st == OK
    kept = pts[np.isfinite(pts[:, :3]).all(1) & ~((skip != 0) & (pts[:, 3] < 0))]
    cent, idx, uniq = voxel_grid(kept[:, :3], leaf)
    assert len(ref) == len(uniq)
    counts = np.bincount(np.searchsorted(uniq, idx), minlength=len(uniq))
    tol = 4 * counts[:, None] * np.finfo(np.float32).eps * (np.abs(kept[:, :3]).max() + 1e-30)
    assert (np.abs(ref[:, :3] - cent) <= tol).all()


# ---- GPU: single calls, then mixed waves through the scan cache -------------------------------------------------------------------
def _single(h, pts, leaf, skip):
    got, st = h.voxelize(pts, leaf, skip)
    return got, st


@pytest.mark.gpu
def test_voxelize_adversarial_single(handle, clouds, oracle_vox):
    bad = []
    for name, pts, leaf, skip in clouds:
        ref, st_r = oracle_vox[name]
        got, st_g = _single(handle, pts, leaf, skip)
        if st_g != st_r or not same_bits(got, ref):
            bad.append(f"{name}: status {st_g} vs {st_r}, {len(got)} vs {len(ref)} points")
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("R", [131072, 100003])
def test_voxelize_full_scan_and_index_width(oracle, R):
    """n = max_raw_points for a power-of-two and a non-power-of-two R (the point index takes clog2(R) key bits)."""
    rng = np.random.default_rng(R)
    pts = P4(rng.uniform(0.0, 1.0, (R, 3)) * np.array([10.0, 10.0, 2.0]))
    pts[rng.random(R) < 0.2, 3] = -1.0
    with Handle(max_batch_slots=2, max_raw_points=R) as h:
        for skip in (1, 0):
            ref, st_r = oracle.voxelize(pts, 0.3, skip)
            got, st_g = h.voxelize(pts, 0.3, skip)
            assert st_g == st_r == OK and same_bits(got, ref)


def _cache_groups(clouds):
    groups = {}
    for i, (name, pts, leaf, skip) in enumerate(clouds):
        groups.setdefault((leaf, skip), []).append(i)
    return groups


@pytest.mark.gpu
@pytest.mark.parametrize("slots", [2, 8])
def test_mixed_waves_through_the_scan_cache(clouds, oracle_vox, oracle, slots):
    """Every cloud in shuffled waves with the others of its (leaf, skip_flagged), plus a CAPACITY_EXCEEDED cloud: each slot equals the
    single-cloud call and the oracle (voxels, normals, descriptors), whatever its neighbours in the wave do."""
    rng = np.random.default_rng(slots)
    cap_cloud = P4(np.stack(np.meshgrid(np.arange(130), np.arange(130), np.arange(1)), -1).reshape(-1, 3) + 0.5)  # 16 900 voxels
    extra = [("capacity_exceeded", cap_cloud, 1.0, 1)]
    allc = clouds + extra
    with Handle(max_batch_slots=slots) as h:
        V = h.cfg.max_voxel_points
        singles = {name: _single(h, pts, leaf, skip) for name, pts, leaf, skip in allc}
        assert singles["capacity_exceeded"][1] == CAPACITY and len(singles["capacity_exceeded"][0]) == V
        h.cache_reserve(len(allc))
        bad = []
        for (leaf, skip), idx in _cache_groups(allc).items():
            idx = [idx[i] for i in rng.permutation(len(idx))]
            p = default_params()
            p.voxel_size, p.skip_flagged = leaf, skip
            h.cache_scans([allc[i][1] for i in idx], idx, p)
            for i in idx:
                name = allc[i][0]
                got, st = singles[name]
                vox, nrm, desc = h.cache_read(i)
                want = got if st in (OK, CAPACITY) else got[:0]
                if not same_bits(vox, want):
                    bad.append(f"{name}: cache {len(vox)} points vs single call {len(want)} (status {st})")
                    continue
                if st == OK and name in oracle_vox:
                    ref, st_r = oracle_vox[name]
                    assert st_r == OK and same_bits(vox, ref), name
                    if len(ref) <= 6000:
                        n_ref, d_ref = oracle.compute_fpfh(ref, p.normal_radius, p.fpfh_radius, DEFAULT_CELL)
                        if not (same_bits(nrm, n_ref, nan_equal=True) and same_bits(desc, d_ref)):
                            bad.append(f"{name}: normals / descriptors differ from the oracle")
        assert not bad, "\n".join(bad)


# ---- normals / FPFH edges -----------------------------------------------------------------------------------------------------------
def star_cloud(k, rng, centre=(2.0, -1.0, 0.5)):
    """A centre point with exactly k neighbours within 0.75 (itself included), each in its own 0.02 m voxel, and a sparse
    background beyond the radius."""
    c = np.asarray(centre, np.float64)
    d = rng.normal(size=(2 * k, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    inner = c + d * rng.uniform(0.15, 0.7, (2 * k, 1))
    far = c + rng.uniform(-3.0, 3.0, (400, 3))
    far = far[np.linalg.norm(far - c, axis=1) > 0.8]
    pts = P4(np.concatenate([[c], inner, far]))
    _, first = np.unique(np.floor(pts[:, :3] * np.float32(50.0)), axis=0, return_index=True)
    keep = np.sort(first)                                   # one point per 0.02 m voxel
    inside = keep[keep <= 2 * k]
    return pts[np.concatenate([inside[:k], keep[keep > 2 * k]])]


def fpfh_clouds():
    rng = np.random.default_rng(77)
    C = [(f"nbrs_{k}", star_cloud(k, rng)) for k in (64, 65, 80, 81, 128, 129)]
    line = np.stack([np.arange(12) * 0.1, np.zeros(12), np.full(12, 0.3)], 1)
    pair = np.array([[5.0, 5.0, 1.0], [5.3, 5.0, 1.0]])
    C.append(("collinear_and_two_point", P4(np.concatenate([line, pair, rng.uniform(-8, 8, (300, 3))]))))
    C.append(("x_40km", street_crop(8, 25.0, (40000.0, 0.0, 0.0))))
    C.append(("beyond_lattice", street_crop(9, 25.0, (120000.0, 0.0, 0.0))))
    return C


def test_fpfh_constructions_hit_their_neighbour_counts(oracle):
    leaf = 0.02
    for name, pts in fpfh_clouds()[:6]:
        k = int(name.split("_")[1])
        vox, st = oracle.voxelize(pts, leaf, 1)
        assert st == OK and len(vox) == len(pts)              # one point per voxel: the centroids are the points
        q = int(np.nonzero((vox[:, :3] == pts[0, :3]).all(1))[0][0])
        idx, _ = oracle.neighbors(vox, DEFAULT_CELL, q, 0.75)
        assert len(idx) == k, (name, len(idx))


@pytest.mark.gpu
def test_fpfh_edges_in_mixed_waves(oracle):
    rng = np.random.default_rng(3)
    C = fpfh_clouds()
    order = rng.permutation(len(C))
    with Handle(max_batch_slots=2) as h:
        h.cache_reserve(len(C))
        bad = []
        for leaf, names in ((0.02, [n for n, _ in C[:7]]), (0.3, ["x_40km", "beyond_lattice"])):
            p = default_params()
            p.voxel_size = leaf
            sel = [i for i in order if C[i][0] in names]
            h.cache_scans([C[i][1] for i in sel], sel, p)
            for i in sel:
                name, pts = C[i]
                ref, st = oracle.voxelize(pts, leaf, 1)
                assert st == OK
                vox, nrm, desc = h.cache_read(i)
                n_ref, d_ref = oracle.compute_fpfh(ref, p.normal_radius, p.fpfh_radius, DEFAULT_CELL)
                if not (same_bits(vox, ref) and same_bits(nrm, n_ref, nan_equal=True) and same_bits(desc, d_ref)):
                    bad.append(name)
                if name == "beyond_lattice":
                    assert np.isnan(nrm).all() and len(vox) > 100
                if name == "collinear_and_two_point":
                    assert np.isnan(n_ref[:, 0]).any()
        assert not bad, bad
        # coincident duplicates (d2 = 0 skips the pair) straight through qb200_compute_fpfh: a voxel filter would merge them
        base = star_cloud(90, rng)
        dup = np.concatenate([base, base[::3], base[:5]])
        n_ref, d_ref = oracle.compute_fpfh(dup, 0.5, 0.75, DEFAULT_CELL)
        n_got, d_got = h.compute_fpfh(dup, 0.5, 0.75, DEFAULT_CELL)
        assert same_bits(n_got, n_ref, nan_equal=True) and same_bits(d_got, d_ref)


def wrap_cloud():
    """65 540 points of one plane (z = 1): a query point q, 65 537 coincident copies of B and two copies of C, all within 0.43 m of
    each other.  The normals are the plane's; every (q, B) pair has the same Darboux features, so q's SPFH has a bin with 65 537
    (+ C) pairs.  Coincident copies keep the oracle's pair-feature work small (d = 0 is skipped)."""
    q, b, c = (0.0, 0.0, 1.0), (0.3, 0.0, 1.0), (0.0, 0.3, 1.0)
    return P4(np.array([q] + [b] * 65537 + [c] * 2))


@pytest.fixture(scope="module")
def wrap_ref(oracle):
    t0 = time.perf_counter()
    n, d, s = oracle.compute_fpfh(wrap_cloud(), 0.5, 0.75, DEFAULT_CELL, want_spfh=True)
    return n, d, s, time.perf_counter() - t0


def test_spfh_bin_count_above_16_bits(wrap_ref):
    _, _, spfh, secs = wrap_ref
    incr = np.float32(100.0) / np.float32(len(wrap_cloud()) - 1)
    assert np.isfinite(spfh).all()
    # the increment is summed once per pair: a bin holding 100 * 65 537 / 65 539 has more than 65 535 pairs
    assert spfh[0].max() > np.float32(65535.5) * incr, spfh[0].max() / incr
    assert secs < 60.0, secs


@pytest.mark.gpu
def test_spfh_counts_beyond_16_bits(wrap_ref):
    n_ref, d_ref, _, _ = wrap_ref
    with Handle(max_batch_slots=1, max_voxel_points=131072) as h:
        n_got, d_got = h.compute_fpfh(wrap_cloud(), 0.5, 0.75, DEFAULT_CELL)
    assert same_bits(n_got, n_ref, nan_equal=True)
    diff = (d_got.view(np.uint32) != d_ref.view(np.uint32)).any(1)
    assert not diff.any(), f"{diff.sum()} descriptors differ (first {np.nonzero(diff)[0][:5]})"


# ---- end to end ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shift", [(30000.0, 0.0, 0.0), (0.0, 0.0, 1700.0)])
def test_far_street_pair_end_to_end(oracle, shift):
    """A street pair moved 30 km in x or 1.7 km in z, voxelised at 0.05 m: the records and the correspondences equal the oracle's."""
    src, tgt, _ = synth.outdoor_pair(12, rings=32, azimuths=900)
    keep_s, keep_t = np.linalg.norm(src[:, :2], axis=1) < 15.0, np.linalg.norm(tgt[:, :2], axis=1) < 15.0
    src, tgt = src[keep_s].copy(), tgt[keep_t].copy()
    src[:, :3] += np.asarray(shift, np.float32)
    tgt[:, :3] += np.asarray(shift, np.float32)
    p = default_params()
    p.voxel_size = 0.05
    r_ref, st_r = oracle.register_pair(src, tgt, p)
    sv, _ = oracle.voxelize(src, p.voxel_size, p.skip_flagged)
    tv, _ = oracle.voxelize(tgt, p.voxel_size, p.skip_flagged)
    corr_ref, _, _, _ = oracle.match_and_pack(sv, tv, p)
    with Handle(max_batch_slots=2, max_voxel_points=32768) as h:
        out, lists = h.register_batch_lists([(src, tgt)], p)
    g = out[0]
    assert st_r == OK and g["valid"] == 1 and g["status"] == 0
    for k in ("n_src_vox", "n_tgt_vox", "n_mutual", "n_corr", "n_edges", "max_core", "clique_size", "gnc_iters", "n_rot_inliers",
              "n_final_inliers"):
        assert g[k] == getattr(r_ref, k), (k, g[k], getattr(r_ref, k))
    assert np.allclose(np.asarray(g["T"]).reshape(4, 4).T, r_ref.matrix(), atol=1e-9)
    assert np.array_equal(np.asarray(lists[0]["corr"]).reshape(-1, 2), corr_ref)
