"""K1, the voxel filter, against the float32 restatement of pcl::VoxelGrid<PointXYZ>::applyFilter in independent_ref.py, on clouds
built to sit on the stage's decisions:
  - PCL's float subtraction ijk = int(floor(p * inv) - float(min_b)): cells 2^24 and more from the cloud's minimum cell that PCL
    merges, a row whose last cell aliases into the next row's first voxel, and largest indices at INT_MAX - 1, INT_MAX and INT_MAX + 1;
  - the summation order: hundreds of order-sensitive voxels whose points are spread over every bbox chunk and several sort tiles, at
    key spans of 1 to 4 digits (both result arrays of the voxel sort);
  - the centroid arithmetic: counts 1, 2, 3, 7 and 2^k +- 1, sums that overflow to +-inf, zero sums, subnormals;
  - leaves with inexact reciprocals, powers of two, FLT_MAX and inf, leaves whose reciprocal overflows, exact cell boundaries +- 1 ulp;
  - the bbox reduction: the extremes alone in the first, middle or last chunk, extremes at +-0.0 and subnormals, n = 1 ... 65, one kept
    point among NaN or flagged records.
On the CPU every construction is checked to reach its edge, the restatement equals the oracle bit for bit and, away from the float
subtraction, the float64 voxel_grid.  On the GPU qb200_voxelize, qb200_voxelize_batch_each and qb200_describe_batch_each equal the
restatement bit for bit: status, count and centroids (or the kept records of a refused cloud)."""
from collections import namedtuple

import numpy as np
import pytest

from quatro_b200.capi import MEM_DEVICE, MEM_HOST
from independent_ref import INT32_MAX, VOX_OK, VOX_OVERFLOW, voxel_grid, voxel_grid_pcl32
from support import P4, _host, device_copies, make_handle, make_params, same_bits

F32 = np.float32
CAPACITY = 3
V_DEFAULT = 16384                     # max_voxel_points of a default handle

Cloud = namedtuple("Cloud", "name family pts leaf skip want")


# ---- builders -----------------------------------------------------------------------------------------------------------------------
def cell_point(F, inv):
    """A float32 coordinate p with floor(p * inv) == F in float32, or None when no float lands in that cell."""
    if int(F32(F)) != F:
        return None
    F = F32(F)
    p = F32((float(F) + 0.5) / float(inv))
    for _ in range(200):
        f = np.floor(p * inv)
        if f == F:
            return p
        p = np.nextafter(p, F32(np.inf) if f < F else F32(-np.inf))
    return None


def merge_cloud(leaf, lo_target, plan, rng):
    """x cells that PCL's float subtraction merges.  A point in cell lo (near lo_target) sets min_b; for each (e, k) of the plan, k
    distinct cells lo + D with D in [2^e, 2^(e+1)) that all round to one even-mantissa value E (the ties at E +- s/2 go to E, s the
    float spacing there).  Every voxel gets 3 points with random y, z inside cell 0.  Returns (pts4, merged cell counts)."""
    inv = F32(1) / F32(leaf)
    for t in range(4000):
        lo_p = cell_point(lo_target - 2 * t, inv)
        if lo_p is not None:
            break
    lo = int(np.floor(lo_p * inv))
    xs, merged = [lo_p], []
    for i, (e, k) in enumerate(plan):
        s = 2 ** (e - 23)
        E = 2 ** e + 2 * s * (1000 + 37 * i)
        while True:
            D = [E - s // 2 + j for j in range(k)]
            ps = [cell_point(lo + d, inv) for d in D]
            if all(p is not None for p in ps) and {int(F32(d)) for d in D} == {E}:
                break
            E += 2 * s
        xs += ps
        merged.append(k)
    xs = np.repeat(np.asarray(xs, np.float32), 3)
    yz = (F32(leaf) * rng.uniform(0.05, 0.95, (len(xs), 2))).astype(np.float32)
    pts = P4(np.column_stack([xs, yz]))
    return pts[rng.permutation(len(pts))], merged


def alias_search(T):
    """(q, r0, D0, c) for a leaf-1 cloud whose largest PCL index is T: x cells -c ... D0 - c with fl(D0) = D0 + r0 (rounded up), y cells
    0 ... q - 1; div_b0 * q = T + 1 - r0 <= INT_MAX."""
    for q in range(2, 4096):
        for r0 in range(1, 33):
            P = T + 1 - r0
            if P % q or P > INT32_MAX:
                continue
            D0 = P // q - 1
            if D0 < 2 ** 24 or int(F32(D0)) - D0 != r0:
                continue
            c = next((c for c in range(1, 300) if int(F32(D0 - c)) == D0 - c), None)
            if c is not None:
                return q, r0, D0, c
    raise AssertionError(T)


def alias_cloud(q, r0, D0, c, rng, fill=0):
    """Leaf 1.  x from cell -c to cell D0 - c, y from cell 0 to q - 1 with the extremes 0.1 inside the bbox (so PCL's truncated spans
    stay below div_b).  The last x cell of row 0 gets ijk0 = fl(D0) = D0 + r0 and so PCL's index of cell (r0 - 1 - c, row 1): PCL
    merges the two, the cells are distinct.  `fill` more points in each of the two aliased cells."""
    lo, hi = F32(-c), F32(D0 - c)
    A = [lo + F32(0.9), 0.9, 0.5]                    # min corner
    B = [hi, q - 1 + 0.1, 0.5]                       # max corner: the largest index
    C = [[hi, y, 0.5] for y in rng.uniform(0.91, 0.99, fill + 1)]
    Dp = [[x, y, 0.5] for x, y in zip(F32(r0 - 1 - c) + rng.uniform(0.91, 0.99, fill + 1), rng.uniform(1.01, 1.09, fill + 1))]
    pts = P4(np.asarray([A, B] + C + Dp, np.float64))
    return pts[rng.permutation(len(pts))]


def order_cloud(dims, n_vox, per_vox, rng):
    """Leaf 1.  n_vox voxels of the lattice `dims` (its two corners among them), per_vox points each with random mantissas; point i
    belongs to voxel i mod n_vox, so every voxel has points in each of the 64 bbox chunks and in every 2048-item sort tile."""
    dims = np.asarray(dims)
    total = int(np.prod(dims))
    lin = np.concatenate([[0, total - 1], 1 + rng.choice(total - 2, n_vox - 2, replace=False)]) if total > n_vox else \
        np.arange(total)
    cells = np.stack(np.unravel_index(lin, dims[::-1]), 1)[:, ::-1].astype(np.float64)   # (i, j, k) with i fastest
    n = len(cells) * per_vox
    frac = rng.uniform(0.01, 0.99, (n, 3))
    return P4(cells[np.arange(n) % len(cells)] + frac)


def boundary_cloud(leaf, rng, n=3000):
    """Coordinates with p * inv an exact integer k (k = -12 ... 12) and one ulp either side."""
    inv = F32(1) / F32(leaf)
    vals = []
    for k in range(-12, 13):
        b = F32(F32(k) / inv)
        for c in range(-300, 301):                          # the float nearest k / inv whose product is exactly k
            t = F32(b + F32(c) * np.spacing(F32(max(abs(b), 1e-3))))
            if F32(t * inv) == F32(k):
                b = t
                break
        vals += [b, np.nextafter(b, F32(np.inf)), np.nextafter(b, F32(-np.inf))]
    vals = np.asarray(vals, np.float32)
    return P4(np.stack([rng.choice(vals, n), rng.choice(vals, n), rng.choice(vals, n)], 1))


def extremes_cloud(where, rng, n=6400):
    """n points in [-5, 5]^3 and the six axis extremes (+-9.5) all in chunk `where` (0, 32 or 63) of the 64 bbox chunks."""
    pts = P4(rng.uniform(-5.0, 5.0, (n, 3)))
    cs = n // 64
    for a in range(3):
        for s, sign in enumerate((-1.0, 1.0)):
            i = where * cs + 7 * (2 * a + s) + 3
            pts[i, :3] = rng.uniform(-5.0, 5.0, 3)
            pts[i, a] = sign * 9.5
    return pts


def build_clouds():
    rng = np.random.default_rng(20261018)
    C = []

    def add(name, family, pts, leaf, skip=1, **want):
        C.append(Cloud(name, family, np.ascontiguousarray(pts, np.float32), float(leaf), skip, want))

    # -- PCL's float subtraction: x from -3e7 to 2.5e7 at a 1 m leaf and from -20 km to 15 km at 1 mm, y = z = 0.5
    add("table_leaf_1", "float_sub", P4([[x, 0.5, 0.5] for x in (-3e7, 0.5, 1.0, 25000006.0, 25000010.0)]), 1.0, voxels=3, cells=5)
    add("table_leaf_1e-3", "float_sub", P4([[x, 0.5, 0.5] for x in (-20000.0, 15000.0, 15000.001, 15000.002)]), 1e-3, voxels=3,
        cells=4)
    for leaf in (1.0, 0.3, 1e-2, 1e-3):
        pts, merged = merge_cloud(leaf, -(2 ** 24) - 2 ** 22, [(24, 2), (24, 3), (25, 4)], rng)
        add(f"straddle_leaf_{leaf:g}", "float_sub", pts, leaf, merged=merged)
    q, r0, D0, c = alias_search(2 * (2 ** 24 + 2 ** 22 + 4))     # x cells D0 = 2^24 + 2^22 + 3 apart: fl(D0) = D0 + 1
    assert q == 2 and r0 == 1
    add("row_alias_dy_2", "float_sub", alias_cloud(q, r0, D0, c, rng, fill=20), 1.0, alias=True)
    for name, T in (("top_index_int_max-1", INT32_MAX - 1), ("top_index_int_max", INT32_MAX), ("top_index_int_max+1", INT32_MAX + 1)):
        q, r0, D0, c = alias_search(T)
        pts = alias_cloud(q, r0, D0, c, rng, fill=5)
        if T > INT32_MAX:
            add(name, "float_sub", pts, 1.0, status=VOX_OVERFLOW, refused="top_index", top_index=T)
        else:
            add(name, "float_sub", pts, 1.0, status=VOX_OK, top_index=T, alias=True)

    # -- summation order: hundreds of order-sensitive voxels at key spans of 1 ... 4 digits
    for dims, digits in (((256, 1, 1), 1), ((65536, 1, 1), 2), ((4096, 4096, 1), 3), ((46340, 46340, 1), 4)):
        add(f"order_{digits}_digits", "order", order_cloud(dims, 200, 100, rng), 1.0, digits=digits)
    add("order_1_digit_small_voxels", "order", order_cloud((13, 7, 2), 182, 20, rng), 1.0, digits=1)

    # -- centroid arithmetic
    counts = [1, 2, 3, 7] + [2 ** k + d for k in (4, 5, 6, 7, 8, 10, 12) for d in (-1, 1)]
    cells = np.repeat(np.arange(len(counts)) * 2.0, counts)
    pts = P4(np.column_stack([cells, np.zeros_like(cells), np.zeros_like(cells)]) + rng.uniform(0.001, 0.999, (len(cells), 3)))
    add("counts", "centroid", pts[rng.permutation(len(pts))], 1.0, counts=sorted(counts))
    add("overflow_to_inf", "centroid", P4([[2.5e38, -2.5e38, 0.5], [2.6e38, -2.6e38, 0.25], [1.0e38, -1.0e38, 0.5],
                                           [2.7e38, -2.7e38, 0.75], [1.5e38, -1.5e38, 0.5]]), 1e38, inf=True)
    z = np.array([[1.5, -2.25, -0.0], [-1.5, 2.25, -0.0], [-0.0, -0.0, -0.0], [1.0e30, 1.0, -0.0], [-1.0e30, -1.0, -0.0]])
    add("cancel_to_zero_leaf_inf", "centroid", P4(z), np.inf, zero=True)
    add("negative_zeros", "centroid", P4([[-0.0, -0.0, -0.0]] * 5 + [[0.5, -0.0, 0.5]] * 3), 1.0, zero=True)
    sub = F32([1e-40, 3e-41, 1.4e-45, -0.0, 2e-39, 1.1754942e-38])
    pts = P4(np.stack([rng.choice(sub, 400), rng.choice(sub, 400), rng.choice(sub, 400)], 1))
    pts[::3, 1] = -pts[::3, 1] - F32(1e-40)                                   # negative subnormals: cell -1
    add("subnormals", "centroid", pts, 1.0, subnormal=True)

    # -- leaves
    for leaf in (0.3, 0.1, 1.0 / 3.0, 0.22, 0.25, 0.5, 2.0, 0.125):
        add(f"boundaries_leaf_{leaf:.4g}", "leaf", boundary_cloud(leaf, rng), leaf, boundaries=True)
    add("leaf_flt_max", "leaf", P4(rng.uniform(0.0, 100.0, (500, 3))), float(np.finfo(np.float32).max), voxels=1)
    add("leaf_inf_recip", "leaf", P4(rng.uniform(-1.0, 1.0, (50, 3))), 1e-45, status=VOX_OVERFLOW)
    add("leaf_floor_overflow", "leaf", P4([[5.0, 5.0, 5.0], [5.0, 5.0, 5.0]]), 1e-30, status=VOX_OVERFLOW, refused="floor")

    # -- the bbox reduction
    for where, name in ((0, "first"), (32, "middle"), (63, "last")):
        add(f"extremes_in_{name}_chunk", "bbox", extremes_cloud(where, rng), 1.0, lo=[-10, -10, -10], hi=[9, 9, 9])
    pz = P4(rng.uniform(0.0, 3.0, (300, 3)))
    pz[17, 0], pz[150, 0], pz[299, 1] = -0.0, 0.0, -0.0
    add("extremes_signed_zero", "bbox", pz, 1.0, lo=[0, 0, 0], hi=[2, 2, 2])
    ps = P4(rng.uniform(-3.0, -0.01, (300, 3)))
    ps[5, 0], ps[250, 1], ps[100, 2] = 1e-40, 1.4e-45, -1e-40
    ps[101, 2] = -1e-40
    ps[101, 0] = -3.5
    add("extremes_subnormal", "bbox", ps, 1.0, lo=[-4, -3, -3], hi=[0, 0, -1])
    for n in range(1, 66):
        pts = P4(rng.uniform(-2.0, 2.0, (n, 3)))
        pts[rng.random(n) < 0.2, 3] = -1.0
        add(f"n_{n}", "bbox", pts, 0.5, skip=n % 2)
    nan = P4(np.full((8192, 3), np.nan))
    nan[4321, :3] = (3.2, -1.1, 0.4)
    add("one_kept_among_nan", "bbox", nan, 1.0, voxels=1)
    flag = P4(rng.uniform(-5, 5, (8192, 3)), w=-1.0)
    flag[8191, 3] = 1.0
    add("one_kept_among_flagged", "bbox", flag, 1.0, voxels=1)
    return C


CLOUDS = build_clouds()
BY_NAME = {c.name: c for c in CLOUDS}
NAMES = [c.name for c in CLOUDS]


def capacity_cloud(rng):
    """130 x 130 voxels of three points each: 16 900 voxels, above a default handle's max_voxel_points."""
    g = np.stack(np.meshgrid(np.arange(130), np.arange(130), np.arange(1), indexing="ij"), -1).reshape(-1, 3).astype(np.float64)
    pts = P4(np.repeat(g, 3, axis=0) + rng.uniform(0.001, 0.999, (3 * len(g), 3)))
    return pts[rng.permutation(len(pts))]


@pytest.fixture(scope="module")
def restated():
    return {c.name: voxel_grid_pcl32(c.pts, c.leaf, c.skip) for c in CLOUDS}


def _digits(top_index):
    return (int(top_index).bit_length() + 7) >> 3


def _kept(c):
    keep = np.isfinite(c.pts[:, :3]).all(1)
    if c.skip:
        keep &= ~(c.pts[:, 3] < 0)
    return c.pts[keep]


def _cells(c):
    """Per kept point its (floor(x * inv), floor(y * inv), floor(z * inv)) cell, as the integer subtraction would key it."""
    inv = F32(1) / F32(c.leaf)
    return np.floor(_kept(c)[:, :3] * inv).astype(np.int64)


def _merges(c, grid):
    """Per PCL voxel the number of distinct cells among its points."""
    cells = _cells(c)
    return [len({tuple(v) for v in cells[grid["order"][s:s + n]]}) for s, n in zip(grid["start"], grid["counts"])]


# ---- CPU: the constructions reach their edges -------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_construction_hits_its_edge(restated, name):
    c = BY_NAME[name]
    out, st, g = restated[name]
    w = c.want
    assert st == w.get("status", VOX_OK), (st, g["refused"])
    if "refused" in w:
        assert g["refused"] == w["refused"]
    if "top_index" in w:
        assert g["top_index"] == w["top_index"]
        assert g["div_b"][0] * g["div_b"][1] * g["div_b"][2] <= INT32_MAX        # only the largest index can refuse it
        assert g["span"][0] * g["span"][1] * g["span"][2] <= INT32_MAX
        assert _digits(min(g["top_index"], INT32_MAX)) == 4
    if st != VOX_OK:
        assert same_bits(out, _kept(c))                                         # PCL's pass-through of the kept records
        return
    merges = _merges(c, g)
    if c.family == "float_sub":
        exact = (_cells(c) - np.asarray(g["min_b"])) @ np.asarray([1, g["div_b"][0], g["div_b"][0] * g["div_b"][1]])
        assert (exact != g["idx"]).any()                                        # PCL's float subtraction rounds somewhere
        assert len(out) < len({tuple(v) for v in _cells(c)})                    # and merges cells
    else:
        assert max(merges) == 1                                                 # every other family keeps its cells apart
    if "voxels" in w:
        assert len(out) == w["voxels"]
    if "cells" in w:
        assert len({tuple(v) for v in _cells(c)}) == w["cells"]
    if "merged" in w:
        assert sorted(m for m in merges if m > 1) == sorted(w["merged"])
    if w.get("alias"):
        rows = [len({tuple(v) for v in _cells(c)[g["order"][s:s + n]][:, 1:]}) for s, n in zip(g["start"], g["counts"])]
        assert max(rows) == 2                                                   # one voxel holds points of two y rows
        assert g["top"][0] >= g["div_b"][0]                                     # the row's last ijk0 is div_b0 or more
    if "digits" in w:
        assert _digits(g["top_index"]) == w["digits"]
        assert len(out) >= 182 and g["counts"].min() >= 20
    if "counts" in w:
        assert sorted(g["counts"].tolist()) == w["counts"]
    if w.get("inf"):
        assert np.isposinf(out[:, 0]).any() and np.isneginf(out[:, 1]).any() and np.isfinite(out[:, 2]).all()
    if w.get("zero"):
        zeros = out[:, :3][out[:, :3] == 0]
        assert len(zeros) and not np.signbit(zeros).any()                       # +0.0 from the +0.0 accumulator
    if w.get("subnormal"):
        tiny = np.abs(out[:, :3])
        assert ((tiny > 0) & (tiny < np.finfo(np.float32).tiny)).any() and g["lo"][1] == -1
    if w.get("boundaries"):
        p = _kept(c)[:, :3]
        exact = (p * g["inv"]) == np.round(p * g["inv"])
        assert exact.sum() > 100 and len(out) > 100
    if "lo" in w:
        assert g["lo"].tolist() == w["lo"] and g["hi"].tolist() == w["hi"]


def test_families_cover_the_sort_parities(restated):
    """The order clouds reach 1, 2, 3 and 4 key digits: results in both of the voxel sort's arrays (B after an odd count)."""
    digits = {_digits(restated[c.name][2]["top_index"]) for c in CLOUDS if c.family == "order"}
    assert digits == {1, 2, 3, 4}


@pytest.mark.parametrize("name", [c.name for c in CLOUDS if c.family == "order"] + ["counts"])
def test_any_other_order_changes_the_bits(restated, name):
    """Summing a voxel's points in another order changes its centroid's bits: reversed, rotated by one, shuffled, or pairwise."""
    c = BY_NAME[name]
    out, st, g = restated[name]
    kept = _kept(c)
    xyz = kept[:, :3][g["order"]]
    changed = np.zeros(len(out), bool)
    for how in ("reverse", "rotate", "shuffle", "pairwise"):
        sums = np.zeros((len(out), 3), np.float32)
        rng = np.random.default_rng(7)
        for v, (s, n) in enumerate(zip(g["start"], g["counts"])):
            seg = xyz[s:s + n]
            if how == "pairwise":
                sums[v] = np.ascontiguousarray(seg.T).sum(1, dtype=np.float32)   # numpy's pairwise summation
                continue
            seg = seg[::-1] if how == "reverse" else np.roll(seg, -1, 0) if how == "rotate" else seg[rng.permutation(n)]
            sums[v] = np.add.accumulate(np.concatenate([np.zeros((1, 3), np.float32), seg]), 0, dtype=np.float32)[-1]
        alt = sums / g["counts"].astype(np.float32)[:, None]
        diff = (alt.view(np.uint32) != out[:, :3].view(np.uint32)).any(1)
        many = g["counts"] >= 8
        assert diff[many].mean() > 0.5, (how, diff[many].mean())
        changed |= diff
    assert changed[g["counts"] >= 8].all()


# ---- CPU: the restatement against the oracle and the float64 reference ------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_restatement_equals_the_oracle(restated, oracle, name):
    c = BY_NAME[name]
    out, st, _ = restated[name]
    ref, st_o = oracle.voxelize(c.pts, c.leaf, c.skip)
    assert st_o == st and len(ref) == len(out) and same_bits(ref, out)


def test_restatement_equals_the_oracle_beyond_capacity(oracle):
    pts = capacity_cloud(np.random.default_rng(11))
    out, st, _ = voxel_grid_pcl32(pts, 1.0, 1)
    assert st == VOX_OK and len(out) == 16900
    ref, st_o = oracle.voxelize(pts, 1.0, 1, cap=V_DEFAULT)
    assert st_o == CAPACITY and same_bits(ref, out[:V_DEFAULT])


@pytest.mark.parametrize("name", [c.name for c in CLOUDS if c.family != "float_sub"])
def test_restatement_matches_float64(restated, name):
    """Same voxels as the float64 voxel_grid (integer subtraction, float64 sums), centroids within 2 n eps of the float64 mean, or
    infinite where the float64 sum passes FLT_MAX."""
    c = BY_NAME[name]
    out, st, g = restated[name]
    if st != VOX_OK or not np.isfinite(g["inv"]) or g["inv"] == 0:
        pytest.skip("refused, or a leaf without a finite non-zero reciprocal")
    kept = _kept(c)[:, :3]
    cent, idx, uniq = voxel_grid(kept, c.leaf)
    assert len(uniq) == len(out)
    # membership: the same partition of the kept points
    assert (np.searchsorted(uniq, idx) == np.searchsorted(g["uniq"], g["idx"])).all()
    counts = g["counts"][:, None].astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        tol = 2 * counts * np.finfo(np.float32).eps * np.maximum(np.abs(cent), np.finfo(np.float32).tiny) + 2.0 ** -149 * counts
        ok = (np.abs(out[:, :3] - cent) <= tol) | (np.isinf(out[:, :3]) & (np.abs(cent * counts) > np.finfo(np.float32).max))
    assert ok.all()


# ---- GPU --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_device_equals_restatement(handle, restated, name):
    c = BY_NAME[name]
    got, st = handle.voxelize(c.pts, c.leaf, c.skip)
    out, st_r, _ = restated[name]
    assert st == st_r and len(got) == len(out), (st, st_r, len(got), len(out))
    assert same_bits(got, out)


@pytest.mark.gpu
def test_device_capacity_exceeded_gives_the_first_centroids(handle):
    pts = capacity_cloud(np.random.default_rng(11))
    out, _, _ = voxel_grid_pcl32(pts, 1.0, 1)
    got, st = handle.voxelize(pts, 1.0, 1)
    assert handle.cfg.max_voxel_points == V_DEFAULT and st == CAPACITY and len(got) == V_DEFAULT
    assert same_bits(got, out[:V_DEFAULT])


WAVE_CFG = dict(max_batch_slots=8, max_raw_points=65536)
KINDS = [(k, d) for k in (MEM_HOST, MEM_DEVICE) for d in (MEM_HOST, MEM_DEVICE)]


@pytest.fixture(scope="module")
def wave_scans():
    """Every cloud (and the capacity cloud) in one shuffled batch, each with its own leaf and skip_flagged."""
    cap = Cloud("capacity_exceeded", "capacity", capacity_cloud(np.random.default_rng(11)), 1.0, 1, {})
    allc = CLOUDS + [cap]
    order = np.random.default_rng(5).permutation(len(allc))
    return [allc[i] for i in order]


@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 4])
def test_batch_wave_equals_restatement(restated, wave_scans, lanes):
    refs = [restated[c.name] if c.name in restated else voxel_grid_pcl32(c.pts, c.leaf, c.skip) for c in wave_scans]
    params = [make_params(voxel_size=c.leaf, skip_flagged=c.skip) for c in wave_scans]
    scans = [c.pts for c in wave_scans]
    with make_handle(lanes, **WAVE_CFG) as h:
        V = h.cfg.max_voxel_points
        dev, keep = device_copies(scans)
        for kind, dest in KINDS:
            per_scan, counts, status = h.voxelize_batch_each(dev if kind == MEM_DEVICE else scans, params, kind, dest)
            bad = []
            for c, ref, v, n, st in zip(wave_scans, refs, per_scan, counts, status):
                out, st_r, _ = ref
                want_st = CAPACITY if st_r == VOX_OK and len(out) > V else st_r
                want_n = min(len(out), V) if st_r == VOX_OK else len(out)
                got = _host(v)
                if st != want_st or n != want_n or not same_bits(got, out[:min(want_n, V)]):
                    bad.append(f"{c.name}: status {st} vs {want_st}, count {n} vs {want_n}")
            assert not bad, (kind, dest, bad)


@pytest.mark.gpu
def test_describe_batch_vox4_equals_restatement(restated):
    """The describe call's voxel keypoints on every accepted cloud."""
    cl = [c for c in CLOUDS if restated[c.name][1] == VOX_OK and 0 < len(restated[c.name][0]) <= V_DEFAULT]
    params = [make_params(voxel_size=c.leaf, skip_flagged=c.skip) for c in cl]
    with make_handle(1, **WAVE_CFG) as h:
        described, counts, status = h.describe_batch_each([c.pts for c in cl], params)
    bad = [c.name for c, d, n, st in zip(cl, described, counts, status)
           if st != VOX_OK or n != len(restated[c.name][0]) or not same_bits(d[0], restated[c.name][0])]
    assert not bad, bad
