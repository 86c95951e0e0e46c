"""Independent float64 numpy / scipy restatements of the third-party stages on the hot path (PCL VoxelGrid, NormalEstimation,
computePairFeatures, FPFHEstimation; FLANN exact 1-NN as brute force; the fp64 TIM mask of quatro.hpp:363-385), written from the
published algorithms, and a float32 restatement of the matcher's back half (feature_matcher.cc:18-76 and :187-264: the swap rule,
normalizePoints' mean, the tuple test with the counter-based Philox4x32-10 of deviation D1 in place of rand(), swap back, sort and
unique), and a list-and-set restatement of pmc's k-core peel and heuristic, findMaxClique and the canonical exact search (src/graph.cc:
12-130).  This module never imports oracle/ or the CUDA library: tools/gen_independent_pins.py uses it to write the
independent_*.npz fixtures, tests/test_independent_pins.py uses it to check the oracle, tests/test_tuple_adversarial.py to check
the oracle and the device matcher, tests/test_clique_adversarial.py the oracle and K9, and tests/test_fpfh_adversarial.py the
oracle's and the device's normals, SPFH and FPFH against the float32 restatement of PCL's NormalEstimation / FPFHEstimation below, and
tests/test_voxel_adversarial.py the oracle's and the device's voxel filter against the float32 restatement of PCL's VoxelGrid at the end."""
import numpy as np
from scipy.spatial import cKDTree


def voxel_grid(pts: np.ndarray, leaf: float):
    """pcl::VoxelGrid::applyFilter: ijk = floor(p / leaf) - floor(min / leaf); linear index i + j*dx + k*dx*dy; centroid per
    occupied voxel, output in ascending linear index.  float32 division like PCL (inverse_leaf_size multiplications), centroids
    in float64."""
    p32 = pts.astype(np.float32)
    inv = np.float32(1.0) / np.float32(leaf)
    mn = np.floor(p32.min(0) * inv).astype(np.int64)
    mx = np.floor(p32.max(0) * inv).astype(np.int64)
    div = mx - mn + 1
    ijk = np.floor(p32 * inv).astype(np.int64) - mn
    idx = ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * div[0] * div[1]
    order = np.argsort(idx, kind="stable")
    uniq, start, counts = np.unique(idx[order], return_index=True, return_counts=True)
    sums = np.add.reduceat(pts[order].astype(np.float64), start, axis=0)
    return (sums / counts[:, None]), idx, uniq


def normals_pcl(pts: np.ndarray, radius: float):
    """pcl::NormalEstimation: neighbours with d < radius (self included), < 3 -> NaN; covariance about the centroid;
    eigenvector of the smallest eigenvalue; flipped towards the viewpoint (0,0,0); curvature = l0 / (l0+l1+l2)."""
    tree = cKDTree(pts)
    out = np.full((len(pts), 4), np.nan)
    gap = np.zeros(len(pts))   # (l1 - l0) / l2: how well the smallest eigenvector is defined
    nbrs = tree.query_ball_point(pts, radius * (1 + 1e-9))
    for i, nb in enumerate(nbrs):
        nb = [j for j in nb if np.sum((pts[j] - pts[i]) ** 2) < radius * radius]
        if len(nb) < 3:
            continue
        q = pts[nb]
        c = q.mean(0)
        cov = (q - c).T @ (q - c) / len(nb)
        w, v = np.linalg.eigh(cov)
        n = v[:, 0]
        if np.dot(n, -pts[i]) < 0:
            n = -n
        out[i, :3] = n
        s = w.sum()
        out[i, 3] = abs(w[0] / s) if s != 0 else 0.0
        gap[i] = (w[1] - w[0]) / w[2] if w[2] > 0 else 0.0
    return out, gap


def pair_features(p1, n1, p2, n2):
    """pcl::computePairFeatures"""
    d = p2 - p1
    f4 = np.linalg.norm(d)
    if f4 == 0.0:
        return None
    a1 = np.dot(n1, d) / f4
    a2 = np.dot(n2, d) / f4
    # C++ semantics: a comparison with NaN is false (no swap when the other normal is NaN); acos argument clipped against rounding
    def acos_abs(x):
        return np.nan if np.isnan(x) else np.arccos(min(1.0, abs(x)))
    if acos_abs(a1) > acos_abs(a2):
        n1, n2 = n2, n1
        d = -d
        f3 = -a2
    else:
        f3 = a1
    v = np.cross(d, n1)
    vn = np.linalg.norm(v)
    if vn == 0.0:
        return None
    v = v / vn
    w = np.cross(n1, v)
    f2 = np.dot(v, n2)
    f1 = np.arctan2(np.dot(w, n2), np.dot(n1, n2))
    return f1, f2, f3


def fpfh_pcl(pts: np.ndarray, normals: np.ndarray, radius: float):
    """pcl::FPFHEstimation: SPFH of every point over its radius neighbours (bins of 11, increment 100/(k-1)), then the
    1/d^2-weighted sum of the neighbours' SPFHs, each third rescaled to sum 100."""
    tree = cKDTree(pts)
    n = len(pts)
    nbrs = []
    for i, nb in enumerate(tree.query_ball_point(pts, radius * (1 + 1e-9))):
        nb = sorted(j for j in nb if np.sum((pts[j] - pts[i]) ** 2) < radius * radius)
        nbrs.append(nb)
    spfh = np.zeros((n, 33))
    for i, nb in enumerate(nbrs):
        k = len(nb)
        if k < 2:
            continue
        inc = 100.0 / (k - 1)
        for j in nb:
            if j == i:
                continue
            f = pair_features(pts[i], normals[i, :3], pts[j], normals[j, :3])
            if f is None:
                continue
            f1, f2, f3 = f
            # PCL casts the bin to int: NaN becomes INT_MIN on x86 and is clamped to bin 0 -- per feature
            b = tuple(0 if np.isnan(x) else int(np.floor(x)) for x in (11 * (f1 + np.pi) / (2 * np.pi), 11 * (f2 + 1.0) * 0.5, 11 * (f3 + 1.0) * 0.5))
            b = [min(10, max(0, x)) for x in b]
            spfh[i, b[0]] += inc
            spfh[i, 11 + b[1]] += inc
            spfh[i, 22 + b[2]] += inc
    out = np.zeros((n, 33))
    for i, nb in enumerate(nbrs):
        acc = np.zeros(33)
        for j in nb:
            d2 = np.sum((pts[j] - pts[i]) ** 2)
            if d2 == 0.0:
                continue
            acc += spfh[j] / d2
        for t in range(3):
            s = acc[11 * t:11 * t + 11].sum()
            if s != 0:
                acc[11 * t:11 * t + 11] *= 100.0 / s
        out[i] = acc
    return out, spfh


def mutual_nn(da: np.ndarray, db: np.ndarray):
    """feature_matcher.cc:79-180 in its dense form: row/column argmins of the squared-distance matrix (float64, lowest index on
    ties), mutual pairs in ascending source index."""
    D = np.empty((len(da), len(db)))
    for i0 in range(0, len(da), 256):   # direct differences (exact ties stay exact), in row chunks
        blk = da[i0:i0 + 256, None, :] - db[None, :, :]
        D[i0:i0 + 256] = (blk * blk).sum(2)
    r = D.argmin(1)
    c = D.argmin(0)
    i = np.arange(len(da))
    keep = c[r] == i
    # second-best margins: pairs whose decision float32 arithmetic could flip
    Ds = np.sort(D, 1)
    margin_r = Ds[:, 1] - Ds[:, 0]
    Dc = np.sort(D, 0)
    margin_c = Dc[1] - Dc[0]
    return np.stack([i[keep], r[keep]], 1), margin_r, margin_c


def tim_graph(a: np.ndarray, b: np.ndarray, beta: float):
    """quatro.hpp:363-385 in float64 numpy: edge <=> |db/da - 1| <= beta/da and |da/db - 1| <= beta/db."""
    da = np.linalg.norm(a[:, None, :] - a[None, :, :], axis=2)
    db = np.linalg.norm(b[:, None, :] - b[None, :, :], axis=2)
    with np.errstate(divide="ignore", invalid="ignore"):
        e = (np.abs(db / da - 1) <= beta / da) & (np.abs(da / db - 1) <= beta / db)
    np.fill_diagonal(e, False)
    knife = np.abs(np.abs(da - db) - beta) < 1e-9
    return e, knife


# ---- the matcher's back half: feature_matcher.cc:18-76 and :187-264, deviation D1 --------------------------------------------------
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10_words(c0, c1, c2, c3, k0, k1):
    """Random123 philox4x32 with 10 rounds on 32-bit words held in numpy uint64 (arrays or scalars): each round multiplies counter
    words 0 and 2 by 0xD2511F53 and 0xCD9E8D57 into 64 bits and returns (hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0); the key is bumped by
    the Weyl constants (0x9E3779B9, 0xBB67AE85) between rounds.  Returns the four output words as uint32 arrays."""
    c0, c1, c2, c3 = (np.asarray(c, np.uint64) & _M32 for c in (c0, c1, c2, c3))
    k0, k1 = np.uint64(int(k0) & 0xFFFFFFFF), np.uint64(int(k1) & 0xFFFFFFFF)
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _M32, (k1 + np.uint64(0xBB67AE85)) & _M32
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _M32
    return tuple(np.asarray(c, np.uint64).astype(np.uint32) for c in (c0, c1, c2, c3))


def philox4x32_10(seed, ctr):
    """D1's generator: the four words of trial `ctr` (a uint64 array or scalar) under key `seed`, counter (ctr lo, ctr hi, 0, 0)
    and key (seed lo, seed hi).  Shape (4, len(ctr)); (4, 1) for a scalar."""
    ctr = np.atleast_1d(np.asarray(ctr, np.uint64))
    seed = int(seed)
    return np.stack(philox4x32_10_words(ctr & _M32, ctr >> np.uint64(32), 0, 0, seed & 0xFFFFFFFF, seed >> 32))


def cloud_mean(pts):
    """normalizePoints' mean (:27-36): an Eigen::Vector3f summed point by point in index order, then divided by float(n).  numpy's
    accumulate adds strictly in order (np.sum would add pairwise)."""
    p = np.asarray(pts, np.float32)[:, :3]
    if len(p) == 0:
        return np.zeros(3, np.float32)
    return np.add.accumulate(p, axis=0, dtype=np.float32)[-1] / np.float32(len(p))


def tuple_decide(li, lj, scale):
    """The six comparisons of :234-235 for one pair of sides, float32: (li*scale < lj, lj < li/scale)."""
    li, lj, s = np.asarray(li, np.float32), np.asarray(lj, np.float32), np.float32(scale)
    with np.errstate(all="ignore"):
        return (li * s < lj), (lj < li / s)


def _sides(c, a, b):
    d = c[a] - c[b]                                                  # centred float32 points: (p - mean) - (q - mean)
    return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])


def _margins_ulp(li, lj, s):
    """Exact margins of li*s < lj and lj < li/s on the float32 operands, in ulps of lj: lj - li*s (the product of two floats is exact
    in float64) and (li - lj*s) / s (its sign exact)."""
    li, lj, s = li.astype(np.float64), lj.astype(np.float64), float(np.float32(s))
    ulp = np.spacing(lj.astype(np.float32)).astype(np.float64)
    with np.errstate(all="ignore"):
        return (lj - li * s) / ulp, ((li - lj * s) / s) / ulp


def tuple_match(src, tgt, mutual, use_tuple_test=1, tuple_scale=0.95, trials_per_corr=100, seed=0x5EED, margins=False,
                mean=cloud_mean, chunk=1 << 22):
    """The matcher after its nearest-neighbour searches, given the mutual pairs as (source index, target index) rows in any order.

    :79-92 fi is the larger cloud (the source on ties); the cross check (:146-177) lists the mutual pairs in ascending fi index.  The
    tuple test (:187-247) runs when use_tuple_test and tuple_scale != 0 (NaN included): the points of both clouds are centred on their
    own cloud_mean (normalizePoints with use_absolute_scale = true, the scale stays 1), trial t draws r0, r1, r2 = Philox(seed, t)
    words 0..2 % ncorr, the sides are float32 sqrt((dx*dx + dy*dy) + dz*dz), and a trial that passes all six comparisons marks its
    three list entries; ncorr * trials_per_corr trials (D1 keeps the reference's 100 as the default).  The marked pairs are swapped
    back to (source, target), sorted and made unique (:249-264).  `mean` replaces the mean (to show what another summation order
    does).  margins=True also returns, per trial, the float32 sides (trials x 6: li0..2, lj0..2) and the exact margins of the six
    comparisons in ulps of lj (trials x 6, the order of :234-235), for scenes small enough to keep them."""
    src, tgt = np.asarray(src, np.float32), np.asarray(tgt, np.float32)
    swapped = len(tgt) > len(src)
    pi, pj = (tgt, src) if swapped else (src, tgt)
    mut = np.asarray(mutual, np.int64).reshape(-1, 2)
    if swapped:
        mut = mut[:, ::-1]
    mut = mut[np.argsort(mut[:, 0], kind="stable")]
    ncorr = len(mut)
    out = {"swapped": bool(swapped), "mutual": mut.copy(), "n_mutual": ncorr}
    corres = mut
    scale = np.float32(tuple_scale)
    if use_tuple_test and scale != 0 and ncorr > 0:
        with np.errstate(all="ignore"):
            ci = (pi[:, :3] - mean(pi)).astype(np.float32)[mut[:, 0]]
            cj = (pj[:, :3] - mean(pj)).astype(np.float32)[mut[:, 1]]
        mark = np.zeros(ncorr, bool)
        trials = ncorr * int(trials_per_corr)
        keep_sides, keep_marg = [], []
        for t0 in range(0, trials, chunk):
            r = philox4x32_10(seed, np.arange(t0, min(trials, t0 + chunk), dtype=np.uint64)).astype(np.int64) % ncorr
            r0, r1, r2 = r[0], r[1], r[2]
            with np.errstate(all="ignore"):
                if margins:
                    L = np.stack([_sides(ci, r0, r1), _sides(ci, r1, r2), _sides(ci, r2, r0),
                                  _sides(cj, r0, r1), _sides(cj, r1, r2), _sides(cj, r2, r0)], 1)
                    ok = np.ones(len(r0), bool)
                    marg = np.empty((len(r0), 6))
                    for k in range(3):
                        lo, hi = tuple_decide(L[:, k], L[:, 3 + k], scale)
                        ok &= lo & hi
                        marg[:, 2 * k], marg[:, 2 * k + 1] = _margins_ulp(L[:, k], L[:, 3 + k], scale)
                    keep_sides.append(L)
                    keep_marg.append(marg)
                else:                       # side 0 first; sides 1 and 2 only for the trials that pass it
                    lo, hi = tuple_decide(_sides(ci, r0, r1), _sides(cj, r0, r1), scale)
                    ok = lo & hi
                    sel = np.flatnonzero(ok)
                    for a, b in ((r1[sel], r2[sel]), (r2[sel], r0[sel])):
                        lo, hi = tuple_decide(_sides(ci, a, b), _sides(cj, a, b), scale)
                        ok[sel] &= lo & hi
            for rk in (r0, r1, r2):
                mark[rk[ok]] = True
        corres = mut[mark]
        out["mark"] = mark
        if margins:
            out["sides"] = np.concatenate(keep_sides) if keep_sides else np.zeros((0, 6), np.float32)
            out["margins"] = np.concatenate(keep_marg) if keep_marg else np.zeros((0, 6))
    if swapped:
        corres = corres[:, ::-1]
    out["corr"] = np.unique(corres, axis=0).astype(np.int32).reshape(-1, 2)
    return out


# ---- K9: pmc's k-core peel and heuristic, findMaxClique (src/graph.cc:12-130) and the canonical exact search -------------------------
# Plain lists and sets, written from the reference text and pmc's published algorithms (Rossi, Gleich, Gebremedhin, "Parallel maximum
# clique algorithms with applications to network analysis", SIAM J. Sci. Comput. 37(5), 2015; Batagelj and Zaversnik, "An O(m)
# algorithm for cores decomposition of networks", 2003).  A graph is (L, nbrs): nbrs[v] = neighbours of v in ascending id, the order
# in which graph.cc:24-29 hands pmc its CSR rows.
KCORE_HEU_MODE, PMC_HEU_MODE, PMC_EXACT_MODE = 2, 1, 0
CLIQUE_TRUNCATED = 1


def pmc_cores(L, nbrs):
    """pmc_graph::compute_cores (Batagelj-Zaversnik with pmc's bucket mechanic): vertices sit in `vert`, grouped by current degree,
    ids ascending inside a bin; peeling v decrements every neighbour u with deg[u] > deg[v] by swapping u with the FIRST vertex of
    u's bin and advancing that bin's start.  Returns (kcore = core + 1 per vertex (pmc's K), peel order, max core)."""
    deg = [len(nbrs[v]) for v in range(L)]
    if L == 0:
        return [], [], 0
    md = max(deg)
    bin_start = [0] * (md + 1)
    for d in deg:
        bin_start[d] += 1
    start = 0
    for d in range(md + 1):                 # bin_start[d] = first position of degree d
        bin_start[d], start = start, start + bin_start[d]
    pos, vert = [0] * L, [0] * L
    fill = list(bin_start)
    for v in range(L):                      # ids ascending inside a bin
        pos[v] = fill[deg[v]]
        vert[pos[v]] = v
        fill[deg[v]] += 1
    for i in range(L):
        v = vert[i]
        for u in nbrs[v]:
            if deg[u] > deg[v]:
                du, pu = deg[u], pos[u]
                pw = bin_start[du]
                w = vert[pw]
                if u != w:                  # u changes places with the first vertex of its bin
                    pos[u], vert[pu], pos[w], vert[pw] = pw, w, pu, u
                bin_start[du] += 1
                deg[u] -= 1
    return [d + 1 for d in deg], vert, deg[vert[L - 1]]


def pmc_heu(L, nbrs, K, order, ub, trace=None):
    """pmc_heu::search with heu_strat = "kcore" (graph.cc:89-91), start vertices sequential in reverse peel order (oracle D4):
    skip v when K[v] <= mc; P = neighbours u with K[u] > mc, skipped when |P| <= mc; P sorted stably by K (D3), so popping its back
    takes the largest (K, id); each step keeps the P members adjacent to the popped vertex with K > mc; a chain longer than mc
    replaces the incumbent; stop once mc >= ub.  Returns (mc, clique in push order); a list `trace` receives (peel position, new mc)
    of every improvement."""
    mc, best = 0, []
    for i in range(L - 1, -1, -1):
        if mc >= ub:
            break
        v = order[i]
        if K[v] <= mc:
            continue
        P = [u for u in nbrs[v] if K[u] > mc]
        if len(P) <= mc:
            continue
        P.sort(key=lambda u: K[u])          # list.sort is stable: ids stay ascending inside one K
        popped = []
        while P:
            u = P.pop()
            popped.append(u)
            nu = set(nbrs[u])
            P = [w for w in P if w in nu and K[w] > mc]
        if len(popped) + 1 > mc:
            mc = len(popped) + 1
            best = popped[::-1] + [v]
            if trace is not None:
                trace.append((i, mc))
    return mc, best


def kcore_heu_limit(thr, L):
    """(int)(thr * L) as x86-64's cvttsd2si computes it (the reference's only platform): the product truncated toward zero when that
    fits in int32, INT_MIN for NaN, infinities and every product outside int range."""
    x = float(thr) * float(L)
    if x != x or not (-2147483649.0 < x < 2147483648.0):
        return -2 ** 31
    return int(x)


def rank_space(L, K):
    """vertices renumbered by (core number, id) ascending: (rank_of, by_rank, first[c] = first rank whose core number >= c)"""
    by_rank = sorted(range(L), key=lambda v: (K[v], v))
    rank_of = [0] * L
    for r, v in enumerate(by_rank):
        rank_of[v] = r
    return rank_of, by_rank


def canonical_exact(L, nbrs, K, max_core, incumbent, node_limit, depth_limit=None, pool_limit=None):
    """The canonical branch and bound of DESIGN.md 5.3 / quatro_b200.h (qb200_max_clique_ex), in (core, id) rank space: root
    candidates = vertices with core number >= |incumbent|; greedy sequential colouring, each class taking the lowest-ranked candidate
    with no neighbour in it, listing only entries with colour > |incumbent| - |C|, in (colour, rank) order; the branch takes the list's
    last entry; a level dies when |C| + colour <= |incumbent|; a strictly larger maximal clique replaces the incumbent and the search
    ends when it reaches max_core + 1; every expanded node counts (++nodes > node_limit stops with the truncation flag).
    depth_limit / pool_limit add the device's scratch limits: expanding to depth depth_limit, or a colour list that would need more
    pool entries than pool_limit minus the entries of the lists on the current path (the consumed entry's slot passes to the child
    level), stops the search like the node limit.  Returns (clique sorted, flags, nodes, stop): stop is None for a search that ran
    out, else a dict of what ended it ("nodes", "depth" or "pool"), the depth of the node being expanded and the pool entries the
    lists on the path held (for "pool": before the list that did not fit)."""
    best = len(incumbent)
    ub = max_core + 1
    if L <= 0 or best <= 0 or best >= ub:
        return sorted(incumbent), 0, 0, None
    rank_of, by_rank = rank_space(L, K)
    adj = [set() for _ in range(L)]
    for v in range(L):
        adj[rank_of[v]] = {rank_of[u] for u in nbrs[v]}
    pool_cap = pool_limit if pool_limit is not None else float("inf")

    def colour_sort(P, kmin, cap):
        """the (rank, colour) list of P, or None when it needs more than cap entries"""
        left = set(P)
        out, col = [], 0
        while left:
            col += 1
            free = left - adj[min(left)]    # candidates with no neighbour in the class so far (its first member included)
            while free:
                v = min(free)
                free -= adj[v]
                free.discard(v)
                left.discard(v)
                if col > kmin:
                    if len(out) >= cap:
                        return None
                    out.append((v, col))
        return out

    core = [K[by_rank[r]] - 1 for r in range(L)]
    root = {r for r in range(L) if core[r] >= min(best, max_core + 1)}
    flags, nodes, best_c, stop = 0, 0, None, None
    lst = colour_sort(root, best, pool_cap)
    if lst is None:
        return sorted(incumbent), CLIQUE_TRUNCATED, 0, dict(reason="pool", depth=0, pool=0)
    stack = [[root, lst, 0]]                # per level: candidates, colour list, first pool slot of the list
    C = []
    while stack:
        depth = len(stack) - 1
        P, lst, begin = stack[-1]
        if not lst:
            stack.pop()
            continue
        v, col = lst.pop()
        if depth + col <= best:
            lst.clear()
            continue
        del C[depth:]
        C.append(v)
        NP = P & adj[v]
        P.discard(v)
        if not NP:
            if depth + 1 > best:
                best, best_c = depth + 1, list(C)
                if best >= ub:
                    break
            continue
        if depth + 1 + len(NP) <= best:
            continue
        nodes += 1
        nbegin = begin + len(lst)           # the consumed entry's slot and everything after it is free again
        if nodes > node_limit or (depth_limit is not None and depth + 1 >= depth_limit):
            flags, stop = CLIQUE_TRUNCATED, dict(reason="nodes" if nodes > node_limit else "depth", depth=depth, pool=nbegin)
            break
        child = colour_sort(NP, best - (depth + 1), pool_cap - nbegin)
        if child is None:
            flags, stop = CLIQUE_TRUNCATED, dict(reason="pool", depth=depth, pool=nbegin)
            break
        stack.append([set(NP), child, nbegin])
    clique = sorted(by_rank[r] for r in best_c) if best_c is not None else sorted(incumbent)
    return clique, flags, nodes, stop


def find_max_clique(L, nbrs, mode, thr=0.5, node_limit=262144, depth_limit=None, pool_limit=None):
    """teaser::MaxCliqueSolver::findMaxClique (src/graph.cc:12-130) with the exact search in its canonical form.  Returns a dict:
    kcore, order, max_core, clique (ascending ids, quatro.hpp:806), flags, heu (the heuristic's size), nodes and stop (canonical_exact)."""
    K, order, max_core = pmc_cores(L, nbrs)
    out = dict(kcore=K, order=order, max_core=max_core, flags=0, nodes=0, heu=0, stop=None)
    # graph.cc:67-82: the literal k_cores >= max_core (K = core + 1), != 1 short-circuits the comparison
    if mode == KCORE_HEU_MODE and thr != 1 and max_core > kcore_heu_limit(thr, L):
        out["clique"] = [v for v in range(L) if K[v] >= max_core]
        return out
    ub = max_core + 1                       # graph.cc:84-86
    lb, C = pmc_heu(L, nbrs, K, order, ub)  # graph.cc:89-91
    out["heu"] = lb
    if lb == 0 or lb == ub or mode != PMC_EXACT_MODE:   # graph.cc:93-104
        out["clique"] = sorted(C)
        return out
    out["clique"], out["flags"], out["nodes"], out["stop"] = canonical_exact(L, nbrs, K, max_core, C, node_limit, depth_limit, pool_limit)
    return out


# ---- one peel step's bucket moves: pmc's swap sequence and the closed form of kcore_apply_moves (clique.cu) ---------------------------
def group_moves_sequential(vert, pos, bin_start, deg, nbl):
    """One peel step as pmc runs it: for each neighbour u of the list in order, swap u with the vertex on the first slot of its bin,
    advance that bin and decrement deg[u].  Returns new (vert, pos, bin_start, deg); bin_start is a dict degree -> first slot."""
    vert, pos, bin_start, deg = list(vert), dict(pos), dict(bin_start), dict(deg)
    for u in nbl:
        du, pu = deg[u], pos[u]
        pw = bin_start[du]
        w = vert[pw]
        pos[u], vert[pu], pos[w], vert[pw] = pw, w, pu, u
        bin_start[du] += 1
        deg[u] -= 1
    return vert, pos, bin_start, deg


def group_moves_closed_form(vert, pos, bin_start, deg, nbl, chunk=32):
    """The same step as kcore_apply_moves computes it: the list in chunks of 32 lanes; inside a chunk the lanes of one current degree
    form a group (__match_any_sync) and lane rank t of a group of m lands on slot bin + t; a member that sat outside the m target
    slots walks the chain slot -> member that sat there -> its rank's slot ... backwards from its own rank until it reaches a
    non-member, which takes the member's old slot; rank 0 advances the bin by m after the chunk.  Every lane reads the state the
    chunk started from."""
    vert, pos, bin_start, deg = list(vert), dict(pos), dict(bin_start), dict(deg)
    for c0 in range(0, len(nbl), chunk):
        lanes = nbl[c0:c0 + chunk]
        du = [deg[u] for u in lanes]
        rank = [sum(1 for j in range(i) if du[j] == du[i]) for i in range(len(lanes))]
        m = [du.count(d) for d in du]
        b0 = [bin_start[d] for d in du]
        pu = [pos[u] for u in lanes]
        mrk = {u: rank[i] + 1 for i, u in enumerate(lanes)}
        ys = []
        for i in range(len(lanes)):
            y = None
            if pu[i] >= b0[i] + m[i]:
                k = rank[i]
                while True:
                    y = vert[b0[i] + k]
                    if y not in mrk:
                        break
                    k = mrk[y] - 1
            ys.append(y)
        for i, u in enumerate(lanes):
            vert[b0[i] + rank[i]] = u
            pos[u] = b0[i] + rank[i]
            if ys[i] is not None:
                vert[pu[i]] = ys[i]
                pos[ys[i]] = pu[i]
            deg[u] = du[i] - 1
            if rank[i] == 0:
                bin_start[du[i]] = b0[i] + m[i]
    return vert, pos, bin_start, deg


# ---- float32 restatement of PCL 1.8.1 NormalEstimation / FPFHEstimation over FLANN's radius search (src/teaser_utils/fpfh.cc:44-75) ----
# Written from the PCL and FLANN texts: KdTreeFLANN::radiusSearch -> flann::L2_Simple<float> with RadiusResultSet's strict '<';
# computeMeanAndCovarianceMatrix (single pass), eigen33 / computeRoots / computeRoots2, solvePlaneParameters, flipNormalTowardsViewpoint;
# computePairFeatures, computePointSPFHSignature, weightPointSPFHSignature.  Every float32 operation is one numpy float32 operation in
# the source's left-to-right order.  The transcendentals are a parameter: F64_MATH (float64 functions rounded once to float32, the
# plain reading of PCL) or D7_MATH (numpy float32 copies of the project's fixed-order polynomials, deviation D7).  The neighbour
# accumulation order is deviation D8's ascending (lattice cell key, index) from DESIGN section 2 (iv).
F32, F64 = np.float32, np.float64
FLT_EPSILON = F32(np.finfo(np.float32).eps)
FLT_MIN = F32(np.finfo(np.float32).tiny)
U32 = 2.0 ** -24                      # float32 unit roundoff
CELL_FACTOR = F32(1.001953125)        # default lattice cell = (1 + 2^-9) * fpfh_radius (D8)
_OFF_IJ, _OFF_K = 1 << 17, 1 << 15


class Math:
    """atan2(y, x), acos(x), sincos(x) -> (sin, cos) on float32 arrays or scalars, returning float32."""

    def __init__(self, name, atan2, acos, sincos):
        self.name, self.atan2, self.acos, self.sincos = name, atan2, acos, sincos


def _f64_atan2(y, x):
    r = np.arctan2(np.asarray(y, F64), np.asarray(x, F64))
    return F32(r) if np.ndim(r) == 0 else r.astype(F32)


def _f64_acos(x):
    with np.errstate(invalid="ignore"):
        r = np.arccos(np.asarray(x, F64))
    return F32(r) if np.ndim(x) == 0 else r.astype(F32)


def _f64_sincos(x):
    x = np.asarray(x, F64)
    s, c = np.sin(x).astype(F32), np.cos(x).astype(F32)
    return (F32(s), F32(c)) if np.ndim(x) == 0 else (s, c)


F64_MATH = Math("float64", _f64_atan2, _f64_acos, _f64_sincos)

# D7's kernels (quatro_b200/csrc/qb_math.cuh, coefficients from tools/fit_math.py), each line one float32 operation
_ATAN_C = [F32(c) for c in ("-4.044491798e-02", "7.135856152e-02", "-9.029050916e-02", "1.110749617e-01", "-1.428561211e-01",
                            "1.999999881e-01", "-3.333333433e-01")]
_ASIN_C = [F32(c) for c in ("3.109041601e-02", "1.048902422e-02", "2.363533154e-02", "3.026617132e-02", "4.464783147e-02",
                            "7.499992102e-02", "1.666666716e-01")]
_SIN_C = [F32(c) for c in ("1.469172284e-10", "-2.501203333e-08", "2.755685500e-06", "-1.984126720e-04", "8.333333768e-03",
                           "-1.666666716e-01")]
_COS_C = [F32(c) for c in ("3.323700412e-06", "-1.105757929e-05", "1.310664993e-05", "1.771735151e-05", "-1.387358177e-03",
                           "4.166657478e-02")]
PI_F, PI_2_F, PI_4_F = F32("3.14159274"), F32("1.57079637"), F32("0.785398185")


def _horner(c, z):
    p = np.full(np.shape(z), c[0], F32)
    for k in c[1:]:
        p = p * z + k
    return p


def _d7_atan2(y, x):
    scalar = np.ndim(y) == 0 and np.ndim(x) == 0
    y, x = np.atleast_1d(np.asarray(y, F32)), np.atleast_1d(np.asarray(x, F32))
    y, x = np.broadcast_arrays(y, x)
    with np.errstate(all="ignore"):
        ax, ay = np.abs(x), np.abs(y)
        hi, lo = np.where(ax > ay, ax, ay), np.where(ax > ay, ay, ax)
        a = np.where(hi == np.inf, np.where(lo == np.inf, F32(1), F32(0)), lo / hi).astype(F32)
        big = a > F32(0.41421357)
        t = np.where(big, (a - F32(1)) / (a + F32(1)), a).astype(F32)
        z = t * t
        core = t + t * (z * _horner(_ATAN_C, z))
        r = np.where(big, PI_4_F, F32(0)).astype(F32) + core
        r = np.where(ay > ax, PI_2_F - r, r)
        r = np.where((ax == 0) & (ay == 0), F32(0), r)
        r = np.where(np.signbit(x), PI_F - r, r)
        r = np.where(np.signbit(y), -r, r)
        r = np.where(np.isnan(x) | np.isnan(y), F32(np.nan), r).astype(F32)
    return r[0] if scalar else r


def _d7_acos(x):
    scalar = np.ndim(x) == 0
    x = np.atleast_1d(np.asarray(x, F32))
    with np.errstate(all="ignore"):
        ax = np.abs(x)
        z1 = ax * ax
        r1 = PI_2_F - (ax + ax * (z1 * _horner(_ASIN_C, z1)))
        z2 = (F32(1) - ax) * F32(0.5)
        s = np.sqrt(z2)
        r2 = F32(2) * (s + s * (z2 * _horner(_ASIN_C, z2)))
        r = np.where(ax <= F32(0.5), r1, r2)
        r = np.where(x < 0, PI_F - r, r)
        r = np.where(np.isnan(x) | (ax > F32(1)), F32(np.nan), r).astype(F32)
    return r[0] if scalar else r


def _d7_sincos(x):
    scalar = np.ndim(x) == 0
    x = np.atleast_1d(np.asarray(x, F32))
    z = x * x
    s = x + x * (z * _horner(_SIN_C, z))
    c = (F32(1) - F32(0.5) * z) + (z * z) * _horner(_COS_C, z)
    return (s[0], c[0]) if scalar else (s, c)


D7_MATH = Math("D7", _d7_atan2, _d7_acos, _d7_sincos)


def flann_radius(pts, q, r):
    """FLANN's radius search as PCL's KdTreeFLANN runs it: diff = query - point in float32, d2 = ((0 + dx*dx) + dy*dy) + dz*dz in
    float32 (L2_Simple<float>), kept when d2 < float(double(r) * double(r)) (RadiusResultSet, strict; radius_sq).  The query is its own
    neighbour.  Returns (mask over pts, d2 of every point)."""
    p = np.asarray(pts, F32)[:, :3]
    with np.errstate(all="ignore"):
        d = p[q] - p
        d2 = ((F32(0) + d[:, 0] * d[:, 0]) + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        return d2 < radius_sq(r), d2


def radius_sq(r):
    """KdTreeFLANN's squared radius, float(double(r) * double(r)).  PCL takes r as a double; the C-ABI takes a float32 radius
    (deviation D19), and callers that restate the library pass float32(r)."""
    return F32(F64(r) * F64(r))


def lattice_rank(pts, cell):
    """D8's canonical order: every point's rank in ascending (cell key, index), and whether it is in the lattice (finite, cell
    (floor(x / cell), ...) with |i|, |j| < 2^17 and |k| < 2^15, the top cell of each range reserved; DESIGN section 2 (iv)).  The cell
    coordinates are floor(p * (1 / cell)) in float32; key = (k + 2^15) << 36 | (j + 2^17) << 18 | (i + 2^17)."""
    p = np.asarray(pts, F32)[:, :3]
    inv = F32(1) / F32(cell)
    with np.errstate(all="ignore"):
        c = np.floor(p * inv)
    ok = np.isfinite(p).all(1) & (c[:, 0] >= -_OFF_IJ) & (c[:, 0] < _OFF_IJ - 1) & (c[:, 1] >= -_OFF_IJ) & (c[:, 1] < _OFF_IJ - 1) \
        & (c[:, 2] >= -_OFF_K) & (c[:, 2] < _OFF_K - 1)
    ci = np.where(ok[:, None], c, 0).astype(np.int64)
    key = ((ci[:, 2] + _OFF_K) << 36) | ((ci[:, 1] + _OFF_IJ) << 18) | (ci[:, 0] + _OFF_IJ)
    order = np.lexsort((np.arange(len(p)), key))
    rank = np.empty(len(p), np.int64)
    rank[order] = np.arange(len(p))
    return rank, ok


def canonical_neighbours(pts, q, r, rank, in_lattice):
    """q's radius neighbours (flann_radius) in D8 order, and their d2; none for a query outside the lattice."""
    if not in_lattice[q]:
        return np.zeros(0, np.int64), np.zeros(0, F32)
    m, d2 = flann_radius(pts, q, r)
    idx = np.flatnonzero(m & in_lattice)
    idx = idx[np.argsort(rank[idx])]
    return idx, d2[idx]


def _compute_roots2(b, c):
    d = F32(F64(b * b) - 4.0 * F64(c))
    if d < 0:
        d = F32(0)
    sd = np.sqrt(d)
    return [F32(0), F32(0.5) * (b - sd), F32(0.5) * (b + sd)]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def normal_pcl32(nb, query, math):
    """computePointNormal of one query over its neighbour points nb ((k, 3) float32, accumulation order): fewer than 3 -> NaN;
    computeMeanAndCovarianceMatrix (float32 sums from 0, accu /= k, cov = accu[i] - accu[a] * accu[b]); eigen33 (scale = the largest
    |coefficient|, 1 when that is <= FLT_MIN; computeRoots, the row cross products, the largest squared norm with '>=' ties to the
    first); curvature |l0 / trace| (0 for a zero trace); the flip (vp - p) . n < 0 with the viewpoint at the origin.
    Returns ((nx, ny, nz, curvature) float32, record): the record holds the float32 covariance, every decision's operands, and each
    transcendental-dependent decision's margin over the error a change of <= 3 ulp in atan2 / sin / cos can cause (ratio > 1 clears)."""
    nan4 = np.full(4, np.nan, F32)
    rec = dict(k=len(nb), branch="few", margins={})
    if len(nb) < 3:
        return nan4, rec
    nb = np.asarray(nb, F32)
    x, y, z = nb[:, 0], nb[:, 1], nb[:, 2]
    terms = np.stack([x * x, x * y, x * z, y * y, y * z, z * z, x, y, z], 1)
    accu = np.add.accumulate(np.concatenate([np.zeros((1, 9), F32), terms]), axis=0, dtype=F32)[-1]
    accu = accu / F32(len(nb))
    cov = np.zeros(9, F32)
    cov[0] = accu[0] - accu[6] * accu[6]
    cov[1] = accu[1] - accu[6] * accu[7]
    cov[2] = accu[2] - accu[6] * accu[8]
    cov[4] = accu[3] - accu[7] * accu[7]
    cov[5] = accu[4] - accu[7] * accu[8]
    cov[8] = accu[5] - accu[8] * accu[8]
    cov[3], cov[6], cov[7] = cov[1], cov[2], cov[5]
    rec["cov"] = cov.reshape(3, 3).copy()
    # eigen33
    scale = F32(0)
    for a in np.abs(cov):
        scale = a if scale < a else scale
    rec["scale_reset"] = not (scale > FLT_MIN)
    if rec["scale_reset"]:
        scale = F32(1)
    s = [cov[i] / scale for i in range(9)]
    m00, m01, m02, m11, m12, m22 = s[0], s[1], s[2], s[4], s[5], s[8]
    c0 = m00 * m11 * m22 + F32(2) * m01 * m02 * m12 - m00 * m12 * m12 - m11 * m02 * m02 - m22 * m01 * m01
    c1 = m00 * m11 - m01 * m01 + m00 * m22 - m02 * m02 + m11 * m22 - m12 * m12
    c2 = m00 + m11 + m22
    rec.update(c0=c0, c1=c1, c2=c2)
    err_r = 0.0                                         # bound on the roots' change under a 3-ulp change of atan2 / sin / cos
    if np.abs(c0) < FLT_EPSILON:
        rec["branch"] = "roots2"
        roots = _compute_roots2(c2, c1)
    else:
        rec["branch"] = "cubic"
        s_inv3, s_sqrt3 = F32(1.0 / 3.0), np.sqrt(F32(3))
        c2_over_3 = c2 * s_inv3
        a_over_3 = (c1 - c2 * c2_over_3) * s_inv3
        rec["a_over_3"] = a_over_3
        if a_over_3 > 0:
            a_over_3 = F32(0)
        half_b = F32(0.5) * (c0 + c2_over_3 * (F32(2) * c2_over_3 * c2_over_3 - c1))
        q = half_b * half_b + a_over_3 * a_over_3 * a_over_3
        rec["q"] = q
        if q > 0:
            q = F32(0)
        rho = np.sqrt(-a_over_3)
        theta = math.atan2(np.sqrt(-q), half_b) * s_inv3
        sin_t, cos_t = math.sincos(theta)
        roots = [c2_over_3 + F32(2) * rho * cos_t, c2_over_3 - rho * (cos_t + s_sqrt3 * sin_t),
                 c2_over_3 - rho * (cos_t - s_sqrt3 * sin_t)]
        rec["roots_cubic"] = list(roots)
        err_r = 16 * U32 * (abs(float(c2_over_3)) + 4 * float(rho))
        gaps = []
        if roots[0] >= roots[1]:
            roots[0], roots[1] = roots[1], roots[0]
        gaps.append(abs(float(roots[0]) - float(roots[1])))
        if roots[1] >= roots[2]:
            roots[1], roots[2] = roots[2], roots[1]
            gaps.append(abs(float(roots[1]) - float(roots[2])))
            if roots[0] >= roots[1]:
                roots[0], roots[1] = roots[1], roots[0]
            gaps.append(abs(float(roots[0]) - float(roots[1])))
        else:
            gaps.append(abs(float(roots[1]) - float(roots[2])))
        rec["margins"]["root_swaps"] = min(gaps) / (2 * err_r) if err_r > 0 else np.inf
        rec["margins"]["root0_sign"] = abs(float(roots[0])) / err_r if err_r > 0 else np.inf
        rec["roots0_nonpositive"] = bool(roots[0] <= 0)
        if roots[0] <= 0:
            roots = _compute_roots2(c2, c1)
            err_r = 0.0
    rec["roots"] = list(roots)
    eigenvalue = roots[0] * scale
    s[0], s[4], s[8] = s[0] - roots[0], s[4] - roots[0], s[8] - roots[0]
    v1, v2, v3 = _cross(s[0:3], s[3:6]), _cross(s[0:3], s[6:9]), _cross(s[3:6], s[6:9])
    l1, l2, l3 = _dot(v1, v1), _dot(v2, v2), _dot(v3, v3)
    rec["l"] = (l1, l2, l3)
    if l1 >= l2 and l1 >= l3:
        v, ll, pick = v1, l1, 0
    elif l2 >= l1 and l2 >= l3:
        v, ll, pick = v2, l2, 1
    else:
        v, ll, pick = v3, l3, 2
    rec["pick"] = pick
    sl = np.sqrt(ll)
    with np.errstate(all="ignore"):
        e = [v[0] / sl, v[1] / sl, v[2] / sl]
        trace = cov[0] + cov[4] + cov[8]
        curv = np.abs(eigenvalue / trace) if trace != 0 else F32(0)
        vp = [F32(0) - F32(query[0]), F32(0) - F32(query[1]), F32(0) - F32(query[2])]
        cos_theta = (vp[0] * e[0] + vp[1] * e[1]) + vp[2] * e[2]
    rec["cos_theta"] = cos_theta
    if cos_theta < 0:
        e = [e[0] * F32(-1), e[1] * F32(-1), e[2] * F32(-1)]
    # margins of the decisions downstream of the roots: which cross product, and the flip
    if err_r > 0:
        rowmax = max(abs(float(t)) for t in s)
        others = sorted((float(l1), float(l2), float(l3)), reverse=True)
        err_l = 16 * err_r * rowmax * (np.sqrt(others[0]) + rowmax * err_r) + 8 * U32 * others[0]
        rec["margins"]["l_choice"] = (others[0] - others[1]) / err_l if err_l > 0 else np.inf
        gap = max(abs(float(roots[1]) - float(roots[0])), 1e-300)
        err_e = 4 * err_r / gap + 8 * U32
        vpn = float(np.sqrt(sum(float(t) ** 2 for t in vp)))
        rec["err_normal"] = err_e
        rec["margins"]["flip"] = abs(float(cos_theta)) / (vpn * err_e) if vpn > 0 else np.inf
    else:
        rec["err_normal"] = 0.0
    return np.array([e[0], e[1], e[2], curv], F32), rec


def eig_reference(cov):
    """The exact smallest eigenpair of a float32 covariance (as formed), in float64: (eigenvalues ascending, unit eigenvector of the
    smallest, bound factor u * ||C|| / (l1 - l0), inf on a zero gap)."""
    w, V = np.linalg.eigh(np.asarray(cov, F64))
    gap = w[1] - w[0]
    norm = np.abs(w).max()
    return w, V[:, 0], (U32 * norm / gap if gap > 0 else np.inf)


def _vec_cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)


def _vec_dot(a, b):
    return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]


D_PI = F32(1) / (F32(2) * F32(np.pi))                 # PCL's d_pi_ = 1.0f / (2.0f * static_cast<float> (M_PI))


def feature_scaled(f1, f2, f3):
    """The double expressions PCL floors: 11 * ((f1 + M_PI) * d_pi_), 11 * ((f2 + 1.0) * 0.5), 11 * ((f3 + 1.0) * 0.5)."""
    return (11 * ((np.asarray(f1, F64) + np.pi) * F64(D_PI)), 11 * ((np.asarray(f2, F64) + 1.0) * 0.5),
            11 * ((np.asarray(f3, F64) + 1.0) * 0.5))


def feature_bin(scaled):
    """floor, clamped to [0, 10]; NaN -> 0 (deviation D6: PCL's cast of NaN is undefined, INT_MIN on x86, clamped to 0)."""
    with np.errstate(invalid="ignore"):
        b = np.clip(np.floor(np.nan_to_num(scaled, nan=0.0)), 0, 10).astype(np.int64)
    return b


def pair_features_pcl32(p1, n1, p2, n2, math, err_n1=None, err_n2=None):
    """computePairFeatures on m pairs at once ((m, 3) float32 arrays).  A pair is skipped (ok False) when f4 == 0 or ||v|| == 0.
    The swap is acos(|a1|) > acos(|a2|) (false on NaN).  Returns dict(ok, f1, f2, f3, swap, a1, a2, and the margins: 'swap' and
    'skip' of the two decisions, 'bins' (m, 3) of each scaled feature's distance to the nearest inner bin edge, each over the error that a
    3-ulp change of acos / atan2 plus normals off by err_n1 / err_n2 radians can cause; ratio > 1 clears)."""
    p1, n1, p2, n2 = (np.atleast_2d(np.asarray(a, F32)) for a in (p1, n1, p2, n2))
    m = len(p1)
    e1 = np.zeros(m) if err_n1 is None else np.broadcast_to(np.asarray(err_n1, F64), (m,))
    e2 = np.zeros(m) if err_n2 is None else np.broadcast_to(np.asarray(err_n2, F64), (m,))
    with np.errstate(all="ignore"):
        dp = p2 - p1
        f4 = np.sqrt(_vec_dot(dp, dp))
        a1 = _vec_dot(n1, dp) / f4
        a2 = _vec_dot(n2, dp) / f4
        c1, c2 = math.acos(np.abs(a1)), math.acos(np.abs(a2))
        swap = c1 > c2
        n1c = np.where(swap[:, None], n2, n1)
        n2c = np.where(swap[:, None], n1, n2)
        dp = np.where(swap[:, None], dp * F32(-1), dp)
        f3 = np.where(swap, -a2, a1)
        v = _vec_cross(dp, n1c)
        vn = np.sqrt(_vec_dot(v, v))
        ok = (f4 != 0) & (vn != 0)
        v = v / vn[:, None]
        w = _vec_cross(n1c, v)
        f2 = _vec_dot(v, n2c)
        y, x = _vec_dot(w, n2c), _vec_dot(n1c, n2c)
        f1 = math.atan2(y, x)
        # margins
        da = e1 + e2 + 8 * U32                                   # change of |a1| - |a2| from the normals and the dot products
        acos_ulp = 3 * np.spacing(np.maximum(c1, c2).astype(F32)).astype(F64)
        slope = np.sqrt(np.maximum(1 - np.maximum(np.abs(a1), np.abs(a2)).astype(F64) ** 2, 0))
        m_swap = np.abs(np.abs(a1.astype(F64)) - np.abs(a2.astype(F64))) / (da + 2 * acos_ulp * np.maximum(slope, 1e-30))
        m_swap = np.where(np.isnan(a1) | np.isnan(a2), np.inf, m_swap)
        en = np.where(swap, e2, e1)
        m_skip = vn.astype(F64) / ((en + 8 * U32) * f4.astype(F64))
        df = 2 * (e1 + e2) + 16 * U32
        df1 = 3 * np.spacing(np.abs(f1).astype(F32)).astype(F64) + df / np.maximum(np.hypot(y.astype(F64), x.astype(F64)), 1e-300) + 8 * U32
        sc = feature_scaled(f1, f2, f3)
        dist = [np.abs(t - np.clip(np.round(t), 1, 10)) for t in sc]
        m_bins = np.stack([dist[0] / (11 / (2 * np.pi) * df1 + 1e-15), dist[1] / (5.5 * df + 1e-15), dist[2] / (5.5 * df + 1e-15)], 1)
        m_bins = np.where(np.isnan(m_bins), np.inf, m_bins)
    return dict(ok=ok, f1=f1, f2=f2, f3=f3, swap=swap, a1=a1, a2=a2, scaled=np.stack(sc, 1), bins=np.stack([feature_bin(t) for t in sc], 1),
                margins=dict(swap=m_swap, skip=np.where(f4 == 0, np.inf, m_skip), bins=m_bins))


def fpfh_pcl32(pts4, normal_radius, fpfh_radius, grid_cell=None, math=D7_MATH):
    """NormalEstimation (normal_radius) and FPFHEstimation (fpfh_radius) of every point of pts4, float32 as PCL 1.8.1 evaluates them,
    neighbours from flann_radius in D8 order (cell = grid_cell, else (1 + 2^-9) * fpfh_radius in float32).
    SPFH (computePointSPFHSignature): k = every radius neighbour (the query, coincident duplicates and skipped pairs included); k < 2 ->
    a zero row; hist_incr = 100.0f / (float)(k - 1) added once per pair and feature to bin floor(scaled) (pairs skipped by index, the
    query's own); FPFH (weightPointSPFHSignature): neighbours with d2 == 0 skipped, weight = 1.0f / d2, float val = spfh * weight summed
    into float bins and a double sum per third, then bins *= (float)(100.0 / sum) when sum != 0.
    Returns dict(normals (n, 4), spfh (n, 33), desc (n, 33), nbr_n / nbr_f (index lists), d2_f, nrec (normal records), pairs (per
    point: pair_features_pcl32's dict of its neighbour pairs), stable (n,) bool: every transcendental-dependent decision behind the
    point's normal, SPFH row and descriptor clears its margin)."""
    p4 = np.asarray(pts4, F32)
    p = p4[:, :3]
    n = len(p)
    cell = F32(grid_cell) if grid_cell else F32(fpfh_radius) * CELL_FACTOR
    rank, inl = lattice_rank(p, cell)
    nbr_n, nbr_f, d2_f = [], [], []
    for q in range(n):
        i, _ = canonical_neighbours(p, q, F32(normal_radius), rank, inl)     # float32 radii (D19)
        j, d2 = canonical_neighbours(p, q, F32(fpfh_radius), rank, inl)
        nbr_n.append(i)
        nbr_f.append(j)
        d2_f.append(d2)
    normals = np.zeros((n, 4), F32)
    nrec = []
    for q in range(n):
        normals[q], r = normal_pcl32(p[nbr_n[q]], p[q], math)
        nrec.append(r)
    err_n = np.array([r.get("err_normal", 0.0) for r in nrec])
    n_ok = np.array([all(v > 1 for v in r["margins"].values()) for r in nrec])
    spfh = np.zeros((n, 33), F32)
    pairs, spfh_ok = [], np.ones(n, bool)
    for q in range(n):
        nb = nbr_f[q]
        k = len(nb)
        other = nb[nb != q]
        pf = pair_features_pcl32(np.broadcast_to(p[q], (len(other), 3)), np.broadcast_to(normals[q, :3], (len(other), 3)), p[other],
                                 normals[other, :3], math, err_n[q], err_n[other])
        pf["other"] = other
        pairs.append(pf)
        mg = pf["margins"]
        spfh_ok[q] = n_ok[q] and n_ok[other].all() and (mg["swap"] > 1).all() and (mg["skip"] > 1).all() and \
            (mg["bins"][pf["ok"]] > 1).all()
        if k < 2:
            continue
        incr = F32(100) / F32(k - 1)
        counts = np.zeros(33, np.int64)
        for t in range(3):
            np.add.at(counts, 11 * t + pf["bins"][pf["ok"], t], 1)
        for b in np.flatnonzero(counts):
            spfh[q, b] = np.add.accumulate(np.concatenate([[F32(0)], np.full(counts[b], incr, F32)]), dtype=F32)[-1]
    desc = np.zeros((n, 33), F32)
    for q in range(n):
        keep = d2_f[q] != 0
        nb, d2 = nbr_f[q][keep], d2_f[q][keep]
        if len(nb) == 0:
            continue
        with np.errstate(all="ignore"):
            weight = F32(1) / d2
            val = spfh[nb] * weight[:, None]
        desc[q] = np.add.accumulate(np.concatenate([np.zeros((1, 33), F32), val]), axis=0, dtype=F32)[-1]
        for t in range(3):
            ssum = np.add.accumulate(np.concatenate([[0.0], val[:, 11 * t:11 * t + 11].astype(F64).ravel()]))[-1]
            if ssum != 0:
                ssum = 100.0 / ssum
            with np.errstate(all="ignore"):
                desc[q, 11 * t:11 * t + 11] = desc[q, 11 * t:11 * t + 11] * F32(ssum)
    stable = np.array([spfh_ok[nbr_f[q]].all() and n_ok[q] for q in range(n)], bool)
    return dict(normals=normals, spfh=spfh, desc=desc, nbr_n=nbr_n, nbr_f=nbr_f, d2_f=d2_f, nrec=nrec, pairs=pairs, stable=stable,
                normal_stable=n_ok, spfh_stable=spfh_ok, cell=cell)


# ---- float32 restatement of pcl::VoxelGrid<PointXYZ>::applyFilter (PCL 1.8.1), include/quatro.hpp:49-57 ------------------------------
# Written from the PCL text: inverse_leaf_size_ = 1 / leaf in float; getMinMax3D over the points the filter keeps; the int64 check of the
# truncated spans; min_b_ / max_b_ by float floor; div_b_ and divb_mul_; ijk = int(floor(p * inv) - float(min_b)) with the subtraction in
# FLOAT; the int index ijk0 + ijk1 * divb_mul[1] + ijk2 * divb_mul[2]; the sort of (index, point) pairs; a CentroidPoint per voxel (float
# accumulators from +0.0, points added in sorted order, divided by float(count), w = 1).  Every float operation is one numpy float32
# operation; index arithmetic is Python int or int64.
VOX_OK, VOX_OVERFLOW = 0, -5            # QB200_OK, QB200_ERR_VOXEL_OVERFLOW
INT32_MAX = 2 ** 31 - 1


def _sequential_sums(xyz, start, counts):
    """Per voxel, the float32 sum of its rows of xyz [start, start + count) added one by one from +0.0 (no pairwise reduction)."""
    acc = np.zeros((len(start), 3), np.float32)
    small = counts <= 64
    with np.errstate(over="ignore"):                              # a voxel's sum may overflow to +-inf, as in float
        for k in range(int(counts[small].max(initial=0))):       # round k adds the k-th point of every voxel that has one
            v = np.nonzero(small & (counts > k))[0]
            acc[v] = acc[v] + xyz[start[v] + k]
        for v in np.nonzero(~small)[0]:                           # np.add.accumulate is sequential; +0.0 first, as the accumulator
            seg = np.concatenate([np.zeros((1, 3), np.float32), xyz[start[v]:start[v] + counts[v]]])
            acc[v] = np.add.accumulate(seg, axis=0, dtype=np.float32)[-1]
    return acc


def voxel_grid_pcl32(pts4, leaf, skip_flagged=1):
    """pcl::VoxelGrid<PointXYZ>::applyFilter in float32 on n x 4 records.  Returns (out, status, grid):
    out     the centroids (x, y, z, 1) in ascending voxel index, or on a refusal the kept records as they are (DESIGN section 2 (ii));
    status  VOX_OK or VOX_OVERFLOW;
    grid    dict: inv, lo / hi (float floors of the bbox corners), span (PCL's truncated spans), min_b, div_b, top (per axis, the
            largest ijk: the float subtraction at the bbox corners), top_index (the largest linear index), refused (None or the rule),
            and for accepted clouds idx (index per kept point), order (the stable sort), uniq / start / counts of the voxels.
    Kept points: finite x, y, z and, with skip_flagged, not w < 0 (the library's ground flag).  Deviations from the PCL text:
      D3   the sort is stable (PCL's std::sort leaves tied indices in an unspecified order);
      D10  refused, besides PCL's own check, wherever PCL's int arithmetic would overflow: a floor outside int32 ("floor"), a product of
           div_b above INT_MAX ("div_b"), or a largest linear index above INT_MAX ("top_index": the float subtraction can round ijk up to
           div_b, so the index can exceed div_b0 * div_b1 * div_b2 - 1)."""
    pts4 = np.asarray(pts4, np.float32).reshape(-1, 4)
    keep = np.isfinite(pts4[:, :3]).all(1)
    if skip_flagged:
        keep &= ~(pts4[:, 3] < 0)
    kept = pts4[keep]
    with np.errstate(over="ignore", divide="ignore"):
        inv = F32(1) / F32(leaf)
    grid = dict(inv=inv, refused=None)
    if len(kept) == 0:
        return np.zeros((0, 4), np.float32), VOX_OK, grid
    xyz = kept[:, :3]
    mn, mx = xyz.min(0), xyz.max(0)
    with np.errstate(over="ignore", invalid="ignore"):
        lo, hi = np.floor(mn * inv), np.floor(mx * inv)
        s = (mx - mn) * inv
    grid.update(lo=lo, hi=hi)

    def refuse(rule):
        grid["refused"] = rule
        return kept.copy(), VOX_OVERFLOW, grid

    # PCL: dx = static_cast<int64_t>((max_p[0] - min_p[0]) * inverse_leaf_size_[0]) + 1, ...; dx * dy * dz > INT_MAX -> input returned.
    # A span of 2^31 or more (or inf / NaN, where the int64 cast is undefined) fails that check on its own.
    if not (s < 2.0 ** 31).all():
        return refuse("span")
    span = [int(v) + 1 for v in s]
    if span[0] * span[1] * span[2] > INT32_MAX:
        return refuse("span")
    if not ((lo >= -2.0 ** 31).all() and (hi < 2.0 ** 31).all()):       # D10: min_b_ = static_cast<int>(floor(...)) must fit
        return refuse("floor")
    min_b = [int(v) for v in lo]
    div_b = [int(h) - int(l) + 1 for h, l in zip(hi, lo)]               # div_b_ = max_b_ - min_b_ + 1
    grid.update(span=span, min_b=min_b, div_b=div_b)
    if div_b[0] * div_b[1] * div_b[2] > INT32_MAX:                       # D10: divb_mul_ and the index must fit an int
        return refuse("div_b")
    mul = [1, div_b[0], div_b[0] * div_b[1]]                             # divb_mul_
    top = [int(F32(h - l)) for h, l in zip(hi, lo)]                      # floor(max * inv) - float(min_b), monotone in the point
    top_index = top[0] * mul[0] + top[1] * mul[1] + top[2] * mul[2]
    grid.update(top=top, top_index=top_index)
    if top_index > INT32_MAX:                                            # D10: the largest index PCL computes must fit an int
        return refuse("top_index")
    with np.errstate(over="ignore", invalid="ignore"):
        ijk = (np.floor(xyz * inv) - lo.astype(np.float32)).astype(np.int64)   # float(min_b) == lo exactly: lo is a float integer
    idx = ijk[:, 0] * mul[0] + ijk[:, 1] * mul[1] + ijk[:, 2] * mul[2]
    order = np.argsort(idx, kind="stable")                               # D3
    uniq, start, counts = np.unique(idx[order], return_index=True, return_counts=True)
    sums = _sequential_sums(xyz[order], start, counts)
    out = np.ones((len(uniq), 4), np.float32)
    out[:, :3] = sums / counts.astype(np.float32)[:, None]
    grid.update(idx=idx, order=order, uniq=uniq, start=start, counts=counts)
    return out, VOX_OK, grid
