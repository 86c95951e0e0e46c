"""Independent float64 numpy / scipy restatements of the third-party stages on the hot path (PCL VoxelGrid, NormalEstimation,
computePairFeatures, FPFHEstimation; FLANN exact 1-NN as brute force; the fp64 TIM mask of quatro.hpp:363-385), written from the
published algorithms, and a float32 restatement of the matcher's back half (feature_matcher.cc:18-76 and :187-264: the swap rule,
normalizePoints' mean, the tuple test with the counter-based Philox4x32-10 of deviation D1 in place of rand(), swap back, sort and
unique), and a list-and-set restatement of pmc's k-core peel and heuristic, findMaxClique and the canonical exact search (src/graph.cc:
12-130).  This module never imports oracle/ or the CUDA library: tools/gen_independent_pins.py uses it to write the
independent_*.npz fixtures, tests/test_independent_pins.py uses it to check the oracle, tests/test_tuple_adversarial.py to check
the oracle and the device matcher, and tests/test_clique_adversarial.py the oracle and K9."""
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
