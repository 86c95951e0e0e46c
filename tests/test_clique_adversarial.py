"""K9 (clique.cu: kcore_kernel, permute_adj_kernel, clique_cta_kernel, clique_exact_kernel) against a plain restatement of pmc and
findMaxClique (tests/independent_ref.py) on graphs aimed at the kernels' code paths: equal-degree buckets whose moves need the chain
walk, one bucket group split across 32-neighbour chunks, every size switch of the launch formulas +-1, heuristic rounds whose winners
sit at chosen warps, planted cliques under higher-core decoys, node limits around the count, the device-only list-pool and
stack stops,
KCORE_HEU thresholds around the cut-off and beyond int range, and adjacency rows with stray bits past column L.

CPU tier: the closed form of kcore_apply_moves equals pmc's swap sequence (exhaustively for buckets of up to 8 slots, and on random
configurations with groups split across chunks); restatement == oracle field by field on the catalogue; core numbers == networkx;
exact sizes == networkx's maximum clique.  GPU tier: qb200_max_clique_ex == restatement on the catalogue on handles of max_corr 1024
... 32768 (every WPL instance), stray bits in the single call, the batch call and the oracle, and one mixed
wave through qb200_max_clique_batch_each on 1 and 4 lanes."""
import itertools
import math

import numpy as np
import pytest

import independent_ref as ref
from independent_ref import KCORE_HEU_MODE, PMC_EXACT_MODE, PMC_HEU_MODE
from quatro_b200.capi import GRAPH_LISTS, KCORE_HEU, MEM_HOST, PMC_EXACT, PMC_HEU, ListBuffers, default_params
from support import make_handle

assert (KCORE_HEU, PMC_HEU, PMC_EXACT) == (KCORE_HEU_MODE, PMC_HEU_MODE, PMC_EXACT_MODE)
MODES = (PMC_EXACT, PMC_HEU, KCORE_HEU)
TRUNCATED = 1
DEFAULT_NODE_LIMIT = 262144          # QB200_DEFAULT_CLIQUE_NODE_LIMIT


# ---- graphs -------------------------------------------------------------------------------------------------------------------------
class G:
    """An undirected graph on L vertices from an edge array (E x 2): adjacency rows for the library and the oracle, ascending
    neighbour lists for the restatement."""

    def __init__(self, name, L, edges):
        e = np.asarray(edges, np.int64).reshape(-1, 2)
        e = e[e[:, 0] != e[:, 1]]
        e = np.unique(np.sort(e, 1), axis=0)
        self.name, self.L, self.edges = name, int(L), e

    def rows(self, wpr=None):
        L = self.L
        wpr = wpr or max((L + 31) // 32, 1)
        a = np.zeros(max(L, 1) * wpr, np.uint32)
        r, c = np.concatenate([self.edges[:, 0], self.edges[:, 1]]), np.concatenate([self.edges[:, 1], self.edges[:, 0]])
        np.bitwise_or.at(a, r * wpr + (c >> 5), np.uint32(1) << (c & 31).astype(np.uint32))
        return a.reshape(max(L, 1), wpr)[:L]

    def nbrs(self):
        out = [[] for _ in range(self.L)]
        for u, v in self.edges.tolist():
            out[u].append(v)
            out[v].append(u)
        return [sorted(x) for x in out]

    def nx(self):
        import networkx as nx
        g = nx.Graph()
        g.add_nodes_from(range(self.L))
        g.add_edges_from(self.edges.tolist())
        return g

    def relabel(self, perm):
        """vertex v becomes perm[v]"""
        p = np.asarray(perm, np.int64)
        return G(self.name, self.L, p[self.edges] if len(self.edges) else self.edges)


def from_nx(name, g, rng=None):
    import networkx as nx
    g = nx.convert_node_labels_to_integers(g)
    out = G(name, g.number_of_nodes(), np.array(list(g.edges()), np.int64).reshape(-1, 2))
    return out.relabel(rng.permutation(out.L)) if rng is not None else out


def gnp(name, rng, L, p):
    u, v = np.triu_indices(L, 1)
    keep = rng.random(len(u)) < p
    return G(name, L, np.stack([u[keep], v[keep]], 1))


def sparse(name, rng, L, deg):
    m = L * deg // 2
    return G(name, L, np.stack([rng.integers(0, L, m), rng.integers(0, L, m)], 1))


def regular(name, rng, L, d):
    import networkx as nx
    return from_nx(name, nx.random_regular_graph(d, L, seed=int(rng.integers(1 << 30))))


def complete(L):
    u, v = np.triu_indices(L, 1)
    return G(f"K{L}", L, np.stack([u, v], 1))


def complete_rows(L):
    """adjacency rows of K_L built directly: every bit below column L except the diagonal"""
    w = (L + 31) // 32
    bits = np.ones((L, w * 32), np.uint8)
    bits[:, L:] = 0
    bits[np.arange(L), np.arange(L)] = 0
    return np.packbits(bits, axis=1, bitorder="little").view(np.uint32).reshape(L, w)


def cocktail_party(n2, rng=None):
    """K_n minus a perfect matching (2i, 2i + 1)"""
    u, v = np.triu_indices(n2, 1)
    keep = ~((u % 2 == 0) & (v == u + 1))
    g = G(f"cocktail{n2}", n2, np.stack([u[keep], v[keep]], 1))
    return g.relabel(rng.permutation(n2)) if rng is not None else g


def paley(q):
    sq = {(x * x) % q for x in range(1, q)}
    e = [(i, j) for i in range(q) for j in range(i + 1, q) if (j - i) % q in sq]
    return G(f"paley{q}", q, e)


def kneser(n, k):
    subs = [frozenset(c) for c in itertools.combinations(range(n), k)]
    e = [(i, j) for i in range(len(subs)) for j in range(i + 1, len(subs)) if not (subs[i] & subs[j])]
    return G(f"kneser{n},{k}", len(subs), e)


def hub_group(rng, m, layout, D=None):
    """A vertex (the hub) whose m neighbours share one degree with 2 * ceil(m / 2) non-neighbours of the same bucket.  A D-regular
    base on N vertices, D > m + 1, so the hub (degree m) is peeled first and its whole neighbour list is one bucket group; the
    members' ids are the lowest of the bucket ("low": every member on its target slot), the highest ("high": every member outside,
    chains through all non-members), or interleaved with the non-members ("mixed")."""
    import networkx as nx
    D = D or m + 2 + (m % 2)
    N = max(3 * m + 40, D + 8)
    N += (N * D) % 2
    base = nx.random_regular_graph(D, N, seed=int(rng.integers(1 << 30)))
    e = [tuple(x) for x in base.edges()]
    k = 2 * ((m + 1) // 2)
    pick = rng.permutation(N)
    members, extra = pick[:m], pick[m:m + k]
    hub = N
    e += [(hub, int(u)) for u in members]
    e += [(int(extra[2 * i]), int(extra[2 * i + 1])) for i in range(k // 2)]   # the non-members join the members' bucket (D + 1)
    L = N + 1
    # ids: the bucket D + 1 = members + extra; the rest keep the remaining ids in random order
    bucket = list(members) + list(extra)
    if layout == "low":
        order = list(members) + list(extra)
    elif layout == "high":
        order = list(extra) + list(members)
    else:
        order = [x for pair in itertools.zip_longest(extra, members) for x in pair if x is not None]
    others = [v for v in range(L) if v not in set(bucket)]
    others = [others[i] for i in rng.permutation(len(others))]
    # bucket members get a block of consecutive ids in the middle of the id range, the others fill around them
    lo = len(others) // 2
    new = np.empty(L, np.int64)
    ids = list(range(L))
    bucket_ids = ids[lo:lo + len(order)]
    rest_ids = ids[:lo] + ids[lo + len(order):]
    for v, i in zip(order, bucket_ids):
        new[v] = i
    for v, i in zip(others, rest_ids):
        new[v] = i
    return G(f"hub{m}-{layout}", L, np.array(e, np.int64)).relabel(new)


def multipartite_rounds(rng, c, seq):
    """Heuristic rounds with chosen winners.  Complete multipartite graphs of w parts of c / (w - 1) vertices, one for every w - 1
    dividing c: each is c-regular, so every vertex has core c, the peel never moves a vertex (order = ids) and the reversed peel order
    runs from the highest id down; a descent from any vertex of the w-partite graph finds w, and the last one (w = c + 1, a clique)
    meets the bound max_core + 1.  seq[k] names the graph of the start vertex with the k-th highest id, so a start vertex improves
    exactly when its w exceeds every w before it: seq fixes which warp of which 8-vertex round wins and where mc reaches ub."""
    import networkx as nx
    ws = [w for w in range(2, c + 2) if c % (w - 1) == 0]
    comps = [nx.complete_multipartite_graph(*([c // (w - 1)] * w)) for w in ws]
    g = nx.disjoint_union_all(comps)
    offs = np.cumsum([0] + [x.number_of_nodes() for x in comps])
    used = [0] * len(ws)
    head = []
    for j in seq:
        head.append(int(offs[j]) + used[j])
        used[j] += 1
    L = g.number_of_nodes()
    hs = set(head)
    rest = [v for v in range(L) if v not in hs]
    order = [rest[i] for i in rng.permutation(len(rest))] + head[::-1]   # order[id] = vertex
    new = np.empty(L, np.int64)
    new[order] = np.arange(L)
    return from_nx(f"rounds{c}:{seq}", g).relabel(new)


def decoy_clique(a, b, rng=None):
    """A = K_a hidden under a decoy D = cocktail party on 2b vertices (K_2b minus a perfect matching: core 2b - 2, cliques of b), each
    vertex of A joined to one private vertex of D, a < 2b - 2.  D's core is the higher, so the reversed peel order starts there and the
    heuristic's incumbent is b; a descent from a vertex of A pops its private D vertex first (the largest (K, id)), which has no other
    neighbour in A, and stops at 2.  The exact search finds the a-clique.  Vertices 0 .. a-1 are A, vertex a + i is the partner of i."""
    assert a < 2 * b - 2
    u, v = np.triu_indices(a, 1)
    cp = cocktail_party(2 * b)
    e = np.concatenate([np.stack([u, v], 1), cp.edges + a, np.stack([np.arange(a), a + np.arange(a)], 1)])
    g = G(f"decoyK{a}/cocktail{2 * b}", a + 2 * b, e)
    return g.relabel(rng.permutation(g.L)) if rng is not None else g


def catalogue_small(seed=2026):
    """The CPU catalogue: every graph here is cheap for the Python restatement."""
    import networkx as nx
    rng = np.random.default_rng(seed)
    gs = []
    for L, d in ((64, 5), (200, 7), (300, 31), (257, 64)):
        gs.append(regular(f"regular{L},{d}", rng, L, d))
    for L, offs in ((97, [1, 3, 7]), (128, [1, 2, 4, 8, 16]), (300, list(range(1, 40)))):
        gs.append(from_nx(f"circulant{L}", nx.circulant_graph(L, offs), rng))
    gs += [cocktail_party(40, rng), cocktail_party(130, rng)]
    gs.append(from_nx("K40,60", nx.complete_bipartite_graph(40, 60), rng))
    gs.append(from_nx("multipartite", nx.complete_multipartite_graph(3, 5, 8, 13, 21, 34), rng))
    gs += [paley(101), paley(197).relabel(rng.permutation(197)), kneser(7, 2), kneser(9, 3).relabel(rng.permutation(84))]
    gs.append(from_nx("friendship20", nx.windmill_graph(20, 3), rng))
    gs.append(from_nx("K40,40", nx.complete_bipartite_graph(40, 40), rng))
    crown = nx.complete_bipartite_graph(40, 40)
    crown.remove_edges_from([(i, 40 + i) for i in range(40)])
    gs.append(from_nx("crown40", crown, rng))
    for m in (1, 31, 32, 33, 63, 64, 65, 100):
        for layout in ("low", "high", "mixed"):
            gs.append(hub_group(rng, m, layout))
    gs += [complete(32), complete(33), complete(1), complete(2), G("empty5", 5, np.zeros((0, 2)))]
    # heuristic rounds: 8 consecutive winners (warp 0) ending on the bound; a warp-7 winner; the bound met mid-round
    gs.append(multipartite_rounds(rng, 24, list(range(8))))
    gs.append(multipartite_rounds(rng, 12, [0] * 8 + [1] + [1] * 4 + [2] + [5]))
    gs.append(multipartite_rounds(rng, 12, [1, 0, 0, 2, 3, 3, 3, 4, 1, 5]))
    gs.append(multipartite_rounds(rng, 24, [0, 1] + [0] * 6 + [2] + [1] * 7 + [3, 4, 7]))
    # the exact search beats the heuristic: planted cliques under higher-core decoys
    gs += [decoy_clique(12, 10, rng), decoy_clique(30, 20, rng), decoy_clique(60, 40)]
    # the heuristic is already maximum but below max_core + 1: the exact search has to prove it with the colour bound
    for n in (3, 4, 5):
        gs.append(from_nx(f"mycielski{n}", nx.mycielski_graph(n), rng))
    for n in (5, 7, 9, 11, 31):
        gs.append(from_nx(f"co-C{n}", nx.complement(nx.cycle_graph(n)), rng))
    # two disjoint maximum cliques that tie on (core, id) order
    two = nx.disjoint_union(nx.complete_graph(9), nx.complete_graph(9))
    gs.append(from_nx("twoK9", two))
    gs.append(from_nx("twoK9-shuffled", two, rng))
    for L, p in ((60, 0.3), (120, 0.5), (200, 0.1), (90, 0.8)):
        gs.append(gnp(f"gnp{L},{p}", rng, L, p))
    return gs


_SMALL = None


def small():
    global _SMALL
    if _SMALL is None:
        _SMALL = [(g, g.rows(), g.nbrs()) for g in catalogue_small()]
    return _SMALL


def restated(g, nb, mode, thr=0.5, node_limit=0, **kw):
    return ref.find_max_clique(g.L, nb, mode, thr, node_limit if node_limit > 0 else DEFAULT_NODE_LIMIT, **kw)


def assert_same(got, want, label):
    """got: (clique, kcore, order, max_core, flags) from the library or the oracle; want: a find_max_clique dict"""
    clique, kcore, order, mc, fl = got
    assert list(kcore) == want["kcore"], (label, "kcore")
    assert list(order) == want["order"], (label, "order")
    assert mc == want["max_core"], (label, "max_core", mc, want["max_core"])
    assert list(clique) == want["clique"], (label, "clique", list(clique)[:20], want["clique"][:20])
    assert fl == want["flags"], (label, "flags", fl, want["flags"])


# ---- CPU: the closed form of the bucket moves ------------------------------------------------------------------------------------------
def _step_state(slots, members_at, others_before=3, others_after=3, lower=2):
    """A peel-step state: a lower bucket (degree 4) of `lower` vertices, then the bucket of degree 5 whose slot s holds member rank
    members_at[s] (or a non-member when None), then `others_after` vertices of degree 6.  Member ids ascend with rank (pmc applies a
    group in list order = id order); non-member ids are spread below, between and above them."""
    n_m = sum(1 for x in members_at if x is not None)
    mem_id = [100 + 10 * r for r in range(n_m)]
    vert, deg = [], {}
    nid = iter(range(1000, 2000))
    for _ in range(lower):
        v = next(nid)
        vert.append(v)
        deg[v] = 4
    for s in range(slots):
        r = members_at[s]
        v = mem_id[r] if r is not None else (95 + 10 * s + 3) if s % 2 else next(nid)
        vert.append(v)
        deg[v] = 5
    for _ in range(others_after):
        v = next(nid)
        vert.append(v)
        deg[v] = 6
    pos = {v: i for i, v in enumerate(vert)}
    bins = {4: 0, 5: lower, 6: lower + slots}
    return vert, pos, bins, deg, mem_id


def test_closed_form_equals_pmc_swaps_on_every_small_bucket():
    """Every bucket of up to 8 slots, every subset of member slots and every placement of the member ranks on them."""
    n = 0
    for slots in range(1, 9):
        for k in range(0, slots + 1):
            for where in itertools.combinations(range(slots), k):
                for ranks in itertools.permutations(range(k)):
                    at = [None] * slots
                    for s, r in zip(where, ranks):
                        at[s] = r
                    vert, pos, bins, deg, nbl = _step_state(slots, at)
                    a = ref.group_moves_sequential(vert, pos, bins, deg, nbl)
                    b = ref.group_moves_closed_form(vert, pos, bins, deg, nbl)
                    assert a == b, (slots, at)
                    n += 1
    assert n == sum(math.comb(s, k) * math.factorial(k) for s in range(1, 9) for k in range(s + 1))


def _random_step(rng, group_sizes, pad):
    """Several buckets, one group each (sizes group_sizes), members scattered among `pad` non-members per bucket, member ids drawn
    so that the groups interleave in the ascending neighbour list."""
    vert, deg, bins, nbl = [], {}, {}, []
    ids = iter(rng.permutation(100000).tolist())
    d = 10
    for m in group_sizes:
        bins[d] = len(vert)
        bucket = [next(ids) for _ in range(m + pad)]
        members = bucket[:m]
        bucket = [bucket[i] for i in rng.permutation(len(bucket))]
        for v in bucket:
            vert.append(v)
            deg[v] = d
        nbl += members
        d += 1
    bins[d] = len(vert)
    pos = {v: i for i, v in enumerate(vert)}
    return vert, pos, bins, deg, sorted(nbl)


def test_closed_form_equals_pmc_swaps_on_random_groups():
    """Groups of 1 ... 100 members; single groups of 31 ... 100 put one group across the 32-neighbour chunks at 32/33, 64/65 and
    96/97; several groups interleave in one list."""
    rng = np.random.default_rng(5)
    cases = [[m] for m in (1, 2, 31, 32, 33, 34, 63, 64, 65, 66, 95, 96, 97, 98, 100)]
    cases += [list(rng.integers(1, 101, int(rng.integers(1, 5)))) for _ in range(400)]
    n_split = 0
    for sizes in cases:
        for pad in (0, 1, 5, 40):
            vert, pos, bins, deg, nbl = _random_step(rng, [int(s) for s in sizes], pad)
            a = ref.group_moves_sequential(vert, pos, bins, deg, nbl)
            b = ref.group_moves_closed_form(vert, pos, bins, deg, nbl)
            assert a == b, (sizes, pad)
            n_split += any(deg[nbl[i]] == deg[nbl[i + 1]] for i in range(31, len(nbl) - 1, 32))
    assert n_split > 100


def test_the_chain_walk_and_the_per_chunk_bin_update_are_needed():
    """Each half of the closed form matters: without the chain walk (the non-member on the member's own target slot takes its old
    slot) or with the bins advanced only after the whole list, the model disagrees with pmc's swaps."""
    rng = np.random.default_rng(6)

    def no_chain(vert, pos, bins, deg, nbl):
        vert, pos, bins, deg = list(vert), dict(pos), dict(bins), dict(deg)
        for c0 in range(0, len(nbl), 32):
            lanes = nbl[c0:c0 + 32]
            du = [deg[u] for u in lanes]
            rank = [sum(1 for j in range(i) if du[j] == du[i]) for i in range(len(lanes))]
            m = [du.count(x) for x in du]
            b0 = [bins[x] for x in du]
            pu = [pos[u] for u in lanes]
            ys = [vert[b0[i] + rank[i]] if pu[i] >= b0[i] + m[i] else None for i in range(len(lanes))]
            for i, u in enumerate(lanes):
                vert[b0[i] + rank[i]], pos[u] = u, b0[i] + rank[i]
                if ys[i] is not None:
                    vert[pu[i]], pos[ys[i]] = ys[i], pu[i]
                deg[u] -= 1
                if rank[i] == 0:
                    bins[du[i]] = b0[i] + m[i]
        return vert, pos, bins, deg

    def whole_list(vert, pos, bins, deg, nbl):
        return ref.group_moves_closed_form(vert, pos, bins, deg, nbl, chunk=10 ** 9)

    caught = {"chain": False, "bins": False}
    for _ in range(200):
        vert, pos, bins, deg, nbl = _random_step(rng, [int(rng.integers(20, 70))], int(rng.integers(1, 30)))
        want = ref.group_moves_sequential(vert, pos, bins, deg, nbl)
        caught["chain"] |= no_chain(vert, pos, bins, deg, nbl) != want
        if len(nbl) > 32:   # a whole-list "chunk" only differs from pmc when the group spans more than one chunk of the kernel
            caught["bins"] |= group_moves_per_list(vert, pos, bins, deg, nbl) != want
    assert caught["chain"] and caught["bins"]


def group_moves_per_list(vert, pos, bins, deg, nbl):
    """kcore_apply_moves with the bin update applied after the whole list instead of per chunk: every chunk reads the bins the
    step started from"""
    vert, pos, deg = list(vert), dict(pos), dict(deg)
    start, after = dict(bins), dict(bins)
    for c0 in range(0, len(nbl), 32):
        vert, pos, b, deg = ref.group_moves_closed_form(vert, pos, start, deg, nbl[c0:c0 + 32])
        after.update({d: x for d, x in b.items() if x != start[d]})
    return vert, pos, after, deg


# ---- CPU: restatement == oracle == networkx --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_restatement_equals_the_oracle_on_the_catalogue(oracle, mode):
    for g, rows, nb in small():
        if g.L:   # the oracle's entry point, like the library's, returns at once for L = 0
            assert_same(oracle.max_clique_ex(rows, mode, 0.5, 0), restated(g, nb, mode), (g.name, mode))


def test_restatement_core_numbers_and_exact_sizes_equal_networkx():
    import networkx as nx
    for g, rows, nb in small():
        gx = g.nx()
        want = restated(g, nb, PMC_EXACT)
        cn = nx.core_number(gx)
        assert [want["kcore"][v] - 1 for v in range(g.L)] == [cn[v] for v in range(g.L)], g.name
        c = want["clique"]
        assert all(gx.has_edge(a, b) for a, b in itertools.combinations(c, 2)), g.name
        if 0 < g.L <= 100 and not g.name.startswith(("cocktail", "crown")):   # cocktail parties have 2^(L/2) maximal cliques
            omega = len(nx.max_weight_clique(gx, weight=None)[0]) if g.edges.size else 0
            assert len(c) == omega, g.name


def test_the_catalogue_reaches_the_heuristic_cases():
    """The heuristic-round graphs do what they are for: consecutive start vertices improve (winner warp 0, runs of 2 ... 8), an
    improvement 7 positions after the previous one (warp 7), mc reaches ub in the middle of a round, and the exact search beats
    the heuristic on every decoy graph."""
    winners, ub_mid, beaten, run = set(), False, set(), 0
    for g, rows, nb in small():
        K, order, max_core = ref.pmc_cores(g.L, nb)
        hits = []
        ref.pmc_heu(g.L, nb, K, order, max_core + 1, trace=hits)
        best_run, cur = 0, 0
        prev = g.L   # the first round starts at L - 1
        for i, mc in hits:
            w = (prev - 1 - i) % 8
            winners.add(w)
            cur = cur + 1 if prev - 1 == i else 1
            best_run = max(best_run, cur)
            prev = i
            if mc >= max_core + 1 and w != 7:
                ub_mid = True
        run = max(run, best_run)
        w = restated(g, nb, PMC_EXACT)
        if len(w["clique"]) > w["heu"]:
            beaten.add(g.name)
    decoys = {g.name for g, _, _ in small() if g.name.startswith("decoy")}
    assert {0, 7} <= winners and run >= 8 and ub_mid and len(decoys) == 3 and decoys <= beaten, (winners, run, ub_mid, beaten)


# ---- CPU: KCORE_HEU thresholds ------------------------------------------------------------------------------------------------------------
def threshold_cases(L, max_core):
    """thresholds around the cut-off of a graph with L vertices and this max core, and values the int cast cannot hold"""
    t = [max_core / L, (max_core + 1) / L, (max_core - 1) / L, np.nextafter(max_core / L, 0), np.nextafter((max_core + 1) / L, 2),
         0.29, 1.0, 1 - 2.0 ** -53, 0.0, -0.0, -0.5, -1e-300, float("nan"), float("inf"), float("-inf"), 1e300, -1e300,
         2.0 ** 31 / L, (2.0 ** 31 - 1) / L, np.nextafter(2.0 ** 31 / L, 0), -(2.0 ** 31) / L, -(2.0 ** 31 + 1) / L, 1e10, -1e10]
    return [float(x) for x in t]


def test_kcore_heu_limit_is_the_x86_conversion():
    assert ref.kcore_heu_limit(0.29, 100) == 28              # 0.29 * 100 = 28.999999999999996
    assert ref.kcore_heu_limit(0.5, 100) == 50
    assert ref.kcore_heu_limit(-0.5, 3) == -1                 # truncation toward zero
    for thr in (float("nan"), float("inf"), float("-inf"), 1e300, -1e300, 2.0 ** 31, -(2.0 ** 31) - 1):
        assert ref.kcore_heu_limit(thr, 1) == -2 ** 31
    assert ref.kcore_heu_limit(2.0 ** 31 - 1, 1) == 2 ** 31 - 1
    assert ref.kcore_heu_limit(-(2.0 ** 31), 1) == -2 ** 31
    assert ref.kcore_heu_limit(-(2.0 ** 31) - 0.5, 1) == -2 ** 31


def threshold_graphs():
    rng = np.random.default_rng(41)
    return [gnp("thr-gnp100", rng, 100, 0.3), complete(29), cocktail_party(40, rng), G("edgeless7", 7, np.zeros((0, 2))),
            regular("thr-regular60", rng, 60, 9)]


def test_kcore_heu_thresholds_on_the_oracle(oracle):
    for g in threshold_graphs():
        rows, nb = g.rows(), g.nbrs()
        mc = ref.pmc_cores(g.L, nb)[2]
        shortcut = set()
        for thr in threshold_cases(g.L, mc):
            want = restated(g, nb, KCORE_HEU, thr)
            assert_same(oracle.max_clique_ex(rows, KCORE_HEU, thr, 0), want, (g.name, thr))
            shortcut.add(mc > ref.kcore_heu_limit(thr, g.L) and thr != 1)
        assert shortcut == {True, False}, g.name


# ---- GPU --------------------------------------------------------------------------------------------------------------------------------
HANDLE_SIZES = (1024, 2048, 4096, 8192, 16384, 32768)


def wpl(Lc):
    """clique.cu launch_clique: the WPL instance of a handle of max_corr Lc (W = Lc / 32 words per row)"""
    W = Lc // 32
    return next(w for lim, w in ((32, 1), (64, 2), (128, 4), (256, 8), (512, 16)) if W <= lim) if W <= 512 else 32


def clique_cu_constant(name):
    """a constant of clique.cu as the launch code uses it (the switches below follow the source, not copies of its numbers)"""
    import re
    from support import ROOT
    src = (ROOT / "quatro_b200" / "csrc" / "clique.cu").read_text()
    m = re.search(r"(?:constexpr (?:int|size_t)|const int) " + name + r" = ([0-9* ]+);", src)
    assert m, name
    return eval(m.group(1), {})


def kcore_row_cache_switch(Lc):
    """The largest L whose whole adjacency kcore_kernel caches in shared memory (launch_kcore: row_words from kKcoreSmemBudget minus
    the fixed arrays, clamped to [kRing * Ws, Ls * Ws]; kcore_kernel: cached <=> L * ceil(L / 32) <= row_words)."""
    Ls = min(Lc, 8192)
    Ws = Ls // 32
    warps, ring, budget = clique_cu_constant("kKcWarps"), clique_cu_constant("kRing"), clique_cu_constant("kKcoreSmemBudget")
    bits = 3 * warps * 32 * wpl(Lc) * 4
    fixed = (Ls + 2) * 4 + bits + (4 + warps) * Ls * 2
    row_words = (budget - fixed) // 4 if fixed + 8 * 1024 < budget else 0
    row_words = min(max(row_words, ring * Ws), Ls * Ws)
    L = 1
    while L + 1 <= Ls and (L + 1) * ((L + 32) // 32) <= row_words:
        L += 1
    return L


def descent_cache_switch():
    """clique_cta_kernel / clique_exact_kernel: the rank-space adjacency is cached while L * ceil(L / 32) <= cache_words (launch_clique)"""
    words = clique_cu_constant("cache_words")
    L = 1
    while (L + 1) * ((L + 32) // 32) <= words:
        L += 1
    return L


# clique_descent<WPL>: ceil(L / 32) words over 32 lanes -> nwl = 1, <= 4, <= 8, <= 16, else 32: switches at ceil(L / 32) = 32 / 33,
# 128 / 129, 256 / 257, 512 / 513
DESCENT_WIDTH_SWITCHES = (32 * 32, 128 * 32, 256 * 32, 512 * 32)
SMEM_VERTS = 8192   # kKcoreSmemVerts: graphs above it keep their k-core arrays and chains in global scratch


def switch_graphs(rng, L0, Lc, dense_ok):
    out = []
    for L in (L0 - 1, L0, L0 + 1):
        if L < 2 or L > Lc:
            continue
        out.append(sparse(f"sparse{L}", rng, L, 8))
        out.append(regular(f"regular{L}", rng, L, 16 if L > 2000 else 40 if L > 200 else 6))
        if dense_ok and L <= 1100:
            out.append(gnp(f"dense{L}", rng, L, 0.5))
    return out


def handle_graphs(Lc, rng):
    """graphs of one handle: every switch of this handle +-1 and the small catalogue where it fits"""
    gs = []
    for L0 in sorted({kcore_row_cache_switch(Lc), descent_cache_switch()}):
        gs += switch_graphs(rng, L0, Lc, True)
    for L0 in DESCENT_WIDTH_SWITCHES:
        if L0 + 1 <= Lc:
            gs += switch_graphs(rng, L0, Lc, False)
    if Lc > SMEM_VERTS:
        gs += switch_graphs(rng, SMEM_VERTS, Lc, False)
    return gs


def device_vs_restatement(h, g, modes=MODES, thr=0.5, node_limit=0):
    rows, nb = g.rows(), g.nbrs()
    for mode in modes:
        want = restated(g, nb, mode, thr, node_limit)
        assert_same(h.max_clique_ex(rows, mode, thr, node_limit), want, (g.name, g.L, mode))


@pytest.mark.gpu
def test_device_equals_the_restatement_on_the_catalogue():
    h = make_handle(1, max_batch_slots=1, max_corr=1024)
    try:
        for g, rows, nb in small():
            for mode in MODES:
                want = restated(g, nb, mode)
                if g.L:
                    assert_same(h.max_clique_ex(rows, mode, 0.5, 0), want, (g.name, mode))
    finally:
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("Lc", HANDLE_SIZES)
def test_device_equals_the_restatement_at_every_switch(Lc):
    rng = np.random.default_rng(Lc)
    h = make_handle(1, max_batch_slots=1, max_corr=Lc)
    try:
        gs = handle_graphs(Lc, rng)
        small_here = [g for g, _, _ in small() if g.L <= Lc][:: max(1, Lc // 4096)]
        for g in gs:   # the exact search only where the Python restatement stays cheap
            device_vs_restatement(h, g, modes=MODES if g.L <= 1100 and not g.name.startswith("dense") else (PMC_HEU, KCORE_HEU))
        for g in small_here:
            device_vs_restatement(h, g)
        # complete graphs: the closed form (no vertex is ever decremented: identity order, every core L - 1, the clique is all)
        for n in (32, 33, 674, 675, 4096, 8192):
            if n <= Lc:
                c, k, o, mc, fl = h.max_clique_ex(complete_rows(n), PMC_EXACT, 0.5, 0)
                assert list(c) == list(range(n)) and (k == n).all() and list(o) == list(range(n)) and mc == n - 1 and fl == 0, n
        if Lc == 32768:   # a hub of degree 32767 over a sparse graph
            g = sparse("hub32767", rng, 32768, 4)
            g = G("hub32767", 32768, np.concatenate([g.edges, np.stack([np.zeros(32767, np.int64), np.arange(1, 32768)], 1)]))
            device_vs_restatement(h, g, modes=(PMC_HEU,))
    finally:
        h.close()


@pytest.mark.gpu
def test_node_limits_around_the_restatements_count():
    h = make_handle(1, max_batch_slots=1, max_corr=1024)
    try:
        tried = 0
        for g, rows, nb in small():
            w = restated(g, nb, PMC_EXACT)
            n = w["nodes"]
            if n < 2:
                continue
            tried += 1
            for lim in (n - 1, n, n + 1, 1):
                want = restated(g, nb, PMC_EXACT, node_limit=lim)
                assert (want["flags"] == TRUNCATED) == (lim < n), (g.name, lim, n)
                assert_same(h.max_clique_ex(rows, PMC_EXACT, 0.5, lim), want, (g.name, lim))
        assert tried >= 3
    finally:
        h.close()


@pytest.mark.gpu
def test_kcore_heu_thresholds_on_the_device():
    h = make_handle(1, max_batch_slots=1, max_corr=1024)
    try:
        for g in threshold_graphs():
            rows, nb = g.rows(), g.nbrs()
            mc = ref.pmc_cores(g.L, nb)[2]
            for thr in threshold_cases(g.L, mc):
                want = restated(g, nb, KCORE_HEU, thr)
                assert_same(h.max_clique_ex(rows, KCORE_HEU, thr, 0), want, (g.name, thr))
    finally:
        h.close()


def stray(rows, L, extra, rng):
    """rows with `extra` random padding words and random bits at columns L ... 32 * ceil(L / 32) - 1"""
    n, w = rows.shape
    out = np.zeros((n, w + extra), np.uint32)
    out[:, :w] = rows
    out[:, w:] = rng.integers(0, 2 ** 32, (n, extra), dtype=np.uint64).astype(np.uint32)
    if L % 32:
        junk = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32) & np.uint32(~((1 << (L % 32)) - 1) & 0xFFFFFFFF)
        junk[0] |= np.uint32(1 << 31)
        out[:, w - 1] |= junk
    return out


@pytest.mark.gpu
def test_stray_bits_past_column_L_are_ignored(oracle):
    rng = np.random.default_rng(77)
    h = make_handle(1, max_batch_slots=4, max_corr=2048)
    try:
        gs = [gnp("gnp45", rng, 45, 0.3), gnp("gnp100", rng, 100, 0.2), regular("reg333", rng, 333, 12), cocktail_party(40, rng),
              sparse("sparse1000", rng, 1000, 10), hub_group(rng, 33, "mixed"), G("edgeless37", 37, np.zeros((0, 2)))]
        for g in gs:
            clean, nb = g.rows(), g.nbrs()
            for extra in (0, 2):
                dirty = stray(clean, g.L, extra, rng)
                for mode in MODES:
                    want = restated(g, nb, mode)
                    label = (g.name, extra, mode)
                    assert_same(h.max_clique_ex(dirty, mode, 0.5, 0), want, label + ("single",))
                    assert_same(oracle.max_clique_ex(dirty, mode, 0.5, 0), want, label + ("oracle",))
                    p = default_params()
                    p.inlier_selection_mode = mode
                    recs, lists = h.max_clique_batch_each([dirty], [p], buffers=ListBuffers(1, g.L, MEM_HOST, GRAPH_LISTS))
                    assert recs[0]["max_core"] == want["max_core"] and list(lists[0]["clique"]) == want["clique"], label + ("batch",)
                    assert recs[0]["n_edges"] == len(g.edges), label + ("batch",)
    finally:
        h.close()


# The device-only stops of clique_exact_kernel: a planted clique under a cocktail-party decoy (decoy_clique), the heuristic's b
# below the clique's a.  Inside the clique a level's colour list holds the entries of the a - b highest colours, and a child list
# starts on its parent's consumed entry, so the lists on the path grow by at most a - b - 1 pool entries per level:
#   pool:  a = 600, b = 310: the restatement with the device's limits runs out of the 2^17-entry pool at depth 560;
#   depth: a = 1030, b = 930: 1023 levels hold at most 1023 * 99 = 101 277 < 2^17 entries, so the 1024-level stack stops first.
# The depth graph's search (about 10^9 set operations in the Python restatement) is not restated; its device result is pinned by
# what the stop must leave: the flag, and the heuristic clique, which no clique up to depth 1024 can beat before the stop.
EXACT_DEPTH, EXACT_POOL = 1024, 1 << 17   # clique.cu: kExactDepth, kExactPool
STOP_GRAPHS = {"pool": (600, 310), "depth": (1030, 930)}
_POOL = []


def pool_case():
    """(graph, rows, restatement with the device's limits) of the pool-stop graph, computed once per session"""
    if not _POOL:
        g = decoy_clique(*STOP_GRAPHS["pool"])
        _POOL.append((g, g.rows(), restated(g, g.nbrs(), PMC_EXACT, depth_limit=EXACT_DEPTH, pool_limit=EXACT_POOL)))
    return _POOL[0]


def test_the_pool_graph_reaches_the_pool_stop(oracle):
    """With the device's limits the restatement runs out of the list pool (not the stack) inside the planted clique, keeps the
    heuristic clique and flags the truncation; the oracle, which has neither limit, finds the planted clique without the flag."""
    g, rows, want = pool_case()
    a, b = STOP_GRAPHS["pool"]
    st = want["stop"]
    assert want["flags"] == TRUNCATED and want["heu"] == b and len(want["clique"]) == b, want["stop"]
    assert st["reason"] == "pool" and st["depth"] < EXACT_DEPTH - 1 and st["pool"] > EXACT_POOL - (a - b), st
    oc, _, _, _, ofl = oracle.max_clique_ex(rows, PMC_EXACT, 0.5, 0)
    assert ofl == 0 and list(oc) == list(range(a))


def test_the_depth_graph_fits_the_pool():
    a, b = STOP_GRAPHS["depth"]
    assert (EXACT_DEPTH - 1) * (a - b - 1) + a < EXACT_POOL and a > EXACT_DEPTH


@pytest.mark.gpu
def test_device_pool_stop_equals_the_restatement():
    """qb200_max_clique_ex stops with QB200_FLAG_CLIQUE_TRUNCATED and exactly the restatement's result under the same limits."""
    g, rows, want = pool_case()
    h = make_handle(1, max_batch_slots=1, max_corr=4096)
    try:
        got = h.max_clique_ex(rows, PMC_EXACT, 0.5, 0)
        assert got[4] == TRUNCATED
        assert_same(got, want, g.name)
    finally:
        h.close()


@pytest.mark.gpu
def test_device_depth_stop(oracle):
    """The 1030-clique needs 1030 levels: the device stops at the 1024-level stack with the flag and the heuristic's clique, while the
    oracle finds the planted clique without the flag.  Cores and order are restated; the heuristic clique (1860 descents of up to 930
    steps, too slow in Python) is the oracle's, which the catalogue tests pin to the restatement."""
    a, b = STOP_GRAPHS["depth"]
    g = decoy_clique(a, b)
    rows = g.rows()
    K, order, max_core = ref.pmc_cores(g.L, g.nbrs())
    hc, hk, ho, hmc, _ = oracle.max_clique_ex(rows, PMC_HEU, 0.5, 0)
    assert list(hk) == K and list(ho) == order and hmc == max_core and len(hc) == b
    heu = dict(kcore=K, order=order, max_core=max_core, clique=list(hc))
    h = make_handle(1, max_batch_slots=1, max_corr=4096)
    try:
        got = h.max_clique_ex(rows, PMC_EXACT, 0.5, 0)
    finally:
        h.close()
    assert_same(got, dict(heu, flags=TRUNCATED), g.name)
    oc, _, _, _, ofl = oracle.max_clique_ex(rows, PMC_EXACT, 0.5, 0)
    assert ofl == 0 and list(oc) == list(range(a))


@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 4])
def test_mixed_wave_equals_the_single_call(lanes):
    """The catalogue in one call of qb200_max_clique_batch_each, every mode, per-graph thresholds and node limits: each record's
    max_core, clique size, flags and clique byte-identical to qb200_max_clique_ex."""
    h = make_handle(lanes, max_batch_slots=8, max_corr=1024)
    try:
        graphs, params, want = [], [], []
        for k, (g, rows, nb) in enumerate(small()):
            mode = MODES[k % 3]
            thr = (0.5, 0.1, float("inf"), 0.9, float("nan"), 1.0)[k % 6]
            lim = (0, 1, 7, 100)[k % 4]
            p = default_params()
            p.inlier_selection_mode, p.kcore_heuristic_threshold, p.max_clique_node_limit = mode, thr, lim
            graphs.append(rows if g.L else (0, np.zeros((0, 2), np.int32)))
            params.append(p)
            want.append(h.max_clique_ex(rows, mode, thr, lim) if g.L else None)
        recs, lists = h.max_clique_batch_each(graphs, params, buffers=ListBuffers(len(graphs), 1024, MEM_HOST, GRAPH_LISTS))
        for i, w in enumerate(want):
            if w is None:
                continue
            c, _, _, mc, fl = w
            assert recs[i]["status"] == 0 and recs[i]["max_core"] == mc and recs[i]["flags"] == fl, i
            assert recs[i]["clique_size"] == len(c) and lists[i]["clique"].tobytes() == np.asarray(c, np.int32).tobytes(), i
    finally:
        h.close()
