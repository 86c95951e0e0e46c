"""What solving caller graphs in batches buys: qb200_max_clique_batch_each against the per-graph qb200_max_clique_ex loop it replaces.

Three workloads, each as host-memory adjacency rows:
  street  the TIM graphs of 256 street pairs (synth.outdoor_pair, seeds 0..255, default front end and params): the pairs are matched
          with qb200_match_batch_mixed and each correspondence set's graph is built with qb200_build_graph (untimed), on a default
          handle (max_corr 4096, 64 slots);
  8192    8 random graphs of 8192 vertices (average degree 24, a planted 16-clique) on a handle of max_corr 32768 and 2 slots;
  32768   2 random graphs of 32768 vertices (average degree 12, a planted 16-clique) on the same handle.
Each workload is solved in the default mode (PMC_HEU, k-core threshold 0.5) two ways: one batch call, and the loop of
qb200_max_clique_ex, which clears, copies and synchronises once per graph.  Both are warmed up first and the rounds alternate them; each
is timed with the host clock.  After every timed batch (outside the timed region) its cliques are compared with the loop's.  Prints one
JSON line with the card and its power limit, and exits 1 if any clique differs.

  python tools/clique_batch_bench.py [--pairs 256] [--rounds 5] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

from harness import card, timed

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def random_adj(rng, L, deg, k=16):
    m = L * deg // 2
    u, v = rng.integers(0, L, m), rng.integers(0, L, m)
    mem = rng.choice(L, k, replace=False)
    a, b = np.triu_indices(k, 1)
    u, v = np.concatenate([u, mem[a], v, mem[b]]), np.concatenate([v, mem[b], u, mem[a]])
    keep = u != v
    u, v = u[keep], v[keep]
    W = (L + 31) // 32
    adj = np.zeros(L * W, np.uint32)
    np.bitwise_or.at(adj, u * W + (v >> 5), np.uint32(1) << (v & 31).astype(np.uint32))
    return adj.reshape(L, W)


def workload(h, graphs, p, warmup, rounds):
    from quatro_b200.capi import GRAPH_LISTS, ListBuffers
    params = [p] * len(graphs)
    lb = ListBuffers(len(graphs), h.cfg.max_corr, 0, GRAPH_LISTS)
    mode, thr = p.inlier_selection_mode, p.kcore_heuristic_threshold
    state = {}

    def batch():
        state["batch"] = h.max_clique_batch_each(graphs, params, buffers=lb)

    def loop():
        state["loop"] = [h.max_clique_ex(a, mode, thr)[0] for a in graphs]

    def same():
        _, lists = state["batch"]
        return all(d["clique"].tobytes() == c.astype(np.int32).tobytes() for d, c in zip(lists, state["loop"]))

    out, ok = timed({"batch": batch, "loop": loop}, warmup, rounds, {"loop": same})
    out["speedup"] = out["loop"]["median"] / out["batch"]["median"]
    out["graphs"] = len(graphs)
    out["vertices_mean"] = float(np.mean([a.shape[0] for a in graphs]))
    return out, ok["loop"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    from quatro_b200 import synth
    from quatro_b200.capi import MATCH_LISTS, Handle, ListBuffers, default_params

    p = default_params()
    p.rot_noise_bound = 2 * p.noise_bound
    res, ok = {}, True
    with Handle() as h:
        pairs = [synth.outdoor_pair(s)[:2] for s in range(args.pairs)]
        _, ml = h.match_batch_mixed(pairs, [p] * len(pairs), buffers=ListBuffers(len(pairs), h.cfg.max_corr, 0, MATCH_LISTS))
        graphs = [h.build_graph(m["src_matched4"], m["tgt_matched4"], p.noise_bound, p.cbar2)[0] for m in ml]
        res["street"], same = workload(h, graphs, p, args.warmup, args.rounds)
        ok &= same
    rng = np.random.default_rng(0)
    with Handle(max_batch_slots=2, max_corr=32768) as h:
        for L, n, deg in ((8192, 8, 24), (32768, 2, 12)):
            res[str(L)], same = workload(h, [random_adj(rng, L, deg) for _ in range(n)], p, args.warmup, args.rounds)
            ok &= same
    print(json.dumps({"card": card(), "rounds": args.rounds, "workloads": res, "cliques_equal": bool(ok)}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
