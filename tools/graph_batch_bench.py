"""What building TIM graphs in batches buys: qb200_build_graph_batch_each against the per-set qb200_build_graph loop it replaces.

Three workloads of host-memory correspondence sets:
  street  the matched points of 256 street pairs (synth.outdoor_pair, seeds 0..255, default front end and params), matched with
          qb200_match_batch_mixed (untimed) on a default handle (max_corr 4096, 64 slots);
  8192    8 sets of 8192 matched points (synth.matched_pairs) on a handle of max_corr 32768 and 2 slots;
  32768   2 sets of 32768 matched points on the same handle.
Every set is built with the default noise_bound and cbar2, four ways: the loop of qb200_build_graph (adjacency rows, degrees and edge
count into host memory, one synchronisation per set), and one batch call with host-kind adjacency rows and degrees (what the loop
produces), with device-kind rows and degrees, and with device-kind edge lists.  All four are warmed up first, the rounds alternate them,
and each is timed with the host clock after a device synchronise.  After every round (outside the timed region) the batch outputs are
compared with the loop's byte for byte; an edge list is checked to hold n_edges strictly ascending pairs (u, v), u < v, each of them an
edge of the loop's matrix.  Prints one JSON line with the card and its power limit, and exits 1 on any difference.

  python tools/graph_batch_bench.py [--pairs 256] [--rounds 5] [--warmup 2]
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


def edges_match(edges, n_edges, adj_dev, L):
    """edges (cap, 2) int32 on the device holds exactly the n_edges upper edges of adj_dev (L, words) in ascending (u, v) order"""
    import torch
    e = edges[:n_edges].long()
    u, v = e[:, 0], e[:, 1]
    if n_edges == 0:
        return True
    key = u * L + v
    bits = (adj_dev[u, v >> 5].long() >> (v & 31)) & 1
    return bool((u < v).all() and (v < L).all() and (key[1:] > key[:-1]).all() and (bits == 1).all()) and \
        int(torch.count_nonzero(edges[n_edges:] != 0x5A5A5A5A)) == 0


def workload(h, sets, p, warmup, rounds):
    import torch
    from quatro_b200.capi import MEM_DEVICE, MEM_HOST, GraphBuffers
    n = len(sets)
    Ls = [len(a) for a, _ in sets]
    rows = max(Ls)
    wpr = (rows + 31) // 32
    params = [p] * n
    state = {}

    def loop():
        state["loop"] = [h.build_graph(a, b, p.noise_bound, p.cbar2, wpr) for a, b in sets]

    loop()
    cap = max(max(ne for _, _, ne in state["loop"]), 1)
    bufs = {"host_adj": GraphBuffers(n, rows, wpr, 1, MEM_HOST, ("adj", "degree")),
            "device_adj": GraphBuffers(n, rows, wpr, 1, MEM_DEVICE, ("adj", "degree")),
            "device_edges": GraphBuffers(n, 0, 0, cap, MEM_DEVICE, ("edges",), fill=0x5A5A5A5A)}

    def batch(name):
        def run():
            state[name] = h.build_graph_batch_each(sets, params, MEM_HOST, bufs[name])
            torch.cuda.synchronize()
        return run

    def same():
        ok = True
        ref = state["loop"]
        host_adj, host_deg = bufs["host_adj"].host("adj"), bufs["host_adj"].host("degree")
        dev_adj, dev_deg = bufs["device_adj"].host("adj"), bufs["device_adj"].host("degree")
        for i, (adj, deg, ne) in enumerate(ref):
            L = Ls[i]
            for recs in (state["host_adj"], state["device_adj"], state["device_edges"]):
                ok &= int(recs[i]["n_edges"]) == ne and int(recs[i]["n_corr"]) == L and int(recs[i]["flags"]) == 0
            ok &= host_adj[i, :L].tobytes() == adj.tobytes() and host_deg[i, :L].tobytes() == deg.tobytes()
            ok &= dev_adj[i, :L].tobytes() == adj.tobytes() and dev_deg[i, :L].tobytes() == deg.tobytes()
            ok &= edges_match(bufs["device_edges"].arrays["edges"][i], ne, bufs["device_adj"].arrays["adj"][i], L)
        return ok

    out, ok = timed({"loop": loop, **{k: batch(k) for k in bufs}}, warmup, rounds, {"device_edges": same})
    for k in bufs:
        out[k]["speedup"] = out["loop"]["median"] / out[k]["median"]
    out["sets"] = n
    out["L_mean"] = float(np.mean(Ls))
    out["edges_mean"] = float(np.mean([ne for _, _, ne in state["loop"]]))
    return out, ok["device_edges"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    from quatro_b200 import synth
    from quatro_b200.capi import MATCH_LISTS, Handle, ListBuffers, default_params

    p = default_params()
    res, ok = {}, True
    with Handle() as h:
        pairs = [synth.outdoor_pair(s)[:2] for s in range(args.pairs)]
        _, ml = h.match_batch_mixed(pairs, [p] * len(pairs), buffers=ListBuffers(len(pairs), h.cfg.max_corr, 0, MATCH_LISTS))
        sets = [(m["src_matched4"], m["tgt_matched4"]) for m in ml]
        res["street"], same = workload(h, sets, p, args.warmup, args.rounds)
        ok &= same
    with Handle(max_batch_slots=2, max_corr=32768) as h:
        for L, n in ((8192, 8), (32768, 2)):
            sets = [synth.matched_pairs(100 + s, L)[:2] for s in range(n)]
            res[str(L)], same = workload(h, sets, p, args.warmup, args.rounds)
            ok &= same
    print(json.dumps({"card": card(), "rounds": args.rounds, "workloads": res, "outputs_equal": bool(ok)}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
