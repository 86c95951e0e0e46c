"""What solving caller inlier sets in batches buys: qb200_solve_pose_batch_each against the per-set qb200_solve_pose loop it replaces.

Three workloads:
  street  the 256 correspondence sets of street pairs (synth.outdoor_pair, seeds 0..255, default front end and params), matched with
          qb200_match_batch_mixed, and the cliques qb200_solve_batch_ex lists for them (untimed), on a default handle (max_corr 4096,
          64 slots);
  8192    8 random scenes of 9000 matched points (30 % outliers, random yaw and translation) with an ascending 8192-member subset as
          the inlier list, on a handle of max_corr 32768 and 2 slots;
  32768   2 such scenes of 32768 points whose inlier list is every id, on the same handle.
Each workload is solved with the default params (rot_noise_bound 2 noise_bound) three ways: the batch call with host-kind inputs, the
batch call with the points and ids already in device memory, both with host-kind lists (clique, final inliers, both masks), and the
loop of qb200_solve_pose (record and both masks), which copies, launches and synchronises per set.  All are warmed up first and the
rounds alternate them; each is timed with the host clock.  After every timed batch (outside the timed region) its records and masks
are compared with the loop's byte for byte.  Prints one JSON line with the card and its power limit, and exits 1 if anything differs.

  python tools/pose_batch_bench.py [--pairs 256] [--rounds 5] [--warmup 2]
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


def scene(rng, L, c):
    """L matched {x,y,z,1} points (30 % outliers) and an ascending c-subset of their ids"""
    yaw = rng.uniform(-np.pi, np.pi)
    R = np.array([[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]])
    a = rng.uniform(-40, 40, (L, 3)) * [1, 1, 0.1]
    b = a @ R.T + [12.0, -7.0, 1.0] + rng.normal(0, 0.02, (L, 3))
    out = rng.random(L) < 0.3
    b[out] = rng.uniform(-40, 40, (int(out.sum()), 3)) * [1, 1, 0.1]
    a4, b4 = np.ones((L, 4), np.float32), np.ones((L, 4), np.float32)
    a4[:, :3], b4[:, :3] = a, b
    return (a4, b4), np.sort(rng.choice(L, c, replace=False)).astype(np.int32)


def workload(h, sets, inliers, p, warmup, rounds):
    import torch
    from quatro_b200.capi import MEM_DEVICE, MEM_HOST, SET_LISTS, ListBuffers
    n = len(sets)
    params = [p] * n
    lb = ListBuffers(n, max(1, max(len(i) for i in inliers)), MEM_HOST, SET_LISTS)
    keep = [(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda(), torch.from_numpy(np.ascontiguousarray(i)).cuda())
            for (a, b), i in zip(sets, inliers)]
    torch.cuda.synchronize()
    dsets = [(ta.data_ptr(), tb.data_ptr(), len(ta)) for ta, tb, _ in keep]
    dids = [(ti.data_ptr(), len(ti)) for _, _, ti in keep]
    state = {}

    def batch(kind):
        def run():
            ss, ii = (sets, inliers) if kind == MEM_HOST else (dsets, dids)
            state["batch"] = h.solve_pose_batch_each(ss, ii, params, kind, lb)
        return run

    def loop():
        state["loop"] = [h.solve_pose(a, b, i, p)[:3] for (a, b), i in zip(sets, inliers)]

    def keep_batch():
        recs, lists = state["batch"]
        state["last"] = (recs.copy(), [{k: v.copy() for k, v in d.items()} for d in lists])
        return True

    def same():
        ok = True
        recs, lists = state["last"]
        for r, d, (res, rm, tm) in zip(recs, lists, state["loop"]):
            ok &= r.tobytes() == bytes(res) and d["rot_inlier_mask"].tobytes() == rm.tobytes()
            ok &= d["trans_inlier_mask"].tobytes() == tm.tobytes()
        return ok

    out, ok = timed({"batch_host": batch(MEM_HOST), "batch_device": batch(MEM_DEVICE), "loop": loop}, warmup, rounds,
                    {"batch_host": keep_batch, "batch_device": keep_batch, "loop": same})
    for k in ("batch_host", "batch_device"):
        out[k]["speedup"] = out["loop"]["median"] / out[k]["median"]
    out["sets"] = n
    out["inliers_mean"] = float(np.mean([len(i) for i in inliers]))
    out["points_mean"] = float(np.mean([len(a) for a, _ in sets]))
    del keep
    return out, ok["loop"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    from quatro_b200 import synth
    from quatro_b200.capi import MATCH_LISTS, SET_LISTS, Handle, ListBuffers, default_params

    p = default_params()
    p.rot_noise_bound = 2 * p.noise_bound
    res, ok = {}, True
    with Handle() as h:
        pairs = [synth.outdoor_pair(s)[:2] for s in range(args.pairs)]
        _, ml = h.match_batch_mixed(pairs, [p] * len(pairs), buffers=ListBuffers(len(pairs), h.cfg.max_corr, 0, MATCH_LISTS))
        sets = [(m["src_matched4"], m["tgt_matched4"]) for m in ml]
        _, sl = h.solve_batch_lists(sets, p, buffers=ListBuffers(len(sets), h.cfg.max_corr, 0, SET_LISTS))
        res["street"], same = workload(h, sets, [d["clique"] for d in sl], p, args.warmup, args.rounds)
        ok &= same
    rng = np.random.default_rng(0)
    with Handle(max_batch_slots=2, max_corr=32768) as h:
        for L, c, n in ((9000, 8192, 8), (32768, 32768, 2)):
            made = [scene(rng, L, c) for _ in range(n)]
            res[str(c)], same = workload(h, [s for s, _ in made], [i for _, i in made], p, args.warmup, args.rounds)
            ok &= same
    print(json.dumps({"card": card(), "rounds": args.rounds, "workloads": res, "records_equal": bool(ok)}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
