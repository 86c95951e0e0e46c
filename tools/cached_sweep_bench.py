"""What the lane rotation buys a loop-closure sweep of cached scans, and a multi-wave batch of correspondence sets.

Sweep: bench.py's street scans (synth.outdoor_pair, seeds 0..31: 64 scans of 32 scenes, two poses each, device-resident) are cached
once, and every pair (i, j), 0 < j - i <= --window, of the 64 scans is registered with bench.py's street preset: 1 988 pairs at the
default window of 56.  Most of them pair two different scenes, as most candidates of a real loop-closure sweep are false loops.  Four
schedules of the same pairs:
  cached_lanes1  one blocking qb200_register_cached call on a handle created with QB200_LANES=1;
  cached_lanes   the same call on a handle with the default lanes;
  cached_stream  qb200_register_cached_enqueue_mixed batches of --batch pairs on the default handle, one flush at the end;
  uncached       one qb200_register_batch call of the same pairs from the device-resident raw scans (front end every pair).
Sets: --sets synthetic correspondence sets (synth.matched_pairs, 300 .. 2 500 correspondences, device-resident) solved as
  solve_lanes1 / solve_lanes (blocking qb200_solve_batch on either handle) and solve_stream (qb200_solve_batch_enqueue_each batches,
  one flush).
Every schedule is warmed up first and the rounds alternate them; each is timed with the host clock around calls that end with every
lane synchronised.  The records of the schedules of one input are compared byte for byte.  Prints one JSON line with the card and its
power limit, ms per schedule (median, min, max) and pairs per second.

  python tools/cached_sweep_bench.py [--rounds 5] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from pathlib import Path

import numpy as np

from harness import card, timed

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def handle(lanes, **cfg):
    from quatro_b200.capi import Handle
    old = os.environ.pop("QB200_LANES", None)
    if lanes:
        os.environ["QB200_LANES"] = str(lanes)   # read when the handle is created
    try:
        return Handle(**cfg)
    finally:
        os.environ.pop("QB200_LANES", None)
        if old is not None:
            os.environ["QB200_LANES"] = old


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=64)
    ap.add_argument("--window", type=int, default=56)
    ap.add_argument("--slots", type=int, default=64)
    ap.add_argument("--batch", type=int, default=256, help="pairs (sets) per enqueued batch of the stream schedules")
    ap.add_argument("--sets", type=int, default=1024)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()

    import ctypes as C

    import torch
    from bench import gen_pairs, scene_params
    from quatro_b200 import synth
    from quatro_b200.capi import MEM_DEVICE, RESULT_DTYPE, CorrSet, Pair

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    p = scene_params("street")
    p.rot_noise_bound = 2 * p.noise_bound
    scans = [c for pr in gen_pairs(range((args.scans + 1) // 2)) for c in pr][:args.scans]
    flat = torch.from_numpy(np.concatenate(scans).astype(np.float32)).to(dev)
    ptr, o = [], 0
    for s in scans:
        ptr.append(flat.data_ptr() + 16 * o)
        o += len(s)
    pairs = [(i, j) for j in range(args.scans) for i in range(max(0, j - args.window), j)]
    P = len(pairs)
    h1 = handle(1, max_batch_slots=args.slots)
    hd = handle(None, max_batch_slots=args.slots)
    for h in (h1, hd):
        h.cache_reserve(args.scans)
        h.cache_scans([(ptr[i], len(s)) for i, s in enumerate(scans)], list(range(args.scans)), p, MEM_DEVICE)
    slot_arr = np.ascontiguousarray(np.asarray(pairs, np.int32))
    raw = (Pair * P)()
    for k, (i, j) in enumerate(pairs):
        raw[k].src, raw[k].n_src, raw[k].tgt, raw[k].n_tgt = ptr[i], len(scans[i]), ptr[j], len(scans[j])
    cuts = list(range(0, P, args.batch)) + [P]
    pb = C.byref(p)
    par = hd.params_array([p] * args.batch)   # copied by every enqueue: one array serves every batch
    out = {k: np.zeros(P, RESULT_DTYPE) for k in ("cached_lanes1", "cached_lanes", "cached_stream", "uncached")}

    def cached(h, name):
        return lambda: h._check(h.lib.qb200_register_cached(h.h, slot_arr.ctypes.data, P, pb, out[name].ctypes.data), name)

    def cached_stream():
        for a, b in zip(cuts[:-1], cuts[1:]):
            hd.register_cached_enqueue_mixed_raw(slot_arr[a:b], b - a, par, out["cached_stream"][a:b])
        hd.register_batch_flush()

    sweep, _ = timed({"cached_lanes1": cached(h1, "cached_lanes1"), "cached_lanes": cached(hd, "cached_lanes"), "cached_stream": cached_stream,
                      "uncached": lambda: hd.register_batch_raw(raw, P, p, MEM_DEVICE, out["uncached"])}, args.warmup, args.rounds)
    same_sweep = {k: out[k].tobytes() == out["cached_lanes1"].tobytes() for k in out}

    # correspondence sets
    S = args.sets
    sizes = [(300, 800, 1500, 2500)[i % 4] for i in range(S)]
    mats = [synth.matched_pairs(5000 + i, L, inlier_ratio=(0.1, 0.2, 0.3)[i % 3], noise=0.03)[:2] for i, L in enumerate(sizes)]
    dsets = [(torch.from_numpy(a).to(dev), torch.from_numpy(b).to(dev)) for a, b in mats]
    torch.cuda.synchronize(dev)
    sets = (CorrSet * S)()
    for k, (a, b) in enumerate(dsets):
        sets[k].a, sets[k].b, sets[k].L = a.data_ptr(), b.data_ptr(), sizes[k]
    scuts = list(range(0, S, args.batch)) + [S]
    sout = {k: np.zeros(S, RESULT_DTYPE) for k in ("solve_lanes1", "solve_lanes", "solve_stream")}

    def solve(h, name):
        return lambda: h._check(h.lib.qb200_solve_batch(h.h, sets, S, pb, MEM_DEVICE, sout[name].ctypes.data), name)

    def solve_stream():
        for a, b in zip(scuts[:-1], scuts[1:]):
            hd.solve_batch_enqueue_each_raw(C.addressof(sets) + a * C.sizeof(CorrSet), b - a, par, MEM_DEVICE, sout["solve_stream"][a:b])
        hd.register_batch_flush()

    solve_ms, _ = timed({"solve_lanes1": solve(h1, "solve_lanes1"), "solve_lanes": solve(hd, "solve_lanes"), "solve_stream": solve_stream},
                        args.warmup, args.rounds)
    same_sets = {k: sout[k].tobytes() == sout["solve_lanes1"].tobytes() for k in sout}

    print(json.dumps({
        "card": card(), "lanes": {"lanes1": 1, "default": 4}, "slots": args.slots, "batch": args.batch,
        "rounds": args.rounds,
        "sweep": {"scans": args.scans, "window": args.window, "pairs": P, "registered": int((out["cached_lanes"]["status"] == 0).sum()),
                  "n_corr_mean": float(out["cached_lanes"]["n_corr"].mean()), "ms": sweep,
                  "pairs_per_s": {k: P / (v["median"] / 1e3) for k, v in sweep.items()},
                  "lanes_speedup_over_lanes1": sweep["cached_lanes1"]["median"] / sweep["cached_lanes"]["median"],
                  "stream_speedup_over_lanes1": sweep["cached_lanes1"]["median"] / sweep["cached_stream"]["median"],
                  "records_equal": same_sweep},
        "sets": {"sets": S, "ms": solve_ms, "sets_per_s": {k: S / (v["median"] / 1e3) for k, v in solve_ms.items()},
                 "lanes_speedup_over_lanes1": solve_ms["solve_lanes1"]["median"] / solve_ms["solve_lanes"]["median"],
                 "stream_speedup_over_lanes1": solve_ms["solve_lanes1"]["median"] / solve_ms["solve_stream"]["median"],
                 "records_equal": same_sets},
    }))
    for h in (h1, hd):
        h.close()
    if not (all(same_sweep.values()) and all(same_sets.values())):
        sys.exit("records differ between schedules")


if __name__ == "__main__":
    main()
