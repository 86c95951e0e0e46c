"""What queuing scan-cache writes in the batch stream buys a SLAM back end, and what the lane rotation buys a bulk fill of the cache.

Keyframe loop: bench.py's street scans (synth.outdoor_pair, seeds 0..31: 64 scans of 32 scenes, two poses each, device-resident) arrive
as keyframes.  Keyframe k is cached into slot k % --ring, then registered with bench.py's street preset against the --window keyframes
before it.  The ring is smaller than the sequence, so slots are overwritten while batches that read them are still queued.  Two
schedules of the same calls:
  keyframe_blocking  qb200_cache_scans_each + qb200_register_cached_mixed per keyframe;
  keyframe_stream    qb200_cache_scans_enqueue_each + qb200_register_cached_enqueue_mixed per keyframe, one flush at the end.
Bulk fill: --bulk scans (the 64 scans, repeated) into as many slots through one blocking qb200_cache_scans, on a handle created with
  QB200_LANES=1 (bulk_lanes1) and on one with the default lanes (bulk_lanes).
Every schedule is warmed up first and the rounds alternate them; each is timed with the host clock around calls that end with every
lane synchronised.  The records, lists and cache_read contents of the schedules are compared byte for byte.  Prints one JSON line with
the card and its power limit, ms per schedule (median, min, max) and a digest of the bulk-filled slots.

--bulk-only --tree DIR times only the bulk fill, with the quatro_b200 package of the checkout DIR (its library built): the same
measurement of an older tree, whose digest must equal this one's.

  python tools/keyframe_stream_bench.py [--rounds 5] [--warmup 1]
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import sys
from pathlib import Path

import numpy as np

from harness import card, timed

ROOT = Path(__file__).resolve().parent.parent


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


def cache_digest(h, n):
    """sha256 of every slot's cache_read (voxels, normals, descriptors, count), slots 0 .. n-1"""
    d = hashlib.sha256()
    for s in range(n):
        for a in h.cache_read(s):
            d.update(np.ascontiguousarray(a).tobytes())
        d.update(np.int64(len(a)).tobytes())
    return d.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=64)
    ap.add_argument("--ring", type=int, default=24, help="cache slots of the keyframe loop (fewer than --scans)")
    ap.add_argument("--window", type=int, default=16, help="earlier keyframes each keyframe is registered against")
    ap.add_argument("--bulk", type=int, default=512)
    ap.add_argument("--slots", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--bulk-only", action="store_true")
    ap.add_argument("--tree", type=Path, default=ROOT, help="checkout whose quatro_b200 package is timed")
    args = ap.parse_args()
    assert args.ring < args.scans and args.window < args.ring
    sys.path.insert(0, str(args.tree.resolve()))
    sys.path.insert(1, str(ROOT))            # bench.py's scan generator and preset

    import ctypes as C

    import torch
    from bench import gen_pairs, scene_params
    from quatro_b200 import capi
    from quatro_b200.capi import MEM_DEVICE, RESULT_DTYPE, ListBuffers
    assert Path(capi.__file__).resolve().is_relative_to(args.tree.resolve()), capi.__file__

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
    torch.cuda.synchronize(dev)
    K = args.scans
    h1 = handle(1, max_batch_slots=args.slots)
    hd = handle(None, max_batch_slots=args.slots)

    # ---- bulk fill ----
    B = args.bulk
    bulk_ptrs = (C.c_void_p * B)(*[ptr[i % K] for i in range(B)])
    bulk_n = (C.c_int32 * B)(*[len(scans[i % K]) for i in range(B)])
    bulk_ids = (C.c_int32 * B)(*range(B))
    pb = C.byref(p)

    def bulk(h, name):
        return lambda: h._check(h.lib.qb200_cache_scans(h.h, bulk_ptrs, bulk_n, bulk_ids, B, pb, MEM_DEVICE), name)

    for h in (h1, hd):
        h.cache_reserve(B)
    bulk_ms, _ = timed({"bulk_lanes1": bulk(h1, "bulk_lanes1"), "bulk_lanes": bulk(hd, "bulk_lanes")}, args.warmup, args.rounds)
    digests = {"bulk_lanes1": cache_digest(h1, B), "bulk_lanes": cache_digest(hd, B)}
    out = {"card": card(), "tree": "this" if args.tree.resolve() == ROOT else str(args.tree), "slots": args.slots, "rounds": args.rounds,
           "bulk": {"scans": B, "ms": bulk_ms, "scans_per_s": {k: B / (v["median"] / 1e3) for k, v in bulk_ms.items()},
                    "lanes_speedup_over_lanes1": bulk_ms["bulk_lanes1"]["median"] / bulk_ms["bulk_lanes"]["median"],
                    "digest": digests["bulk_lanes"], "digests_equal": digests["bulk_lanes1"] == digests["bulk_lanes"]}}
    ok = out["bulk"]["digests_equal"]

    if not args.bulk_only:
        # ---- keyframe loop, on the default handle ----
        R, Wn = args.ring, args.window
        batches = [np.ascontiguousarray(np.asarray([((k - d) % R, k % R) for d in range(1, min(Wn, k) + 1)], np.int32).reshape(-1, 2))
                   for k in range(K)]
        P = sum(len(b) for b in batches)
        par = hd.params_array([p] * Wn)                # copied by every call: one array serves every keyframe
        one = hd.params_array([p])
        kf_ptrs = [(C.c_void_p * 1)(ptr[k]) for k in range(K)]
        kf_n = [(C.c_int32 * 1)(len(scans[k])) for k in range(K)]
        kf_ids = [(C.c_int32 * 1)(k % R) for k in range(K)]
        recs = {k: [np.zeros(len(b), RESULT_DTYPE) for b in batches] for k in ("keyframe_blocking", "keyframe_stream")}
        lists = {k: [ListBuffers(max(len(b), 1), hd.cfg.max_corr, capi.MEM_HOST) for b in batches] for k in recs}
        lib, hh = hd.lib, hd.h

        def keyframes(name, stream):
            cache = lib.qb200_cache_scans_enqueue_each if stream else lib.qb200_cache_scans_each
            reg = lib.qb200_register_cached_enqueue_mixed if stream else lib.qb200_register_cached_mixed

            def run():
                for k in range(K):
                    hd._check(cache(hh, kf_ptrs[k], kf_n[k], kf_ids[k], 1, one, MEM_DEVICE), name)
                    if len(batches[k]):
                        hd._check(reg(hh, batches[k].ctypes.data, len(batches[k]), par, recs[name][k].ctypes.data,
                                      C.byref(lists[name][k].descriptor())), name)
                if stream:
                    hd.register_batch_flush()
            return run

        hd.cache_reserve(R)
        kf_ms, _ = timed({"keyframe_blocking": keyframes("keyframe_blocking", False), "keyframe_stream": keyframes("keyframe_stream", True)},
                         args.warmup, args.rounds)
        ring_digest = cache_digest(hd, R)

        def flat_out(name):
            return [r.tobytes() for r in recs[name]], [[{k: v.tobytes() for k, v in d.items()} for d in lb.trimmed(r)]
                                                       for r, lb in zip(recs[name], lists[name])]

        same = flat_out("keyframe_blocking") == flat_out("keyframe_stream")
        # the blocking loop once more on its own: the ring it leaves equals the one the alternating rounds left (the stream ran last)
        keyframes("keyframe_blocking", False)()
        same_ring = cache_digest(hd, R) == ring_digest
        allrec = np.concatenate(recs["keyframe_stream"])
        out["keyframe"] = {"keyframes": K, "ring": R, "window": Wn, "pairs": P, "registered": int((allrec["status"] == 0).sum()),
                           "ms": kf_ms, "pairs_per_s": {k: P / (v["median"] / 1e3) for k, v in kf_ms.items()},
                           "stream_speedup_over_blocking": kf_ms["keyframe_blocking"]["median"] / kf_ms["keyframe_stream"]["median"],
                           "records_and_lists_equal": same, "ring_contents_equal": same_ring}
        ok = ok and same and same_ring
    print(json.dumps(out))
    for h in (h1, hd):
        h.close()
    if not ok:
        sys.exit("schedules differ")


if __name__ == "__main__":
    main()
