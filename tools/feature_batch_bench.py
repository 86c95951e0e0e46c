"""What registering caller keypoints and FPFH-33 descriptors in batches buys over today's per-pair loop.

256 street pairs (synth.outdoor_pair, seeds 0..255, default front end) are cached once on a default handle; every scan's voxel points
and descriptors are read back with qb200_cache_read and serve as the caller's features.  Four schedules register the same pairs
with the default params:
  features_device  one qb200_register_features_each call, features in device memory;
  features_host    the same call, features in (pageable) host memory: 148 B per keypoint cross PCIe;
  cached           one qb200_register_cached_mixed call on the slots the features came from;
  match_loop       the loop a caller writes without the batch form: qb200_match per pair (one matcher launch and one host sync
                   each), the matched points gathered on the host, then one qb200_solve_batch.
Every schedule is warmed up first and the rounds alternate them; each is timed with the host clock around calls that end with every
lane synchronised.  The records of the four are compared: the three batch forms byte for byte, the loop on every counter except
n_src_vox / n_tgt_vox / n_mutual (qb200_solve_batch has no front end) and on the pose.  A separate torch.profiler run of
features_device times feature_import_kernel; its bytes are 2 x 148 B per keypoint (a 16-byte keypoint and a 132-byte descriptor
row read, the same written).  Prints one JSON line with the card and its power limit.

  python tools/feature_batch_bench.py [--pairs 256] [--rounds 5] [--warmup 2]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()

    import torch
    from quatro_b200 import synth
    from quatro_b200.capi import MEM_DEVICE, MEM_HOST, Handle, default_params

    n = a.pairs
    p = default_params()
    p.rot_noise_bound = 2 * p.noise_bound
    params = [p] * n
    h = Handle()
    scans = [s for i in range(n) for s in synth.outdoor_pair(i)[:2]]
    h.cache_reserve(2 * n)
    h.cache_scans(scans, list(range(2 * n)), p)
    del scans
    slot_pairs = [(2 * i, 2 * i + 1) for i in range(n)]
    feats = []
    for i in range(n):
        (sv, _, sd), (tv, _, td) = h.cache_read(2 * i), h.cache_read(2 * i + 1)
        feats.append((sv, sd, tv, td))
    dev_keep = [[torch.from_numpy(x).cuda() for x in f] for f in feats]
    torch.cuda.synchronize()
    dev = [(d[0].data_ptr(), d[1].data_ptr(), len(f[0]), d[2].data_ptr(), d[3].data_ptr(), len(f[2])) for d, f in zip(dev_keep, feats)]
    keypoints = sum(len(f[0]) + len(f[2]) for f in feats)

    out = {}

    def match_loop():
        sets = []
        for s, sd, t, td in feats:
            corr, _, _ = h.match(s, sd, t, td, p, cap=h.cfg.max_corr)
            sets.append((s[corr[:, 0]], t[corr[:, 1]]))
        return h.solve_batch(sets, p)

    ways = {
        "features_device": lambda: out.__setitem__("features_device", h.register_features_each(dev, params, MEM_DEVICE)[0]),
        "features_host": lambda: out.__setitem__("features_host", h.register_features_each(feats, params, MEM_HOST)[0]),
        "cached": lambda: out.__setitem__("cached", h.register_cached_mixed(slot_pairs, params)[0]),
        "match_loop": lambda: out.__setitem__("match_loop", match_loop()),
    }
    ms, _ = timed(ways, a.warmup, a.rounds)

    same = {k: out[k].tobytes() == out["cached"].tobytes() for k in ("features_device", "features_host")}
    skip = {"n_src_vox", "n_tgt_vox", "n_mutual"}
    loop, ref = out["match_loop"], out["cached"]
    same["match_loop"] = all(np.array_equal(loop[f], ref[f]) for f in ref.dtype.names if f not in skip | {"T", "cost"}) and \
        bool(np.allclose(loop["T"], ref["T"], atol=1e-9, rtol=0))

    # the import kernel on its own, from a profiled run of the device-kind call
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        h.register_features_each(dev, params, MEM_DEVICE)
        torch.cuda.synchronize()
    imp = [e for e in prof.events() if "feature_import_kernel" in e.name]
    import_us = sum(e.device_time for e in imp) if hasattr(imp[0], "device_time") else sum(e.cuda_time for e in imp)
    import_bytes = 2 * 148 * keypoints

    rate = {k: 1e3 * n / v["median"] for k, v in ms.items()}
    print(json.dumps({
        "card": card(), "pairs": n, "keypoints": keypoints, "ms": ms, "pairs_per_s": rate,
        "speedup_vs_match_loop": {k: rate[k] / rate["match_loop"] for k in ("features_device", "features_host", "cached")},
        "records_equal_cached": same,
        "import_kernel": {"launches": len(imp), "us": import_us, "bytes": import_bytes, "GB_per_s": import_bytes / (import_us * 1e3)},
    }))
    h.close()
    if not all(same.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
