"""What matching pairs in batches without the solve buys: the match calls against the register calls on the same pairs (the solver
tail they skip) and against the per-pair qb200_match loop they replace.

256 street pairs (synth.outdoor_pair, seeds 0..255, default front end) are cached once on a default handle; every scan's voxel points
and descriptors are read back with qb200_cache_read and copied to the device as the caller's features, and the raw scans are copied
to the device as well.  With the default params (rotation noise bound explicit), each input is timed three ways:
  match_*     qb200_match_features_each (device features), qb200_match_cached_mixed (the slots), qb200_match_batch_mixed (device
              scans), correspondences and matched points into device lists;
  register_*  the register call of the same input (qb200_register_features_each, _cached_mixed, _batch_mixed) with the same lists;
  match_loop  qb200_match per pair on host features (one matcher launch and one host sync each), the loop a caller writes without
              the batch form.
Every way is warmed up first and the rounds alternate them; each call is timed with the host clock and ends with every lane
synchronised.  After every timed run (outside the timed region) its records' matcher fields and its lists are compared byte for byte
with the register call of its input; the loop's correspondence lists with the feature register call's.  Prints one JSON line with the
card and its power limit, and exits 1 if any output differs.

  python tools/match_batch_bench.py [--pairs 256] [--rounds 5] [--warmup 2]
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

MATCHER = ("n_src_vox", "n_tgt_vox", "n_mutual", "n_corr")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()

    import torch
    from quatro_b200 import synth
    from quatro_b200.capi import MATCH_LISTS, MEM_DEVICE, Handle, ListBuffers, default_params

    n = a.pairs
    p = default_params()
    p.rot_noise_bound = 2 * p.noise_bound
    params = [p] * n
    h = Handle()
    cap = h.cfg.max_corr
    raw = [synth.outdoor_pair(i)[:2] for i in range(n)]
    h.cache_reserve(2 * n)
    h.cache_scans([s for pr in raw for s in pr], list(range(2 * n)), p)
    slot_pairs = [(2 * i, 2 * i + 1) for i in range(n)]
    feats = []
    for i in range(n):
        (sv, _, sd), (tv, _, td) = h.cache_read(2 * i), h.cache_read(2 * i + 1)
        feats.append((sv, sd, tv, td))
    feat_keep = [[torch.from_numpy(x).cuda() for x in f] for f in feats]
    raw_keep = [[torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in pr] for pr in raw]
    torch.cuda.synchronize()
    feat_dev = [(d[0].data_ptr(), d[1].data_ptr(), len(f[0]), d[2].data_ptr(), d[3].data_ptr(), len(f[2])) for d, f in zip(feat_keep, feats)]
    raw_dev = [(d[0].data_ptr(), len(pr[0]), d[1].data_ptr(), len(pr[1])) for d, pr in zip(raw_keep, raw)]
    calls = {
        "features": (lambda lb: h.match_features_each(feat_dev, params, MEM_DEVICE, buffers=lb),
                     lambda lb: h.register_features_each(feat_dev, params, MEM_DEVICE, buffers=lb)),
        "cached": (lambda lb: h.match_cached_mixed(slot_pairs, params, buffers=lb),
                   lambda lb: h.register_cached_mixed(slot_pairs, params, buffers=lb)),
        "raw": (lambda lb: h.match_batch_mixed(raw_dev, params, MEM_DEVICE, buffers=lb),
                lambda lb: h.register_batch_mixed(raw_dev, params, MEM_DEVICE, buffers=lb)),
    }

    def flat(recs, lb):
        """the records' matcher fields and the live lists, as bytes"""
        lists = lb.trimmed(recs)
        return np.stack([recs[k] for k in MATCHER], 1).tobytes(), [b"".join(d[k].cpu().numpy().tobytes() for k in MATCH_LISTS) for d in lists]

    # the reference outputs: one register call of every input
    want, lbs, out = {}, {}, {}
    for src, (_, register) in calls.items():
        lb = ListBuffers(n, cap, MEM_DEVICE, MATCH_LISTS, device=h.cfg.device)
        want[src] = flat(register(lb)[0], lb)
        lbs["match_" + src] = ListBuffers(n, cap, MEM_DEVICE, MATCH_LISTS, device=h.cfg.device)
        lbs["register_" + src] = ListBuffers(n, cap, MEM_DEVICE, MATCH_LISTS, device=h.cfg.device)
    n_corr = np.frombuffer(want["features"][0], np.int32).reshape(n, len(MATCHER))[:, MATCHER.index("n_corr")]
    want_corr = [b[: 8 * int(c)] for b, c in zip(want["features"][1], n_corr)]   # corr leads each pair's bytes

    def match_loop():
        out["match_loop"] = [h.match(s, sd, t, td, p, cap=cap)[0] for s, sd, t, td in feats]

    ways, checks = {}, {}
    for src, (match, register) in calls.items():
        for kind, fn in (("match", match), ("register", register)):
            name = f"{kind}_{src}"
            ways[name] = lambda fn=fn, name=name: out.__setitem__(name, fn(lbs[name])[0])
            checks[name] = lambda src=src, name=name: flat(out[name], lbs[name]) == want[src]
    ways["match_loop"] = match_loop
    checks["match_loop"] = lambda: [np.ascontiguousarray(c).tobytes() for c in out["match_loop"]] == want_corr
    ms, same = timed(ways, a.warmup, a.rounds, checks)

    rec = out["match_features"]
    rate = {k: 1e3 * n / v["median"] for k, v in ms.items()}
    print(json.dumps({
        "card": card(), "pairs": n, "mean_n_corr": float(rec["n_corr"].mean()), "ms": ms, "pairs_per_s": rate,
        "solver_tail_skipped_ms": {src: ms[f"register_{src}"]["median"] - ms[f"match_{src}"]["median"] for src in calls},
        "speedup_vs_match_loop": {f"match_{src}": rate[f"match_{src}"] / rate["match_loop"] for src in calls},
        "outputs_equal_register": same,
    }))
    h.close()
    if not all(same.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
