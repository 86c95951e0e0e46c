"""Golden digests of scan-cache slots (tests/golden/cache_slots.json): 12 street scans (synth.outdoor_pair, seeds 700..705, both
poses) cached by one qb200_cache_scans_each call with three front-end configurations, on a handle of max_batch_slots = 2, so the call
spans three waves of four scans.  Slot 5 is named by the first and the last scan, in different waves.  The file records the inputs and
the sha256 of every slot's qb200_cache_read (voxel points, normals, descriptors, then the count as int64), so
tests/test_cache_stream.py can check any cache path against slots computed by an earlier tree.

  python tools/gen_golden_cache.py [--tree DIR] [--out tests/golden/cache_slots.json]
"""
from __future__ import annotations

import argparse
import hashlib
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent

SEEDS = list(range(700, 706))
SLOTS = [5, 0, 1, 2, 3, 4, 6, 7, 8, 9, 10, 5]
# front-end fields of the three configurations (the rest: qb200_default_params)
FRONTS = [{}, {"voxel_size": 0.4, "grid_cell": 0.4, "seed": 14}, {"voxel_size": 0.25, "grid_cell": 0.4, "seed": 13}]
CONFIG = {"max_batch_slots": 2, "max_raw_points": 32768}


def scans():
    from quatro_b200 import synth
    return [c for s in SEEDS for c in synth.outdoor_pair(s, rings=32, azimuths=900)[:2]]


def entries():
    from quatro_b200.capi import default_params
    out = []
    for i in range(len(SLOTS)):
        p = default_params()
        for k, v in FRONTS[i % 3].items():
            setattr(p, k, v)
        out.append(p)
    return out


def slot_digest(h, slot):
    v, n, d = h.cache_read(slot)
    return hashlib.sha256(v.tobytes() + n.tobytes() + d.tobytes() + np.int64(len(v)).tobytes()).hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", type=Path, default=ROOT, help="checkout whose quatro_b200 package computes the slots")
    ap.add_argument("--out", type=Path, default=ROOT / "tests" / "golden" / "cache_slots.json")
    args = ap.parse_args()
    sys.path.insert(0, str(args.tree.resolve()))
    from quatro_b200.capi import Handle
    with Handle(**CONFIG) as h:
        h.cache_reserve(max(SLOTS) + 1)
        h.cache_scans_each(scans(), SLOTS, entries())
        digests = [slot_digest(h, s) for s in range(max(SLOTS) + 1)]
    args.out.write_text(json.dumps({"config": CONFIG, "seeds": SEEDS, "slots": SLOTS, "fronts": FRONTS, "digests": digests}, indent=1) + "\n")
    print(args.out, len(digests), "slots")


if __name__ == "__main__":
    main()
