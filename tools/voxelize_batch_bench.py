"""What voxelizing scans in batches buys over the ways a caller gets voxel centroids without the batch form.

512 street scans from a 64-ring lidar (synth.outdoor_pair, seeds 0..255, both scans of each pair) are voxelized at the default
entry (0.3 m leaf, skip_flagged 1), and every scan's centroids end in caller memory.  Six schedules:
  voxelize_hh   one qb200_voxelize_batch_each call, scans in (pageable) host memory, outputs to host arrays;
  voxelize_hd   host scans, outputs to device arrays;
  voxelize_dh   scans in device memory, outputs to host arrays;
  voxelize_dd   device scans, device outputs;
  describe_dd   qb200_describe_batch_each with vox4 alone, device scans and outputs: the batch route before this call, which
                still computes normals and FPFH-33 of every scan;
  stage_loop    the per-scan loop: qb200_voxelize, one host sync per scan.
Each batch schedule writes into its own output arrays (cap_per_scan = max_voxel_points), allocated and, on the host, touched once; its
timed window is the C call alone.  Every schedule runs twice as warm-up, then the rounds alternate them (the median of 5); each is
timed with the host clock around calls that return with their outputs complete (device outputs: after a torch.cuda.synchronize).  The
outputs of all six are compared byte for byte, scan by scan.  Prints one JSON line with the card and its power limit.

  python tools/voxelize_batch_bench.py [--scans 512] [--rounds 5] [--warmup 2]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import sys
from pathlib import Path

import numpy as np

from harness import card, timed

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=512)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()

    import torch
    from quatro_b200 import synth
    from quatro_b200.capi import MEM_DEVICE, MEM_HOST, Handle, _scan_arrays, default_params

    p = default_params()
    n = a.scans
    scans = [s for i in range((n + 1) // 2) for s in synth.outdoor_pair(i)[:2]][:n]
    dev_keep = [torch.from_numpy(s).cuda() for s in scans]
    torch.cuda.synchronize()
    dev = [(t.data_ptr(), len(t)) for t in dev_keep]
    h = Handle()
    cap = h.cfg.max_voxel_points
    out = {}
    pa = h.params_array([p] * n)
    ptrs = {MEM_HOST: _scan_arrays(scans, MEM_HOST), MEM_DEVICE: _scan_arrays(dev, MEM_DEVICE)}
    bufs = {}

    def batch(name, fn, kind, dest):
        # the schedule's own output array, allocated and touched once
        bufs[name] = h.feature_buffers(n, cap, dest, ("vox4",))
        if dest == MEM_HOST:
            bufs[name]["vox4"].fill(0.0)
        counts, status = np.zeros(n, np.int32), np.zeros(n, np.int32)
        fo = h.feature_out(cap, dest, bufs[name], counts, status)
        call = getattr(h.lib, fn)

        def run():
            sp, sc, _ = ptrs[kind]
            assert call(h.h, sp, sc, n, pa, kind, C.byref(fo)) == 0
            if dest == MEM_DEVICE:
                torch.cuda.synchronize()
            out[name] = (dest, counts, status)
        return run

    def stage_loop():
        out["stage_loop"] = [h.voxelize(s, p.voxel_size, p.skip_flagged, cap=cap) for s in scans]

    ways = {
        "voxelize_hh": batch("voxelize_hh", "qb200_voxelize_batch_each", MEM_HOST, MEM_HOST),
        "voxelize_hd": batch("voxelize_hd", "qb200_voxelize_batch_each", MEM_HOST, MEM_DEVICE),
        "voxelize_dh": batch("voxelize_dh", "qb200_voxelize_batch_each", MEM_DEVICE, MEM_HOST),
        "voxelize_dd": batch("voxelize_dd", "qb200_voxelize_batch_each", MEM_DEVICE, MEM_DEVICE),
        "describe_dd": batch("describe_dd", "qb200_describe_batch_each", MEM_DEVICE, MEM_DEVICE),
        "stage_loop": stage_loop,
    }
    ms, _ = timed(ways, a.warmup, a.rounds)

    # every schedule's bytes, scan by scan, against the per-scan loop
    want = [v.tobytes() for v, _ in out["stage_loop"]]
    want_st = [st for _, st in out["stage_loop"]]
    same = {}
    for k in ways:
        if k == "stage_loop":
            continue
        dest, c, st = out[k]
        v = bufs[k]["vox4"] if dest == MEM_HOST else bufs[k]["vox4"].cpu().numpy()
        got = [v[i, :min(c[i], cap)].tobytes() for i in range(n)]
        same[k] = got == want and list(st) == want_st
        del v
    counts = out["voxelize_hh"][1]
    rate = {k: 1e3 * n / v["median"] for k, v in ms.items()}
    print(json.dumps({
        "card": card(), "scans": n, "raw_points": int(sum(len(s) for s in scans)), "centroids": int(counts.sum()), "cap_per_scan": cap,
        "ms": ms, "scans_per_s": rate, "speedup_vs_stage_loop": {k: rate[k] / rate["stage_loop"] for k in ways if k != "stage_loop"},
        "bytes_equal_stage_loop": same,
    }))
    h.close()
    if not all(same.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
