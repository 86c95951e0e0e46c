"""What describing scans in batches buys over the ways a caller gets front-end features without the batch form.

512 street scans (synth.outdoor_pair, seeds 0..255, both scans of each pair, default front end: 0.3 m voxel) are voxelized and
described, and every scan's voxel keypoints, normals and FPFH-33 rows end in caller memory.  Six schedules:
  describe_hh   one qb200_describe_batch_each call, scans in (pageable) host memory, outputs to host arrays;
  describe_hd   host scans, outputs to device arrays;
  describe_dh   scans in device memory, outputs to host arrays;
  describe_dd   device scans, device outputs;
  stage_loop    the per-scan loop: qb200_voxelize + qb200_compute_fpfh (two host syncs and three host copies per scan);
  cache_read    qb200_cache_scans of the whole batch into 512 slots, then one blocking qb200_cache_read per slot.
Each describe schedule writes into its own output arrays (cap_per_scan = max_voxel_points), allocated and, on the host, touched
once, as a caller that keeps a feature store does; its timed window is the C call alone.  Every schedule is warmed up first and the
rounds alternate them; each is timed with the host clock around calls that return with their outputs complete (device outputs:
after a torch.cuda.synchronize).  The outputs of all six are compared byte for byte, scan by scan.  A separate torch.profiler run of describe_dd times feature_export_kernel; its bytes are 2 x 164 B per keypoint (a 16-byte
centroid, a 16-byte normal and a 132-byte descriptor row, read and written).  Prints one JSON line with the card and its power limit.

  python tools/describe_batch_bench.py [--scans 512] [--rounds 3] [--warmup 1]
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
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()

    import torch
    from quatro_b200 import synth
    from quatro_b200.capi import FEATURE_ARRAYS, MEM_DEVICE, MEM_HOST, Handle, _scan_arrays, default_params

    p = default_params()
    n = a.scans
    scans = [s for i in range((n + 1) // 2) for s in synth.outdoor_pair(i)[:2]][:n]
    dev_keep = [torch.from_numpy(s).cuda() for s in scans]
    torch.cuda.synchronize()
    dev = [(t.data_ptr(), len(t)) for t in dev_keep]
    params = [p] * n
    cell = float(np.float32(p.fpfh_radius) * np.float32(1.001953125))   # the default lattice cell
    h = Handle()
    cap = h.cfg.max_voxel_points
    h.cache_reserve(n)
    out = {}
    pa = h.params_array(params)
    ptrs = {MEM_HOST: _scan_arrays(scans, MEM_HOST), MEM_DEVICE: _scan_arrays(dev, MEM_DEVICE)}
    bufs = {}

    def describe(name, kind, dest):
        # the schedule's own output arrays, allocated and touched once
        bufs[name] = h.feature_buffers(n, cap, dest)
        if dest == MEM_HOST:
            for b in bufs[name].values():
                b.fill(0.0)
        counts, status = np.zeros(n, np.int32), np.zeros(n, np.int32)
        fo = h.feature_out(cap, dest, bufs[name], counts, status)

        def run():
            sp, sc, _ = ptrs[kind]
            assert h.lib.qb200_describe_batch_each(h.h, sp, sc, n, pa, kind, C.byref(fo)) == 0
            if dest == MEM_DEVICE:
                torch.cuda.synchronize()
            out[name] = (dest, counts, status)
        return run

    def stage_loop():
        rows = []
        for s in scans:
            vox, st = h.voxelize(s, p.voxel_size, p.skip_flagged, cap=h.cfg.max_voxel_points)
            nrm, desc = h.compute_fpfh(vox, p.normal_radius, p.fpfh_radius, cell)
            rows.append((vox, nrm, desc))
        out["stage_loop"] = rows

    def cache_read():
        h.cache_scans(scans, list(range(n)), p)
        out["cache_read"] = [h.cache_read(i) for i in range(n)]

    ways = {
        "describe_hh": describe("describe_hh", MEM_HOST, MEM_HOST),
        "describe_hd": describe("describe_hd", MEM_HOST, MEM_DEVICE),
        "describe_dh": describe("describe_dh", MEM_DEVICE, MEM_HOST),
        "describe_dd": describe("describe_dd", MEM_DEVICE, MEM_DEVICE),
        "stage_loop": stage_loop,
        "cache_read": cache_read,
    }
    ms, _ = timed(ways, a.warmup, a.rounds)

    # every schedule's bytes, scan by scan, against the cache
    want = [tuple(x.tobytes() for x in row) for row in out["cache_read"]]
    counts = out["describe_hh"][1]
    same = {"stage_loop": [tuple(x.tobytes() for x in row) for row in out["stage_loop"]] == want}
    for k in ("describe_hh", "describe_hd", "describe_dh", "describe_dd"):
        dest, c, st = out[k]
        host = {name: (v if dest == MEM_HOST else v.cpu().numpy()) for name, v in bufs[k].items()}
        got = [tuple(host[name][i, :min(c[i], cap)].tobytes() for name in FEATURE_ARRAYS) for i in range(n)]
        same[k] = got == want and bool((st == 0).all()) and bool((c == counts).all())
        del host
    clipped = int((counts > cap).sum())
    keypoints = int(counts.sum())

    # the export kernel on its own, from a profiled run of the device-to-device call
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ways["describe_dd"]()
    exp = [e for e in prof.events() if "feature_export_kernel" in e.name]
    export_us = sum(e.device_time for e in exp) if hasattr(exp[0], "device_time") else sum(e.cuda_time for e in exp)
    export_bytes = 2 * 4 * sum(FEATURE_ARRAYS.values()) * keypoints

    rate = {k: 1e3 * n / v["median"] for k, v in ms.items()}
    print(json.dumps({
        "card": card(), "scans": n, "cap_per_scan": cap, "keypoints": keypoints, "clipped_scans": clipped, "ms": ms, "scans_per_s": rate,
        "speedup_vs_stage_loop": {k: rate[k] / rate["stage_loop"] for k in ways if k != "stage_loop"},
        "speedup_vs_cache_read": {k: rate[k] / rate["cache_read"] for k in ways if k.startswith("describe")},
        "bytes_equal_cache_read": same,
        "export_kernel": {"launches": len(exp), "us": export_us, "bytes": export_bytes, "GB_per_s": export_bytes / (export_us * 1e3)},
    }))
    h.close()
    if not all(same.values()) or clipped:
        sys.exit(1)


if __name__ == "__main__":
    main()
