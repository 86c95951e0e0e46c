"""What describing caller keypoint clouds in batches buys over the per-cloud qb200_compute_fpfh loop.

512 keypoint clouds: the 0.3 m voxel centroids of 512 street scans (synth.outdoor_pair, seeds 0..255, both scans of each pair), made
once by qb200_describe_batch_each.  Every cloud gets normals and FPFH-33 rows (default radii, default lattice cell) in caller memory.
Three schedules:
  points_dd     one qb200_describe_points_each call, clouds resident in device memory (one tensor), outputs to device arrays;
  points_hh     the same call with the clouds in (pageable) host memory and host outputs;
  fpfh_loop     the per-cloud loop: qb200_compute_fpfh on each host cloud (one host sync and two host copies per cloud).
Each describe schedule writes into its own output arrays (cap_per_scan = max_voxel_points), allocated and, on the host, touched once;
its timed window is the C call alone (device outputs: until a torch.cuda.synchronize).  Every schedule is warmed up first and the
rounds alternate them.  The outputs of all three are compared byte for byte, cloud by cloud.  A separate torch.profiler run of
points_dd times feature_import_kernel and the front-end kernels (K2..K5) of the call.  Prints one JSON line with the card and its
power limit, read in the same run.

  python tools/describe_points_bench.py [--clouds 512] [--rounds 3] [--warmup 1]
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
    ap.add_argument("--clouds", type=int, default=512)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()

    import torch
    from quatro_b200 import synth
    from quatro_b200.capi import MEM_DEVICE, MEM_HOST, POINT_ARRAYS, Handle, _scan_arrays, default_params

    p = default_params()
    n = a.clouds
    scans = [s for i in range((n + 1) // 2) for s in synth.outdoor_pair(i)[:2]][:n]
    cell = float(np.float32(p.fpfh_radius) * np.float32(1.001953125))   # the default lattice cell
    h = Handle()
    cap = h.cfg.max_voxel_points
    params = [p] * n
    pa = h.params_array(params)
    per_scan, counts, status = h.describe_batch_each(scans, params, MEM_HOST, MEM_HOST, arrays=h.feature_buffers(n, cap, MEM_HOST, ("vox4",)))
    assert (status == 0).all() and (counts <= cap).all()
    clouds = [row[0] for row in per_scan]
    flat = torch.from_numpy(np.concatenate(clouds)).cuda()             # the device-resident clouds, back to back
    offs = np.concatenate([[0], np.cumsum(counts)])
    dev = [(flat[offs[i]:offs[i + 1]].data_ptr(), int(counts[i])) for i in range(n)]
    torch.cuda.synchronize()
    ptrs = {MEM_HOST: _scan_arrays(clouds, MEM_HOST), MEM_DEVICE: _scan_arrays(dev, MEM_DEVICE)}
    out, bufs = {}, {}

    def describe(name, kind, dest):
        bufs[name] = h.feature_buffers(n, cap, dest, POINT_ARRAYS)
        if dest == MEM_HOST:
            for b in bufs[name].values():
                b.fill(0.0)
        c, st = np.zeros(n, np.int32), np.zeros(n, np.int32)
        fo = h.feature_out(cap, dest, bufs[name], c, st)

        def run():
            cp, cc, _ = ptrs[kind]
            assert h.lib.qb200_describe_points_each(h.h, cp, cc, n, pa, kind, C.byref(fo)) == 0
            if dest == MEM_DEVICE:
                torch.cuda.synchronize()
            out[name] = (dest, c, st)
        return run

    def fpfh_loop():
        out["fpfh_loop"] = [h.compute_fpfh(v, p.normal_radius, p.fpfh_radius, cell) for v in clouds]

    ways = {"points_dd": describe("points_dd", MEM_DEVICE, MEM_DEVICE), "points_hh": describe("points_hh", MEM_HOST, MEM_HOST),
            "fpfh_loop": fpfh_loop}
    ms, _ = timed(ways, a.warmup, a.rounds)

    want = [tuple(x.tobytes() for x in row) for row in out["fpfh_loop"]]
    same = {}
    for k in ("points_dd", "points_hh"):
        dest, c, st = out[k]
        host = {name: (v if dest == MEM_HOST else v.cpu().numpy()) for name, v in bufs[k].items()}
        got = [tuple(host[name][i, :c[i]].tobytes() for name in POINT_ARRAYS) for i in range(n)]
        same[k] = got == want and bool((st == 0).all()) and bool((c == counts).all())
        del host

    # the kernels of the device-to-device call, from a profiled run
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ways["points_dd"]()
    kern = {}
    for e in prof.events():
        if not str(e.device_type).endswith("CUDA"):
            continue
        t = e.device_time if hasattr(e, "device_time") else e.cuda_time
        name = e.name.split("(")[0].split("<")[0].replace("void ", "").replace("qb::", "")
        kern[name] = kern.get(name, 0.0) + t

    rate = {k: 1e3 * n / v["median"] for k, v in ms.items()}
    print(json.dumps({
        "card": card(), "clouds": n, "keypoints": int(counts.sum()), "ms": ms, "clouds_per_s": rate,
        "speedup_vs_fpfh_loop": {k: rate[k] / rate["fpfh_loop"] for k in ways if k != "fpfh_loop"},
        "bytes_equal_fpfh_loop": same, "kernel_us": {k: round(v, 1) for k, v in sorted(kern.items(), key=lambda x: -x[1])[:12]},
    }))
    h.close()
    if not all(same.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
