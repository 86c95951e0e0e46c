"""What matching caller descriptors of any length in batches costs, and what it buys over the per-pair loop of the same call.

256 street pairs (synth.outdoor_pair, seeds 0..255, default front end) are cached once on a default handle, and every scan's voxel
points and FPFH-33 rows are read back with qb200_cache_read.  Descriptors of other lengths are those rows times a fixed random
33 x dim matrix (seed 0), so they keep FPFH's neighbourhoods; 352 floats sit in rows of 361, as pcl::SHOT352 stores them.  For each
length the schedules are:
  dim<d>_device / dim<d>_host   one qb200_match_descriptors_each call, descriptors in device / pageable host memory;
  dim<d>_loop                   the per-pair loop of the same call (n = 1 per call, device memory);
  dim33_features                qb200_match_features_each on the same 33-float rows (the dim-33 comparison of the two calls).
Every schedule is warmed up first, the rounds alternate them, and each is timed with the host clock around calls that end with every
lane synchronised.  The batch and loop records are compared byte for byte, and at 33 floats also with the _features_ call.  A
separate torch.profiler run of each device-kind call times nn_dim_kernel against its FP32-FMA bound, 2 * n_src * n_tgt * dim FLOP
per pair.  Prints one JSON line with the card and its power limit.

  python tools/descriptor_batch_bench.py [--pairs 256] [--rounds 3] [--warmup 1] [--dims 32,33,125,352]
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
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--dims", default="32,33,125,352")
    a = ap.parse_args()

    import torch
    from quatro_b200 import synth
    from quatro_b200.capi import MATCH_LISTS, MEM_DEVICE, MEM_HOST, Handle, ListBuffers, default_params

    n = a.pairs
    p = default_params()
    params = [p] * n
    h = Handle()
    scans = [s for i in range(n) for s in synth.outdoor_pair(i)[:2]]
    h.cache_reserve(2 * n)
    h.cache_scans(scans, list(range(2 * n)), p)
    del scans
    feats = []
    for i in range(n):
        (sv, _, sd), (tv, _, td) = h.cache_read(2 * i), h.cache_read(2 * i + 1)
        feats.append((sv, sd, tv, td))
    pair_points = [(len(f[0]), len(f[2])) for f in feats]
    rng = np.random.default_rng(0)

    def rows(d33, dim):
        if dim == 33:
            return d33
        stride = 361 if dim == 352 else dim
        out = np.zeros((len(d33), stride), np.float32)
        out[:, :dim] = d33 @ rng_mats[dim]
        return out

    out, ways, dev_keep, batches = {}, {}, [], {}
    rng_mats = {}
    for dim in map(int, a.dims.split(",")):
        if dim != 33:
            rng_mats[dim] = rng.standard_normal((33, dim)).astype(np.float32)
        host = [(s, rows(sd, dim), t, rows(td, dim), dim) for s, sd, t, td in feats]
        keep = [[torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in pr[:4]] for pr in host]
        dev_keep.append(keep)
        dev = [(k[0].data_ptr(), k[1].data_ptr(), len(pr[0]), k[2].data_ptr(), k[3].data_ptr(), len(pr[2]), dim, pr[1].shape[1])
               for k, pr in zip(keep, host)]
        batches[dim] = dev

        def call(prs, kind, key):
            lb = ListBuffers(len(prs), h.cfg.max_corr, MEM_DEVICE, MATCH_LISTS)
            out[key] = h.match_descriptors_each(prs, params[:len(prs)], kind, buffers=lb)[0]

        def loop(prs, key):
            out[key] = np.concatenate([h.match_descriptors_each([pr], [p], MEM_DEVICE)[0] for pr in prs])

        ways[f"dim{dim}_device"] = lambda dev=dev, dim=dim: call(dev, MEM_DEVICE, f"dim{dim}_device")
        ways[f"dim{dim}_host"] = lambda host=host, dim=dim: call(host, MEM_HOST, f"dim{dim}_host")
        ways[f"dim{dim}_loop"] = lambda dev=dev, dim=dim: loop(dev, f"dim{dim}_loop")
        if dim == 33:
            fdev = [d[:6] for d in dev]
            ways["dim33_features"] = lambda fdev=fdev: out.__setitem__(
                "dim33_features", h.match_features_each(fdev, params, MEM_DEVICE, buffers=ListBuffers(n, h.cfg.max_corr, MEM_DEVICE,
                                                                                                         MATCH_LISTS))[0])
    torch.cuda.synchronize()
    ms, _ = timed(ways, a.warmup, a.rounds)

    same = {}
    for dim in batches:
        ref = out[f"dim{dim}_device"].tobytes()
        same[dim] = out[f"dim{dim}_host"].tobytes() == ref and out[f"dim{dim}_loop"].tobytes() == ref
        if dim == 33:
            same["33_features"] = out["dim33_features"].tobytes() == ref

    # nn_dim_kernel on its own, from a profiled run of each device-kind call
    from torch.profiler import ProfilerActivity, profile
    kern = {}
    for dim, dev in batches.items():
        if dim == 33:
            continue
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            h.match_descriptors_each(dev, params, MEM_DEVICE)
            torch.cuda.synchronize()
        ev = [e for e in prof.events() if "nn_dim_kernel" in e.name and "colreset" not in e.name]
        us = sum(getattr(e, "device_time", None) or e.cuda_time for e in ev)
        flop = sum(2.0 * ns * nt * dim for ns, nt in pair_points)
        kern[dim] = {"launches": len(ev), "us": us, "flop": flop, "TFLOP_per_s": flop / (us * 1e6) if us else None,
                     "fp32_fma_bound_us_at_67_TFLOPs": flop / 67e12 * 1e6}

    rate = {k: 1e3 * n / v["median"] for k, v in ms.items()}
    print(json.dumps({
        "card": card(), "pairs": n, "keypoints": sum(a_ + b for a_, b in pair_points), "ms": ms, "pairs_per_s": rate,
        "speedup_vs_loop": {k: rate[k] / rate[k.rsplit("_", 1)[0] + "_loop"] for k in rate if k.endswith(("_device", "_host"))},
        "records_equal": same, "nn_dim_kernel": kern,
    }))
    h.close()
    if not all(same.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
