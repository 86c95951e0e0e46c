"""Throughput of qb200_preprocess_batch against a loop of the single-scan calls (qb200_patchwork + qb200_segment_cloud), and of the
whole chain raw scans -> pre-processing -> registration.

    python tools/preprocess_batch_bench.py [--reps 3] [--pairs 256] [--out result.json]

Part 1: the same 8, 64 and 512 generator scans (64 x 1800 rays) through the loop and through the batch with host and with device
outputs (arrays allocated once), the three alternated, `reps` rounds; scans/s is the median round.  Part 2: `pairs` generator pairs, raw, pre-processed by
one batch call with device outputs whose valid segments go straight into qb200_register_batch(kind = DEVICE); registrations/s over
the whole chain, next to the single-call chain (loop, then qb200_register_batch on host clouds).  Outputs of the batch are checked
against the loop's.  The card's name and power limit are read in the same run."""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from harness import card  # noqa: E402
from quatro_b200 import capi, synth  # noqa: E402
from quatro_b200.capi import MEM_DEVICE, MEM_HOST, default_patchwork_params, default_segment_params  # noqa: E402


def loop(h, scans, pp, sp):
    return [h.segment_cloud(h.patchwork(s, pp)[1], sp)[0] for s in scans]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--sizes", default="8,64,512")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    pp, sp = default_patchwork_params(), default_segment_params()
    pairs = [synth.outdoor_pair(9000 + i)[:2] for i in range(max(a.pairs, 256))]
    scans = [s for pr in pairs for s in pr]
    sizes = [int(x) for x in a.sizes.split(",")]
    res = {"card": card("clocks.max.sm"), "scan_points_mean": float(np.mean([len(s) for s in scans])), "throughput": {}}
    h = capi.Handle()
    cap = sp.n_scan * sp.horizon_scan
    # the batch's output arrays are allocated once and reused, as a caller processing scan after scan would (the loop's small per-call
    # arrays come back from the allocator already mapped)
    dev = {k: torch.zeros((max(sizes), cap, 4), dtype=torch.float32, device="cuda") for k in capi.PREPROCESS_ARRAYS}
    host = {k: np.zeros((max(sizes), cap, 4), np.float32) for k in capi.PREPROCESS_ARRAYS}
    # warm-up of every path at every shape
    loop(h, scans[:2], pp, sp)
    h.preprocess_batch(scans[:max(sizes)], pp, sp, cap=cap, arrays=host)
    h.preprocess_batch(scans[:max(sizes)], pp, sp, cap=cap, dest=MEM_DEVICE, arrays=dev)
    for n in sizes:
        batch = scans[:n]
        times = {"loop": [], "batch_host_out": [], "batch_device_out": []}
        for _ in range(a.reps):
            for name in times:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if name == "loop":
                    ref = loop(h, batch, pp, sp)
                elif name == "batch_host_out":
                    per, _, _ = h.preprocess_batch(batch, pp, sp, cap=cap, arrays=host)
                else:
                    h.preprocess_batch(batch, pp, sp, cap=cap, dest=MEM_DEVICE, arrays=dev)
                torch.cuda.synchronize()
                times[name].append(time.perf_counter() - t0)
        same = all(np.array_equal(per[i][2].view(np.uint32), ref[i].view(np.uint32)) for i in range(n))
        res["throughput"][n] = {k: round(n / float(np.median(v)), 1) for k, v in times.items()}
        res["throughput"][n]["batch_equals_loop"] = bool(same)
        print(n, res["throughput"][n], flush=True)
    # raw scans -> pre-processing -> registration
    p = capi.default_params()
    p.skip_flagged = 0
    P = a.pairs
    raw = scans[:2 * P]
    dv = torch.zeros((2 * P, cap, 4), dtype=torch.float32, device="cuda")
    chain = {"batch_device": [], "single_calls": []}
    for _ in range(a.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _, counts, _ = h.preprocess_batch(raw, pp, sp, cap=cap, dest=MEM_DEVICE, arrays={"valid4": dv})
        rb = h.register_batch([(dv[2 * i].data_ptr(), int(counts[2 * i, 2]), dv[2 * i + 1].data_ptr(), int(counts[2 * i + 1, 2])) for i in range(P)],
                              p, kind=MEM_DEVICE)
        torch.cuda.synchronize()
        chain["batch_device"].append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        v = loop(h, raw, pp, sp)
        rs = h.register_batch([(v[2 * i], v[2 * i + 1]) for i in range(P)], p)
        torch.cuda.synchronize()
        chain["single_calls"].append(time.perf_counter() - t0)
    res["chain_pairs"] = P
    res["chain_registrations_per_s"] = {k: round(P / float(np.median(t)), 1) for k, t in chain.items()}
    res["chain_records_identical"] = rb.tobytes() == rs.tobytes()
    print(json.dumps(res))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))
    h.close()


if __name__ == "__main__":
    main()
