"""Throughput of qb200_preprocess_batch_each on batches whose scans differ in their pre-processing parameters, against what the
broadcast entry point needs for the same batch.

    python tools/preprocess_each_bench.py [--scans 512] [--reps 3] [--out result.json]

Fleet: `scans` generator scans rotating over the five lidar models of the reference (capi.LIDAR_MODELS), each with its model's image;
one _each call against one qb200_preprocess_batch call per model.  Heights: `scans` 64 x 1800 generator scans, each shifted in z and
given its own sensor_height (1.60-1.85 m); one _each call against one call per scan.  Both with host and with device outputs (arrays
allocated once).  Only the C call is timed; configurations alternate, `reps` rounds, scans/s is the median round.  Every
configuration's counts, statuses and output bytes are checked identical to the _each call's in the first round, and the counts in
every round.  The card's name and power limit are read in the same run."""
import argparse
import ctypes as C
import hashlib
import json
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from harness import card  # noqa: E402
from quatro_b200 import capi, synth  # noqa: E402
from quatro_b200.capi import LIDAR_MODELS, MEM_DEVICE, MEM_HOST, PREPROCESS_ARRAYS  # noqa: E402


class Outputs:
    """One set of the four output arrays, (n, cap, 4) float32, host or device, and the descriptors of row ranges of it."""

    def __init__(self, n, cap, dest, device):
        import torch
        self.n, self.cap, self.dest = n, cap, dest
        if dest == MEM_HOST:
            self.arr = {k: np.zeros((n, cap, 4), np.float32) for k in PREPROCESS_ARRAYS}
            self.base = {k: a.ctypes.data for k, a in self.arr.items()}
        else:
            self.arr = {k: torch.zeros((n, cap, 4), dtype=torch.float32, device=f"cuda:{device}") for k in PREPROCESS_ARRAYS}
            self.base = {k: a.data_ptr() for k, a in self.arr.items()}
        self.counts = np.zeros((n, 4), np.int32)
        self.status = np.zeros(n, np.int32)

    def desc(self, row):
        """qb200_preprocess_out of the rows from `row` on."""
        out = capi.PreprocessOut(self.cap, self.dest)
        for k in PREPROCESS_ARRAYS:
            setattr(out, k, self.base[k] + row * self.cap * 16)
        out.counts, out.status = self.counts[row:].ctypes.data, self.status[row:].ctypes.data
        return out

    def digests(self, rows):
        """Per scan (row rows[i]): a digest of its counts, status and the live prefix of its four arrays."""
        host = self.arr if self.dest == MEM_HOST else {k: a.cpu().numpy() for k, a in self.arr.items()}
        out = []
        for r in rows:
            h = hashlib.blake2b(self.counts[r].tobytes() + self.status[r].tobytes())
            for j, k in enumerate(PREPROCESS_ARRAYS):
                h.update(host[k][r, :min(int(self.counts[r, j]), self.cap)].tobytes())
            out.append(h.hexdigest())
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=512)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    lib = capi.load_library()
    N = a.scans
    models = list(LIDAR_MODELS)
    res = {"card": card("clocks.max.sm"), "scans": N, "reps": a.reps}
    h = capi.Handle()

    def run(fn, scans, pp_arg, sp_arg, out):
        ptrs, cnts, keep = capi._scan_arrays(scans, MEM_HOST)
        st = getattr(lib, fn)(h.h, ptrs, cnts, len(scans), MEM_HOST, pp_arg, sp_arg, C.byref(out))
        if st != 0:
            raise capi.QuatroB200Error(st, fn, lib.qb200_last_error(h.h).decode())

    # ---- the two workloads: scans, per-scan entries, and the broadcast calls that cover the same batch ----
    pp0 = capi.default_patchwork_params()
    fleet_scans, fleet_sp = [], []
    for i in range(N):
        m = models[i % 5]
        rings, cols = LIDAR_MODELS[m][:2]
        fleet_scans.append(synth.outdoor_pair(20000 + i, rings=rings, azimuths=cols)[i % 2])
        fleet_sp.append(capi.lidar_segment_params(m))
    fleet_pp = [pp0] * N
    # per model: its scans (in batch order), placed in consecutive rows of the output arrays
    groups = [[i for i in range(N) if i % 5 == g] for g in range(5)]
    fleet_rows = np.empty(N, np.int64)
    r0 = 0
    for g in groups:
        fleet_rows[g] = np.arange(r0, r0 + len(g))
        r0 += len(g)

    base = [s for i in range((N + 1) // 2) for s in synth.outdoor_pair(30000 + i)[:2]][:N]
    heights = [1.60 + 0.25 * i / max(N - 1, 1) for i in range(N)]
    height_scans, height_pp = [], []
    for s, ht in zip(base, heights):
        s = s.copy()
        s[:, 2] += np.float32(1.723 - ht)
        height_scans.append(s)
        p = capi.default_patchwork_params()
        p.sensor_height = ht
        height_pp.append(p)
    sp0 = capi.default_segment_params()
    height_sp = [sp0] * N

    workloads = {
        "fleet": (fleet_scans, fleet_pp, fleet_sp, fleet_rows,
                  [([fleet_scans[i] for i in g], pp0, fleet_sp[g[0]], int(fleet_rows[g[0]])) for g in groups],
                  "one qb200_preprocess_batch call per lidar model"),
        "heights": (height_scans, height_pp, height_sp, np.arange(N),
                    [([s], p, sp0, i) for i, (s, p) in enumerate(zip(height_scans, height_pp))],
                    "one qb200_preprocess_batch call per scan"),
    }
    res["workloads"] = {}
    for name, (scans, pps, sps, rows, broadcast, what) in workloads.items():
        pa, sa = (capi.PatchworkParams * N)(*pps), (capi.SegmentParams * N)(*sps)
        # room for every scan's largest output: counts do not depend on the cap, so a first call with a small cap finds it
        probe = Outputs(N, 1, MEM_HOST, h.cfg.device)
        run("qb200_preprocess_batch_each", scans, pa, sa, probe.desc(0))
        cap = int(probe.counts.max())
        del probe
        entry = {"broadcast_calls": len(broadcast), "broadcast": what, "cap_per_scan": cap, "scans_per_s": {}, "identical": True}
        for dest in (MEM_HOST, MEM_DEVICE):
            outs = Outputs(N, cap, dest, h.cfg.device)
            dname = "host_out" if dest == MEM_HOST else "device_out"
            each_desc = outs.desc(0)
            bc_desc = [(s, C.byref(p), C.byref(q), outs.desc(r)) for s, p, q, r in broadcast]
            # warm-up of both configurations
            run("qb200_preprocess_batch_each", scans, pa, sa, each_desc)
            for s, p, q, d in bc_desc:
                run("qb200_preprocess_batch", s, p, q, d)
            times = {"each": [], "broadcast": []}
            for rep in range(a.reps):
                for cfg in ("each", "broadcast"):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    if cfg == "each":
                        run("qb200_preprocess_batch_each", scans, pa, sa, each_desc)
                    else:
                        for s, p, q, d in bc_desc:
                            run("qb200_preprocess_batch", s, p, q, d)
                    torch.cuda.synchronize()
                    times[cfg].append(time.perf_counter() - t0)
                    if cfg == "each":
                        ref_counts = outs.counts.copy()
                        if rep == 0:
                            ref = outs.digests(range(N))
                    else:
                        same = np.array_equal(outs.counts[rows], ref_counts)
                        if rep == 0:
                            same = same and outs.digests(rows) == ref
                        entry["identical"] = entry["identical"] and bool(same)
            entry["scans_per_s"][dname] = {k: round(N / float(np.median(v)), 1) for k, v in times.items()}
            entry["scans_per_s"][dname]["ms_median"] = {k: round(1e3 * float(np.median(v)), 2) for k, v in times.items()}
            print(name, dname, entry["scans_per_s"][dname], "identical", entry["identical"], flush=True)
            del outs
            torch.cuda.empty_cache()
        res["workloads"][name] = entry
    print(json.dumps(res))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))
    h.close()


if __name__ == "__main__":
    main()
