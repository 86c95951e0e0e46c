"""Where the match stage's time goes: one 64-pair street wave on one lane (QB200_LANES=1) under torch.profiler.

  python tools/match_stage_profile.py [--tree DIR ...] [--pairs 64] [--waves 3] [--out FILE.json]

Every --tree is a source tree with a built library (default: this one); each runs in a process of its own, so two builds (for
example a parent commit and a change) are compared in one call on the same card.  Printed per tree: the device time per wave of
the kernels around the matcher, the match stage's time (stage_ms[3], CUDA events, measured with the profiler off) and, from the
kernel records of the trace, the registers and shared memory each kernel was launched with and how many CTAs of it fit on an SM
beside one tc_nn_kernel CTA.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

KERNELS = ["cloud_sort_kernel", "tuple_test_kernel", "cloud_mean_kernel", "split_desc_kernel", "dedup_kernel", "match_mutual_kernel",
           "scatter_partner_kernel", "pack_corr_kernel", "norm_key_kernel", "broadcast_best_kernel", "tc_nn_kernel"]
CTA_RESERVED = 1024   # shared memory the system reserves per CTA
HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def short(name):
    for k in KERNELS:
        if k in name:
            return k
    return None


def worker(tree, pairs, waves):
    os.environ["QB200_LANES"] = "1"
    sys.path.insert(0, tree)
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    from quatro_b200 import synth
    from quatro_b200.capi import Handle, default_params

    prs = [synth.outdoor_pair(s)[:2] for s in range(pairs)]   # bench.py's street pairs of rank 0
    p = default_params()
    h = Handle(device=0, max_batch_slots=pairs)
    for _ in range(2):
        h.register_batch(prs, p)
    stage = np.zeros(8)
    for _ in range(waves):
        h.register_batch(prs, p)
        stage += h.stage_ms()
    torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        trace = os.path.join(td, "trace.json")
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(waves):
                h.register_batch(prs, p)
            torch.cuda.synchronize()
        prof.export_chrome_trace(trace)
        with open(trace) as f:
            events = json.load(f)["traceEvents"]
    h.close()
    us, calls, res = {}, {}, {}
    all_us = 0.0
    for e in events:
        if e.get("cat") != "kernel":
            continue
        all_us += e["dur"]
        k = short(e["name"])
        if k is None:
            continue
        us[k] = us.get(k, 0.0) + e["dur"]
        calls[k] = calls.get(k, 0) + 1
        a = e.get("args", {})
        res[k] = {"regs": a.get("registers per thread"), "smem": a.get("shared memory"), "block": a.get("block")}
    prop = torch.cuda.get_device_properties(0)
    sm_smem = prop.shared_memory_per_multiprocessor
    tc = res.get("tc_nn_kernel")
    for k, r in res.items():
        if tc is None or r["smem"] is None or r["regs"] is None:
            continue
        threads = 1
        for b in r["block"]:
            threads *= b
        tc_threads = 1
        for b in tc["block"]:
            tc_threads *= b
        by_smem = (sm_smem - (tc["smem"] + CTA_RESERVED)) // (r["smem"] + CTA_RESERVED)
        by_threads = (prop.max_threads_per_multi_processor - tc_threads) // threads
        by_regs = (prop.regs_per_multiprocessor - tc["regs"] * tc_threads) // max(1, r["regs"] * threads)
        r["ctas_beside_tc_nn"] = int(max(0, min(by_smem, by_threads, by_regs)))
    out = {"tree": tree, "gpu": prop.name, "waves": waves, "pairs": pairs,
           "stage_ms": {n: float(v / waves) for n, v in zip(["h2d", "voxel", "fpfh", "match", "graph", "clique", "pose", "d2h"], stage)},
           "kernel_us_per_wave": {k: us[k] / waves for k in KERNELS if k in us},
           "launches_per_wave": {k: calls[k] / waves for k in KERNELS if k in calls},
           "all_kernels_us_per_wave": all_us / waves, "resources": res}
    print("RESULT " + json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", action="append", help="source tree with a built library (repeatable; default: this tree)")
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--waves", type=int, default=3)
    ap.add_argument("--out", help="write the results as JSON here")
    ap.add_argument("--worker", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        worker(a.worker, a.pairs, a.waves)
        return
    results = []
    for tree in a.tree or [HERE]:
        tree = os.path.abspath(tree)
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", tree, "--pairs", str(a.pairs), "--waves", str(a.waves)],
                           capture_output=True, text=True)
        lines = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
        if r.returncode != 0 or not lines:
            raise SystemExit(f"{tree}: worker failed ({r.returncode})\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}")
        results.append(json.loads(lines[-1][len("RESULT "):]))
    names = [os.path.basename(r["tree"].rstrip("/")) or r["tree"] for r in results]
    print(f"{results[0]['gpu']}: {a.pairs}-pair street wave, one lane, mean of {a.waves} waves (us per wave)")
    print(f"{'kernel':<24}" + "".join(f"{n:>16}" for n in names))
    for k in KERNELS:
        print(f"{k:<24}" + "".join(f"{r['kernel_us_per_wave'].get(k, 0.0):>16.1f}" for r in results))
    touched = [k for k in KERNELS if k != "tc_nn_kernel"]
    print(f"{'sum of the above but tc':<24}" + "".join(f"{sum(r['kernel_us_per_wave'].get(k, 0.0) for k in touched):>16.1f}" for r in results))
    print(f"{'all kernels':<24}" + "".join(f"{r['all_kernels_us_per_wave']:>16.1f}" for r in results))
    print(f"{'stage_ms match':<24}" + "".join(f"{r['stage_ms']['match']:>16.3f}" for r in results))
    for k in ("cloud_sort_kernel", "tuple_test_kernel"):
        print(f"{k} regs / smem / CTAs beside tc_nn_kernel: " +
              "  ".join(f"{n}: {r['resources'].get(k, {}).get('regs')} / {r['resources'].get(k, {}).get('smem')} / "
                        f"{r['resources'].get(k, {}).get('ctas_beside_tc_nn')}" for n, r in zip(names, results)))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
