"""Where tc_nn_kernel's time goes: per-role clock64 accounting (QB200_TC_PROF=1 build path), one 64-pair wave of street scans.

  QB200_TC_PROF=1 QB200_LANES=1 python tools/tc_profile.py [--pairs 64] [--scene street|dense]
Prints per-CTA averages in microseconds at the measured SM clock.  Roles: "sched" = the scheduler warp (chooses the tiles,
issues the exact-image copies), "copy" = the operand-copy warp, "epi" = the MMA + filter / evaluation warps (averaged over them).
"stats" holds the wave's exact evaluations, tiles visited and aborted stripes.  "kernel_ms" is the device time per wave of the
seed kernel and of tc_nn_kernel, from torch.profiler on a second handle built without the clock64 accounting.
"""
import argparse, json, os, sys
os.environ.setdefault("QB200_TC_PROF", "1")
os.environ.setdefault("QB200_LANES", "1")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from quatro_b200 import capi, synth

# stats[8 + i] of the kernel (its prof() slots 8..31)
NAMES = {0: "n_cta", 1: "cta_total", 2: "setup", 3: "sched_prologue", 4: "copy_wait_mma", 5: "sched_decide",
         6: "sched_wait_sfree", 11: "epi_wait_a", 12: "epi_wait_x", 13: "epi_wait_hl_and_mma", 14: "epi_vote", 15: "epi_prep",
         16: "epi_filter", 17: "epi_eval", 18: "epi_loop_total", 19: "epi_tiles", 20: "copy_wait_decided", 21: "sched_wait_mma"}

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--scene", default="street")
    ap.add_argument("--mhz", type=float, default=1965.0)
    a = ap.parse_args()
    import bench
    p = bench.scene_params(a.scene)
    pairs = [synth.outdoor_pair(1000 + i)[:2] for i in range(a.pairs)]
    h = capi.Handle(device=0, max_batch_slots=a.pairs, **bench.SCENES[a.scene]["cfg"])
    fp = h.debug_tc_footprint()
    epi_warps = fp["threads"] // 32 - 2   # all warps but the copy and scheduler warps
    for rep in range(3):
        res = h.register_batch(pairs, p)
        prof = h.debug_tc_profile(reset=True)
        st = h.debug_match_stats(reset=True)
    n = float(prof[0])
    out = {"stats": st, "footprint": fp, "n_cta": int(n)}
    cyc_us = 1.0 / a.mhz
    for i, name in sorted(NAMES.items()):
        if i == 0:
            continue
        v = float(prof[i])
        if name.startswith("epi_"):
            v /= epi_warps  # summed over the filter warps
        if name == "epi_tiles":
            out[name + "_per_cta"] = round(v / n, 2)
        else:
            out[name + "_us_per_cta"] = round(v / n * cyc_us, 2)
    h.close()
    # kernel times without the clock64 accounting (the switch is read when a handle is created)
    os.environ["QB200_TC_PROF"] = "0"
    h = capi.Handle(device=0, max_batch_slots=a.pairs, **bench.SCENES[a.scene]["cfg"])
    for rep in range(2):
        h.register_batch(pairs, p)
    waves = 3
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as tp:
        for rep in range(waves):
            h.register_batch(pairs, p)
        torch.cuda.synchronize()
    ms = {}
    for ev in tp.events():
        for k in ("tc_seed_kernel", "tc_nn_kernel"):
            if k in ev.name:
                ms[k] = ms.get(k, 0.0) + (ev.time_range.end - ev.time_range.start) / 1000.0 / waves   # kernel span, us
    out["kernel_ms"] = {k: round(v, 3) for k, v in sorted(ms.items())}
    h.close()
    print(json.dumps(out, indent=1))

if __name__ == "__main__":
    main()
