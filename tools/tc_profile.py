"""Where tc_nn_kernel's time goes: per-role clock64 accounting (QB200_TC_PROF=1 build path), one 64-pair wave of street scans.

  QB200_TC_PROF=1 QB200_LANES=1 python tools/tc_profile.py [--pairs 64] [--scene street|dense]
Prints per-CTA averages in microseconds at the measured SM clock.
"""
import argparse, json, os, sys
os.environ.setdefault("QB200_TC_PROF", "1")
os.environ.setdefault("QB200_LANES", "1")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from quatro_b200 import capi, synth

NAMES = ["n_cta", "cta_total", "setup", "copy_prologue", "copy_wait_mma", "copy_decide", "copy_wait_sfree", "unused_15", "unused_16",
         "unused_17", "unused_18", "epi_wait_a", "epi_wait_x", "epi_wait_hl_and_mma", "epi_vote", "epi_prep", "epi_filter", "epi_eval",
         "epi_loop_total", "epi_tiles"]

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
    for rep in range(3):
        res = h.register_batch(pairs, p)
        prof = h.debug_tc_profile(reset=True)
        st = h.debug_match_stats(reset=True)
    n = float(prof[0])
    out = {"stats": st, "n_cta": int(n)}
    cyc_us = 1.0 / a.mhz
    for i, name in enumerate(NAMES[1:], start=1):
        v = float(prof[i])
        if name.startswith("epi_") and name != "epi_tiles":
            v /= 16.0  # summed over the 16 filter warps
        if name == "epi_tiles":
            out[name + "_per_cta"] = round(v / 16.0 / n, 2)
        else:
            out[name + "_us_per_cta"] = round(v / n * cyc_us, 2)
    print(json.dumps(out, indent=1))

if __name__ == "__main__":
    main()
