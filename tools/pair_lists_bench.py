"""Cost of the per-pair lists of qb200_register_batch_enqueue_ex on the street step of bench.py.

The step is bench.py's: 256 synthetic 64-ring street pairs (synth.outdoor_pair, seeds 0..255) registered as a stream of pipelined
batches from device-resident scans, with the handle on the caller's stream.  Every configuration runs on the same handle and
inputs: records only (qb200_register_batch_enqueue), lists into host (numpy) arrays and lists into device arrays, each at
cap_per_pair 1024 and max_corr.  Rounds alternate the configurations so that drift of the shared machine spreads over all of them.
Prints one JSON line: registrations/s per configuration (median, min, max over the rounds), the card and its power limit.

  python tools/pair_lists_bench.py [--steps 10] [--rounds 5]
  QB200_TIMELINE=1 python tools/pair_lists_bench.py --timeline     (one blocking batch per configuration; wave boundaries on stderr)
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

from harness import card

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--slots", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10, help="batches per timed window")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--timeline", action="store_true", help="one blocking batch per configuration, nothing timed")
    args = ap.parse_args()

    import torch
    from bench import gen_pairs
    from quatro_b200.capi import Handle, ListBuffers, Pair, RESULT_DTYPE, MEM_HOST, MEM_DEVICE, default_params

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream(dev)
    P = args.pairs
    prs = gen_pairs(range(P))
    flat = np.concatenate([c for pr in prs for c in pr]).astype(np.float32)
    dvc = torch.from_numpy(flat).to(dev)
    pa = (Pair * P)()
    o = 0
    for i, (s, t) in enumerate(prs):
        pa[i].src, pa[i].n_src = dvc.data_ptr() + o * 16, len(s); o += len(s)
        pa[i].tgt, pa[i].n_tgt = dvc.data_ptr() + o * 16, len(t); o += len(t)
    h = Handle(max_batch_slots=min(args.slots, P))
    h.set_stream(stream.cuda_stream)
    p = default_params()
    out = np.zeros(P, RESULT_DTYPE)
    mc = h.cfg.max_corr
    configs = {"none": None}
    for cap in (1024, mc):
        configs[f"host_cap{cap}"] = ListBuffers(P, cap, MEM_HOST)
        configs[f"device_cap{cap}"] = ListBuffers(P, cap, MEM_DEVICE, device=0)

    def step(lb):
        if lb is None:
            h.register_batch_enqueue_raw(pa, P, p, MEM_DEVICE, out)
        else:
            h.register_batch_enqueue_lists_raw(pa, P, p, MEM_DEVICE, out, lb)

    if args.timeline:
        for name, lb in configs.items():
            print(f"[{name}]", file=sys.stderr, flush=True)
            step(lb)
            h.register_batch_flush()
        return

    ref = None
    for name, lb in configs.items():       # warm-up: every configuration's staging and kernels; every configuration, the same records
        for _ in range(args.warmup):
            step(lb)
        h.register_batch_flush()
        rec = out.copy()
        rec["flags"] &= ~2
        ref = rec.tobytes() if ref is None else ref
        assert rec.tobytes() == ref, name
    rates = {k: [] for k in configs}
    for _ in range(args.rounds):
        for name, lb in configs.items():
            h.register_batch_flush()
            torch.cuda.synchronize(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(args.steps):
                step(lb)
            h.register_batch_flush()
            e1.record(stream)
            torch.cuda.synchronize(dev)
            rates[name].append(P * args.steps / (e0.elapsed_time(e1) / 1e3))
    n_corr = out["n_corr"]
    print(json.dumps({
        "card": card(), "pairs": P, "slots": h.cfg.max_batch_slots, "steps": args.steps, "rounds": args.rounds,
        "n_corr_mean": float(n_corr.mean()), "n_corr_max": int(n_corr.max()),
        "registrations_per_s": {k: {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))} for k, v in rates.items()},
    }))
    h.close()


if __name__ == "__main__":
    main()
