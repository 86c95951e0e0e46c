"""What one batch of individually configured pairs costs: qb200_register_batch_each against the calls a caller needs without it.

A loop-closure sweep on a tilting platform registers every pair with the IMU roll/pitch of its own scan (setPreEstaimatedRyRx).  The
inputs are bench.py's 256 synthetic 64-ring street pairs (synth.outdoor_pair, seeds 0..255), device-resident, each pair with its own
small roll/pitch prior (uniform in +-3 degrees, seeded).  Three configurations on one handle, on the caller's stream:
  each       one qb200_register_batch_each call, pair i with its own RyRx;
  single     256 qb200_register_batch calls of one pair each, pair i with its own RyRx (without _each, one call per configuration);
  broadcast  one qb200_register_batch call of all 256 pairs without the prior, RyRx = identity (what the batch costs when the
             pairs share one configuration).
Every configuration is warmed up first; rounds alternate the configurations.  Timed with CUDA events on the stream around each
(blocking) call sequence; prints one JSON line with ms per configuration (median, min, max over the rounds), the card and its power
limit, and checks that every record of the each call equals its single-pair call byte for byte.

  python tools/per_pair_params_bench.py [--rounds 5] [--warmup 2]
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


def ryrx(roll, pitch):
    rx = np.array([[1, 0, 0], [0, np.cos(roll), -np.sin(roll)], [0, np.sin(roll), np.cos(roll)]])
    ry = np.array([[np.cos(pitch), 0, np.sin(pitch)], [0, 1, 0], [-np.sin(pitch), 0, np.cos(pitch)]])
    return ry @ rx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--slots", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()

    import torch
    from bench import gen_pairs
    from quatro_b200.capi import Handle, Pair, RESULT_DTYPE, MEM_DEVICE, default_params

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
    one = [(Pair * 1)(pa[i]) for i in range(P)]
    rng = np.random.default_rng(7)
    params = []
    for _ in range(P):
        p = default_params()
        p.rot_noise_bound = 2 * p.noise_bound
        p.use_pre_estimated_RyRx = 1
        for k, v in enumerate(ryrx(*np.radians(rng.uniform(-3.0, 3.0, 2))).ravel()):
            p.RyRx[k] = v
        params.append(p)
    base = default_params()
    base.rot_noise_bound = 2 * base.noise_bound
    h = Handle(max_batch_slots=min(args.slots, P))
    h.set_stream(stream.cuda_stream)
    par = h.params_array(params)
    outs = {k: np.zeros(P, RESULT_DTYPE) for k in ("each", "single", "broadcast")}

    def run_each():
        h._check(h.lib.qb200_register_batch_each(h.h, pa, P, par, MEM_DEVICE, outs["each"].ctypes.data, None), "each")

    def run_single():
        for i in range(P):
            h.register_batch_raw(one[i], 1, params[i], MEM_DEVICE, outs["single"][i:i + 1])

    def run_broadcast():
        h.register_batch_raw(pa, P, base, MEM_DEVICE, outs["broadcast"])

    configs = {"each": run_each, "single": run_single, "broadcast": run_broadcast}
    for fn in configs.values():
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize(dev)
    assert outs["each"].tobytes() == outs["single"].tobytes(), "an _each record differs from its single-pair call"
    ms = {k: [] for k in configs}
    for _ in range(args.rounds):
        for name, fn in configs.items():
            torch.cuda.synchronize(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            fn()
            e1.record(stream)
            torch.cuda.synchronize(dev)
            ms[name].append(e0.elapsed_time(e1))
    med = {k: float(np.median(v)) for k, v in ms.items()}
    print(json.dumps({
        "card": card(), "pairs": P, "slots": h.cfg.max_batch_slots, "rounds": args.rounds,
        "n_corr_mean": float(outs["each"]["n_corr"].mean()),
        "ms": {k: {"median": med[k], "min": float(min(v)), "max": float(max(v))} for k, v in ms.items()},
        "ms_per_pair": {k: med[k] / P for k in med},
        "each_speedup_over_single": med["single"] / med["each"],
        "each_over_broadcast": med["each"] / med["broadcast"],
    }))
    h.close()


if __name__ == "__main__":
    main()
