"""What one batch of pairs with their own front-end configurations costs: qb200_register_batch_mixed against the calls a caller needs
without it.

The inputs are bench.py's 256 synthetic 64-ring street pairs (synth.outdoor_pair, seeds 0..255), device-resident.  Pair i uses bench.py's
street preset (even i) or its dense preset (odd i: voxel 0.22 m, tuple test off) and one of four tuple-test seeds ((i // 2) mod 4): eight
configurations, 32 pairs each.  Three ways to register them on one handle, on the caller's stream:
  mixed       one qb200_register_batch_mixed call;
  per_config  one qb200_register_batch call per configuration (eight calls of 32 pairs);
  single      256 qb200_register_batch calls of one pair each.
Every way is warmed up first; rounds alternate the three.  Timed with CUDA events on the stream around each (blocking) call sequence;
prints one JSON line with ms per way (median, min, max over the rounds), the card and its power limit, and checks that every record of
the mixed call equals its single-pair call and its per-configuration call byte for byte.

  python tools/per_pair_frontend_bench.py [--rounds 5] [--warmup 2]
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
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()

    import torch
    from bench import gen_pairs, scene_params
    from quatro_b200.capi import Handle, Pair, RESULT_DTYPE, MEM_DEVICE

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
    configs = []
    for scene in ("street", "dense"):
        for seed in (0x5EED, 1, 2, 3):
            p = scene_params(scene)
            p.rot_noise_bound = 2 * p.noise_bound
            p.seed = seed
            configs.append(p)
    cfg_of = [(i % 2) * 4 + (i // 2) % 4 for i in range(P)]
    params = [configs[k] for k in cfg_of]
    members = [[i for i in range(P) if cfg_of[i] == k] for k in range(len(configs))]
    subsets = [(Pair * len(m))(*[pa[i] for i in m]) for m in members]
    h = Handle(max_batch_slots=min(args.slots, P), max_corr=8192)   # bench.py's dense preset needs 8192 correspondences
    h.set_stream(stream.cuda_stream)
    par = h.params_array(params)
    outs = {"mixed": np.zeros(P, RESULT_DTYPE), "single": np.zeros(P, RESULT_DTYPE)}
    per_out = [np.zeros(len(m), RESULT_DTYPE) for m in members]

    def run_mixed():
        h._check(h.lib.qb200_register_batch_mixed(h.h, pa, P, par, MEM_DEVICE, outs["mixed"].ctypes.data, None), "mixed")

    def run_per_config():
        for k, sub in enumerate(subsets):
            h.register_batch_raw(sub, len(members[k]), configs[k], MEM_DEVICE, per_out[k])

    def run_single():
        for i in range(P):
            h.register_batch_raw(one[i], 1, params[i], MEM_DEVICE, outs["single"][i:i + 1])

    ways = {"mixed": run_mixed, "per_config": run_per_config, "single": run_single}
    for fn in ways.values():
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize(dev)
    assert outs["mixed"].tobytes() == outs["single"].tobytes(), "a mixed record differs from its single-pair call"
    for k, m in enumerate(members):
        assert outs["mixed"][m].tobytes() == per_out[k].tobytes(), f"a mixed record differs from its configuration's call ({k})"
    n_corr = [float(np.mean(outs["mixed"]["n_corr"][m])) for m in members]
    ms = {k: [] for k in ways}
    for _ in range(args.rounds):
        for name, fn in ways.items():
            torch.cuda.synchronize(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            fn()
            e1.record(stream)
            torch.cuda.synchronize(dev)
            ms[name].append(e0.elapsed_time(e1))
    med = {k: float(np.median(v)) for k, v in ms.items()}
    print(json.dumps({
        "card": card(), "pairs": P, "slots": h.cfg.max_batch_slots, "configurations": len(configs), "rounds": args.rounds,
        "n_corr_mean_street": float(np.mean(n_corr[:4])), "n_corr_mean_dense": float(np.mean(n_corr[4:])),
        "ms": {k: {"median": med[k], "min": float(min(v)), "max": float(max(v))} for k, v in ms.items()},
        "ms_per_pair": {k: med[k] / P for k in med},
        "mixed_speedup_over_single": med["single"] / med["mixed"],
        "mixed_speedup_over_per_config": med["per_config"] / med["mixed"],
    }))
    h.close()


if __name__ == "__main__":
    main()
