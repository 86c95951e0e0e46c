"""One dense indoor hall pair with more than 65536 voxel points per cloud, device-resident, on a max_voxel_points = 262144 handle.

  python tools/large_cloud_bench.py [--reps N] [--seed S] [--no-oracle]

The pair is synth.indoor_pair(seed, extent=9.0) (500 k rays per scan; seed 0: 134 k / 101 k voxel points at the 0.05 m voxel) with
the indoor parameters of tests/test_gpu_parity.py::test_dense_indoor_pair_50k_voxels and max_corr = 8192.  After two warm-up calls
it times --reps calls of qb200_register_batch with the scans already on the device and prints one JSON line: the card and its power
limit, the median wall time of a call (CUDA events around it), the median stage times (qb200_get_stage_ms), the matcher counters of
one call (tensor-core tiles, aborted stripes -> whether the exact fallback kernel ran), the device memory the handle allocated, the
record, and whether it equals the CPU oracle's (every counter, pose within 1e-9).  Nothing is written to disk.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from harness import card  # noqa: E402
from quatro_b200 import capi, synth  # noqa: E402

STAGES = ["h2d", "voxel", "fpfh", "match", "graph", "clique", "pose", "d2h"]
KEYS = ["n_src_vox", "n_tgt_vox", "n_mutual", "n_corr", "n_edges", "max_core", "clique_size", "valid", "status"]


def indoor_params():
    p = capi.default_params()
    p.voxel_size, p.normal_radius, p.fpfh_radius, p.noise_bound, p.cote_noise_bound, p.skip_flagged = 0.05, 0.10, 0.15, 0.05, 0.05, 0
    return p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("large_cloud_bench: no CUDA device (the measurement has no CPU fallback)")

    src, tgt, T = synth.indoor_pair(a.seed, extent=9.0)
    p = indoor_params()
    torch.cuda.init()
    free0, _ = torch.cuda.mem_get_info()
    h = capi.Handle(device=0, max_batch_slots=1, max_raw_points=524288, max_voxel_points=262144, max_corr=8192)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    ds, dt = torch.from_numpy(src).cuda(), torch.from_numpy(tgt).cuda()
    arr = (capi.Pair * 1)()
    arr[0].src, arr[0].n_src, arr[0].tgt, arr[0].n_tgt = ds.data_ptr(), len(src), dt.data_ptr(), len(tgt)
    out = np.zeros(1, capi.RESULT_DTYPE)
    torch.cuda.synchronize()
    for _ in range(2):
        h.register_batch_raw(arr, 1, p, capi.MEM_DEVICE, out)
    torch.cuda.synchronize()
    free2, _ = torch.cuda.mem_get_info()   # lanes / scratch created on first use are included here
    wall, stages, match = [], [], None
    for i in range(a.reps):
        h.debug_match_stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        h.register_batch_raw(arr, 1, p, capi.MEM_DEVICE, out)
        e1.record()
        torch.cuda.synchronize()
        wall.append(e0.elapsed_time(e1))
        stages.append(h.stage_ms())
        if match is None:
            match = h.debug_match_stats()
    rec = out[0]
    name, _, limit = card().partition(",")   # card() is "unknown" without nvidia-smi: name the device as torch does
    res = {
        "card": {"name": name.strip() if limit else torch.cuda.get_device_name(), "power_limit": limit.strip() or "unknown"},
        "pair": {"seed": a.seed, "extent": 9.0, "raw": [len(src), len(tgt)]},
        "wall_ms_median": round(float(np.median(wall)), 3),
        "wall_ms": [round(float(x), 3) for x in wall],
        "stage_ms": {k: round(float(v), 3) for k, v in zip(STAGES, np.median(np.array(stages), axis=0))},
        "match_stats": match,
        "exact_fallback_ran": bool(match["aborted_stripes"] > 0),
        "handle_device_mb": {"at_create": round((free0 - free1) / 2**20, 1), "after_warmup": round((free0 - free2) / 2**20, 1)},
        "record": {k: int(rec[k]) for k in KEYS},
    }
    rot, tr = synth.pose_error(rec["T"].reshape(4, 4).T, T)
    res["error_vs_ground_truth"] = {"deg": round(rot, 4), "m": round(tr, 4)}
    if not a.no_oracle:
        from oracle import Oracle
        ref, st = Oracle().register_pair(src, tgt, p)
        same = all(int(rec[k]) == int(getattr(ref, k)) for k in KEYS) and st == rec["status"]
        res["oracle_equal"] = bool(same and np.allclose(rec["T"].reshape(4, 4).T, ref.matrix(), atol=1e-9))
    h.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
