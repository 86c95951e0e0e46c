"""Back-end device times of wide correspondence sets (max_corr up to QB200_MAX_CORR = 32768) and the hall pair with every mutual
nearest neighbour kept.

  python tools/wide_corr_bench.py [--reps N]

Prints one JSON line with the card and its power limit, read in the same run, and:
  * sets: for L = 8192, 16384, 32768 at inlier ratios 0.05 and 0.5 (synth.matched_pairs) on a one-slot max_corr = 32768 handle,
    the median over --reps qb200_solve_batch calls (after two warm-up calls) of the graph stage (K8 + degrees), of tim_graph_kernel
    alone, of the clique stage (K9: k-core, rank permutation, heuristic clique) and of the pose stage (K10/11), all from CUDA events
    (qb200_get_stage_ms / qb200_get_kernel_ms), plus the clique size;
  * small_pair_switch_cost: the L = 8192 sets on a max_corr = 8192 handle, where every array stays in shared memory by
    construction, next to the same sets on the 32768 handle, where the kernels choose shared memory per pair;
  * hall: synth.indoor_pair(0, extent=9.0) with the indoor parameters and use_tuple_test = 0 (31 713 correspondences) on a
    262144-voxel, 32768-correspondence handle, scans on the device: median wall time of qb200_register_batch (CUDA events), its
    stage times, the record and the device memory the handle allocated.
Nothing is written to disk.
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


def time_set(h, a4, b4, p, reps):
    for _ in range(2):
        out = h.solve_batch([(a4, b4)], p)
    st, km = [], []
    for _ in range(reps):
        out = h.solve_batch([(a4, b4)], p)
        st.append(h.stage_ms())
        km.append(h.kernel_ms()[0][1])
    s = np.median(np.array(st), axis=0)
    return {"graph_ms": round(float(s[4]), 3), "tim_graph_kernel_ms": round(float(np.median(km)), 3), "clique_ms": round(float(s[5]), 3),
            "pose_ms": round(float(s[6]), 3), "clique_size": int(out[0]["clique_size"]), "status": int(out[0]["status"])}


def hall_params():
    p = capi.default_params()
    p.voxel_size, p.normal_radius, p.fpfh_radius, p.noise_bound, p.cote_noise_bound, p.skip_flagged = 0.05, 0.10, 0.15, 0.05, 0.05, 0
    p.use_tuple_test = 0
    return p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wide_corr_bench: no CUDA device (the measurement has no CPU fallback)")
    torch.cuda.init()
    name, _, limit = card().partition(",")   # card() is "unknown" without nvidia-smi: name the device as torch does
    res = {"card": {"name": name.strip() if limit else torch.cuda.get_device_name(), "power_limit": limit.strip() or "unknown"},
           "reps": a.reps}
    p = capi.default_params()
    sets = {(L, r): synth.matched_pairs(L + int(100 * r), L, inlier_ratio=r, noise=0.05)[:2] for L in (8192, 16384, 32768) for r in (0.05, 0.5)}
    with capi.Handle(max_batch_slots=1, max_corr=32768) as h:
        res["sets"] = {f"L{L}_r{r}": time_set(h, *sets[(L, r)], p, a.reps) for (L, r) in sets}
    with capi.Handle(max_batch_slots=1, max_corr=8192) as h8:
        res["small_pair_switch_cost"] = {f"L8192_r{r}": {"handle_8192": time_set(h8, *sets[(8192, r)], p, a.reps),
                                                          "handle_32768": res["sets"][f"L8192_r{r}"]} for r in (0.05, 0.5)}

    src, tgt, _ = synth.indoor_pair(0, extent=9.0)
    hp = hall_params()
    free0, _ = torch.cuda.mem_get_info()
    with capi.Handle(max_batch_slots=1, max_raw_points=524288, max_voxel_points=262144, max_corr=32768) as h:
        torch.cuda.synchronize()
        free1, _ = torch.cuda.mem_get_info()
        ds, dt = torch.from_numpy(src).cuda(), torch.from_numpy(tgt).cuda()
        arr = (capi.Pair * 1)()
        arr[0].src, arr[0].n_src, arr[0].tgt, arr[0].n_tgt = ds.data_ptr(), len(src), dt.data_ptr(), len(tgt)
        out = np.zeros(1, capi.RESULT_DTYPE)
        for _ in range(2):
            h.register_batch_raw(arr, 1, hp, capi.MEM_DEVICE, out)
        torch.cuda.synchronize()
        wall, stages = [], []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            h.register_batch_raw(arr, 1, hp, capi.MEM_DEVICE, out)
            e1.record()
            torch.cuda.synchronize()
            wall.append(e0.elapsed_time(e1))
            stages.append(h.stage_ms())
        res["hall"] = {"wall_ms_median": round(float(np.median(wall)), 3), "wall_ms": [round(float(x), 3) for x in wall],
                       "stage_ms": {k: round(float(v), 3) for k, v in zip(STAGES, np.median(np.array(stages), axis=0))},
                       "handle_device_mb": round((free0 - free1) / 2**20, 1), "record": {k: int(out[0][k]) for k in KEYS}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
