"""What aligning registered pairs in one batch call costs, against the per-set loop of the same call and a torch expression.

256 street pairs from a 64-ring lidar (synth.outdoor_pair, seeds 0..255) are registered once with qb200_register_batch_mixed (the
correspondences kept) and described with qb200_describe_batch_each (the voxel keypoints); every input then lies in device memory.
Each pair is aligned: its raw source scan, its matched source keypoints and its good matches at 3 * voxel_size.  Three ways:
  batch       one qb200_align_batch_each call, device inputs and device outputs (aligned4, matched4, good_ids, good4);
  per_set     the same call once per pair;
  torch       pts @ R.T + t on the padded clouds and matched keypoints, the squared distances and a mask < (3 voxel)^2, in float32
              (not PCL's float64 arithmetic, so its output is not compared byte for byte; its good counts are reported).
Every way runs twice as warm-up, then the rounds alternate them (the median of 5); each is timed with the host clock around calls that
end with a torch.cuda.synchronize.  The batch and per-set outputs are compared byte for byte.  Bytes: 32 per point (16 in, 16 out) and
per correspondence its index pair, both keypoints and the matched point (56), plus each good match's id and point (20).  The rate is
over the whole call, host checks included.  Prints one JSON line with the card and its power limit.

  python tools/align_batch_bench.py [--pairs 256] [--rounds 5] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

from harness import card, timed

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

HBM_PEAK = 3.35e12   # H100 SXM data sheet, bytes/s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    from quatro_b200 import capi, synth
    from quatro_b200.capi import MEM_DEVICE, MEM_HOST, ListBuffers

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU")
    n = a.pairs
    pairs = [synth.outdoor_pair(s)[:2] for s in range(n)]
    p = capi.default_params()
    p.rot_noise_bound = 2 * p.noise_bound
    params = [p] * n
    h = capi.Handle(max_batch_slots=64)
    recs, lists = h.register_batch_mixed(pairs, params, buffers=ListBuffers(n, h.cfg.max_corr, MEM_HOST, capi.MATCH_LISTS))
    vox = lambda: h.feature_buffers(n, h.cfg.max_voxel_points, MEM_HOST, ("vox4",))
    src_kp = h.describe_batch_each([s for s, _ in pairs], params, arrays=vox())[0]
    tgt_kp = h.describe_batch_each([t for _, t in pairs], params, arrays=vox())[0]
    dev = lambda x, dt=torch.float32: torch.from_numpy(np.ascontiguousarray(x)).to("cuda", dt)
    clouds = [dev(s) for s, _ in pairs]
    sk = [dev(k[0]) for k in src_kp]
    tk = [dev(k[0]) for k in tgt_kp]
    corr = [dev(l["corr"], torch.int32) if len(l["corr"]) else None for l in lists]
    Ts = [np.asarray(recs["T"][i]).reshape(4, 4).T for i in range(n)]
    sets = [{"cloud": (clouds[i].data_ptr(), len(clouds[i])), "src_kp": (sk[i].data_ptr(), len(sk[i])),
             "tgt_kp": (tk[i].data_ptr(), len(tk[i])), "corr": None if corr[i] is None else (corr[i].data_ptr(), len(corr[i])),
             "T": Ts[i]} for i in range(n)]
    n_pts = np.array([len(c) for c in clouds])
    n_corr = np.array([len(l["corr"]) for l in lists])
    cp, cc = int(n_pts.max()), max(int(n_corr.max()), 1)
    torch.cuda.synchronize()

    outs = {w: h.align_buffers(n, cp, cc, MEM_DEVICE) for w in ("batch", "per_set")}
    counts = {w: np.zeros((n, 3), np.int32) for w in outs}
    status = {w: np.zeros(n, np.int32) for w in outs}
    arr, _keep = h.align_array(sets, MEM_DEVICE)
    pa = h.params_array(params)
    out_batch = h.align_out(cp, cc, MEM_DEVICE, outs["batch"], counts["batch"], status["batch"])

    def batch():
        h._check(h.lib.qb200_align_batch_each(h.h, arr, n, pa, MEM_DEVICE, capi.C.byref(out_batch)), "align")
        torch.cuda.synchronize()

    one = []
    for i in range(n):
        a1, k1 = h.align_array([sets[i]], MEM_DEVICE)
        views = {k: v[i:i + 1] for k, v in outs["per_set"].items()}
        o1 = h.align_out(cp, cc, MEM_DEVICE, views, counts["per_set"][i:i + 1], status["per_set"][i:i + 1])
        one.append((a1, k1, h.params_array([p]), o1, views))

    def per_set():
        for a1, _, p1, o1, _ in one:
            h._check(h.lib.qb200_align_batch_each(h.h, a1, 1, p1, MEM_DEVICE, capi.C.byref(o1)), "align")
        torch.cuda.synchronize()

    # torch: padded tensors built once, outside the timed region
    P = torch.zeros((n, cp, 3), device="cuda")
    M = torch.zeros((n, cc, 3), device="cuda")
    Q = torch.zeros((n, cc, 3), device="cuda")
    valid = torch.zeros((n, cc), dtype=torch.bool, device="cuda")
    for i in range(n):
        P[i, :len(clouds[i])] = clouds[i][:, :3]
        if corr[i] is not None:
            c = corr[i].long()
            M[i, :len(c)] = sk[i][c[:, 0], :3]
            Q[i, :len(c)] = tk[i][c[:, 1], :3]
            valid[i, :len(c)] = True
    R = torch.tensor(np.stack([T[:3, :3] for T in Ts]), dtype=torch.float32, device="cuda")
    t = torch.tensor(np.stack([T[:3, 3] for T in Ts]), dtype=torch.float32, device="cuda")[:, None, :]
    thr2 = float(3.0 * p.voxel_size) ** 2
    torch_good = {}

    def torch_way():
        aligned = torch.baddbmm(t, P, R.transpose(1, 2))
        matched = torch.baddbmm(t, M, R.transpose(1, 2))
        good = (((matched - Q) ** 2).sum(-1) < thr2) & valid
        torch_good["n"] = good.sum(1)
        torch.cuda.synchronize()
        return aligned

    ms, _ = timed({"batch": batch, "per_set": per_set, "torch": torch_way}, a.warmup, a.rounds)
    same = counts["batch"].tobytes() == counts["per_set"].tobytes() and status["batch"].tobytes() == status["per_set"].tobytes()
    for k in outs["batch"]:
        for i in range(n):
            m = {"aligned4": counts["batch"][i, 0], "matched4": counts["batch"][i, 1]}.get(k, counts["batch"][i, 2])
            same &= bool(torch.equal(outs["batch"][k][i, :m], outs["per_set"][k][i, :m]))
    n_good = counts["batch"][:, 2]
    bytes_moved = 32 * int(n_pts.sum()) + 56 * int(n_corr.sum()) + 20 * int(n_good.sum())
    t_batch = ms["batch"]["median"] * 1e-3
    print(json.dumps({
        "card": card("clocks.max.sm"), "pairs": n, "points": int(n_pts.sum()), "correspondences": int(n_corr.sum()),
        "good": int(n_good.sum()), "torch_good": int(torch_good["n"].sum().item()), "status_ok": int((status["batch"] == 0).sum()),
        "ms": ms, "bytes": bytes_moved, "batch_GBps": bytes_moved / t_batch / 1e9,
        "batch_share_of_hbm_peak": bytes_moved / t_batch / HBM_PEAK,
        "per_set_vs_batch": ms["per_set"]["median"] / ms["batch"]["median"],
        "torch_vs_batch": ms["torch"]["median"] / ms["batch"]["median"], "batch_equals_per_set": bool(same)}))
    h.close()


if __name__ == "__main__":
    main()
