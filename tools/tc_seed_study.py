"""Offline study for tc_nn_kernel's seeds (CPU only): how good are exact distances to a few nearest-norm candidates as the
first row and column bests, and how many 128 x 64 tiles would they let a stripe skip before its first visit?

  python tools/tc_seed_study.py [--pairs 8] [--first-seed 0]

Street pairs of bench.py's generator (synth.outdoor_pair), voxel points and FPFH-33 from the CPU oracle, then the order K6 works
in: the mu-centred fp32 norm chain, a stable sort by norm, runs of bit-identical descriptors collapsed to their first rank.  For
each unique row (column) the seed is the exact distance to the w unique columns (rows) of nearest norm on either side (2 w
candidates), for every w of --widths.  Reported per w, over every unique row and column of every pair:
  ratio_median / ratio_p90 : seeded best / true nearest-neighbour distance (1 = the seed is the answer; pairs at distance 0 count
                             as 1 when the seed is 0 too)
  exact_share              : share of rows and columns whose seed already is the true nearest-neighbour distance
  skip_share               : share of (stripe, column tile) pairs whose norm-gap lower bound (tile_lb in tc_nn_kernel, same
                             slack) is strictly above both the stripe's largest seeded row best and the tile's largest seeded
                             column best -- tiles a stripe can skip before any tile of the pair has been visited
The row "final" uses the true nearest-neighbour distances instead of seeds: the most the same skip test can skip at all.
Distances are float64 here; the kernel's fp32 chain differs in the last bits, which does not move these statistics."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from oracle.oracle_lib import Oracle
from quatro_b200 import capi, synth

MU = np.zeros(33, np.float32)
MU[[5, 16, 27]] = 100.0
TC_M, TC_N = 128, 64
NORM_REL = 4.0e-6   # kTcNormRel of tc_match.cu


def norm_chain(x):
    """|x - mu|^2 by norm_key_kernel's fp32 chain (each square is exact in float64, the sum is rounded to fp32 per step)."""
    xc = (x - MU).astype(np.float32)
    acc = np.zeros(len(x), np.float32)
    for d in range(33):
        acc = (xc[:, d].astype(np.float64) ** 2 + acc.astype(np.float64)).astype(np.float32)
    return acc


def unique_sorted(desc):
    """K6's order: ascending norm (stable: lowest index first), bit-identical runs collapsed to their first rank."""
    nrm = norm_chain(desc)
    order = np.argsort(nrm.view(np.uint32), kind="stable")
    d, n = desc[order], nrm[order]
    keep = np.ones(len(d), bool)
    keep[1:] = ~((n[1:] == n[:-1]) & np.all(d[1:].view(np.uint32) == d[:-1].view(np.uint32), axis=1))
    return d[keep].astype(np.float64), n[keep]


def sqdist(a, b):
    return np.maximum((a * a).sum(1)[:, None] + (b * b).sum(1)[None, :] - 2.0 * a @ b.T, 0.0)


def true_nn(a, b, chunk=1024):
    return np.concatenate([sqdist(a[i:i + chunk], b).min(1) for i in range(0, len(a), chunk)])


def seeds(a, na, b, nb, w):
    """Per unique row of a: min exact distance to the w nearest-norm unique rows of b on either side."""
    p = np.searchsorted(nb, na, side="left")
    best = np.full(len(a), np.inf)
    for k in range(-w, w):
        j = p + k
        ok = (j >= 0) & (j < len(b))
        dd = ((a[ok] - b[j[ok]]) ** 2).sum(1)
        best[ok] = np.minimum(best[ok], dd)
    return best


def tile_skip_share(na, nb, row_best, col_best):
    """Share of (stripe, tile) pairs the scheduler's test skips: lb > max row best of the stripe and > max column best of the tile."""
    sa, sb = np.sqrt(na.astype(np.float32)), np.sqrt(nb.astype(np.float32))
    s_lo, s_hi = sa[::TC_M], sa[np.minimum(np.arange(0, len(sa), TC_M) + TC_M, len(sa)) - 1]
    t_lo, t_hi = sb[::TC_N], sb[np.minimum(np.arange(0, len(sb), TC_N) + TC_N, len(sb)) - 1]
    rmax = np.array([row_best[i:i + TC_M].max() for i in range(0, len(sa), TC_M)])
    cmax = np.array([col_best[j:j + TC_N].max() for j in range(0, len(sb), TC_N)])
    gap = np.maximum(s_lo[:, None] - t_hi[None, :], t_lo[None, :] - s_hi[:, None]) - (2.0e-3 + NORM_REL * (s_hi[:, None] + t_hi[None, :]))
    lb = np.where(gap > 0, gap * gap * 0.9999, 0.0)
    skip = (lb > 0) & (lb > rmax[:, None]) & (lb > cmax[None, :])
    return skip.sum(), skip.size


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=8)
    ap.add_argument("--first-seed", type=int, default=0)
    ap.add_argument("--widths", default="1,2,4,8,16,32")
    a = ap.parse_args()
    widths = [int(x) for x in a.widths.split(",")]
    o = Oracle()
    o.set_num_threads(os.cpu_count() or 8)
    p = capi.default_params()
    acc = {w: {"ratio": [], "skip": 0, "tiles": 0} for w in widths + ["final"]}
    sizes = []
    for s in range(a.first_seed, a.first_seed + a.pairs):
        src, tgt = synth.outdoor_pair(s)[:2]
        clouds = []
        for pts in (src, tgt):
            vox = o.voxelize(pts, p.voxel_size, p.skip_flagged)[0]
            cell = p.grid_cell if p.grid_cell > 0 else p.fpfh_radius * 1.001953125   # the pipeline's default cell
            desc = o.compute_fpfh(vox, p.normal_radius, p.fpfh_radius, cell)[1]
            clouds.append(unique_sorted(desc))
        (A, nA), (B, nB) = clouds
        sizes.append((len(A), len(B)))
        tr, tc = true_nn(A, B), true_nn(B, A)
        for w in widths + ["final"]:
            rb, cb = (tr, tc) if w == "final" else (seeds(A, nA, B, nB, w), seeds(B, nB, A, nA, w))
            for got, ref in ((rb, tr), (cb, tc)):
                acc[w]["ratio"].append(np.where(ref > 0, got / np.where(ref > 0, ref, 1.0), np.where(got > 0, np.inf, 1.0)))
            k, n = tile_skip_share(nA, nB, rb, cb)
            acc[w]["skip"] += k
            acc[w]["tiles"] += n
    out = {"pairs": a.pairs, "unique_rows_cols_mean": [float(np.mean([x[0] for x in sizes])), float(np.mean([x[1] for x in sizes]))]}
    for w in widths + ["final"]:
        r = np.concatenate(acc[w]["ratio"])
        out[str(w)] = {"ratio_median": round(float(np.median(r)), 3), "ratio_p90": round(float(np.percentile(r, 90)), 3),
                       "exact_share": round(float(np.mean(r <= 1.0 + 1e-9)), 3),
                       "skip_share": round(acc[w]["skip"] / max(1, acc[w]["tiles"]), 4)}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
