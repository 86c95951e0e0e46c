"""SPFH rows of the listed points (at most 80 neighbours) from their partial-sum tables.

spfh_kernel<false> turns a bin count c into the SPFH increment added c times in sequence, taking the value from partial sums it
forms 16 at a time.  The descriptors sum the neighbours' SPFH rows, so they are compared with the oracle bit for bit on clouds whose
bins hold counts on both sides of every table boundary: flat grids, where every pair of a neighbourhood shares its f2 and f3 bins
(counts up to k - 1 = 79), a street scan, and a cloud with rare points (more than 80 neighbours) beside listed ones."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

from quatro_b200 import synth
from quatro_b200.capi import Handle, default_params
from support import P4, same_bits

CELL = float(np.float32(0.75) * np.float32(1.001953125))
NORMAL_R, FPFH_R = 0.5, 0.75


def grid(step, origin, n=24):
    g = np.arange(n) * step
    gx, gy = np.meshgrid(g, g)
    return np.c_[gx.ravel(), gy.ravel(), np.zeros(gx.size)] + origin


def clouds(oracle):
    rng = np.random.default_rng(5)
    s, _, _ = synth.outdoor_pair(3, rings=32, azimuths=900)
    street, st = oracle.voxelize(s, 0.3, 1)
    assert st == 0
    # flat grids at 0.2, 0.16 and 0.15 m (about 44, 69 and 78 neighbours inside), one tilted about the x axis
    flat = np.concatenate([grid(0.2, [0, 0, 1]), grid(0.16, [10, 0, 1]), grid(0.15, [20, 0, 1])])
    t = grid(0.2, [0, 10, 0])
    tilted = np.c_[t[:, 0], t[:, 1], 0.5 * (t[:, 1] - 10)]
    planar = P4(np.concatenate([flat, tilted]))
    rare = P4(np.concatenate([rng.normal(0, 0.25, (1500, 3)), rng.uniform(-1.5, 1.5, (500, 3)), rng.normal(0, 0.3, (300, 3)) + [3, 0, 0]]))
    return [("street", street), ("planar", planar), ("rare", rare)]


def neighbour_counts(pts):
    xyz = pts[:, :3].astype(np.float64)
    return np.array([len(x) for x in cKDTree(xyz).query_ball_point(xyz, FPFH_R)])


def test_constructions_reach_the_table_boundaries(oracle):
    k = {name: neighbour_counts(c) for name, c in clouds(oracle)}
    assert k["street"].max() <= 80
    listed = k["planar"][k["planar"] <= 80]
    # listed points whose flat neighbourhoods put more than 16, 32, 48 and 64 pairs into one bin
    assert all(((listed > b + 1) & (listed <= 80)).any() for b in (16, 32, 48, 64)), np.bincount(listed)
    assert (k["rare"] > 80).any() and (k["rare"] <= 80).any()


@pytest.mark.gpu
def test_spfh_rows_match_the_oracle(oracle):
    cs = clouds(oracle)
    refs = [oracle.compute_fpfh(c, NORMAL_R, FPFH_R, CELL) for _, c in cs]
    with Handle(max_batch_slots=2) as h:
        for (name, c), (n_ref, d_ref) in zip(cs, refs):
            n_got, d_got = h.compute_fpfh(c, NORMAL_R, FPFH_R, CELL)
            assert same_bits(n_got, n_ref, nan_equal=True), name
            diff = (d_got.view(np.uint32) != d_ref.view(np.uint32)).any(1)
            assert not diff.any(), f"{name}: {diff.sum()} descriptors differ (first {np.nonzero(diff)[0][:5]})"
        # the three clouds in one describe wave
        p = default_params()
        p.normal_radius, p.fpfh_radius, p.grid_cell = NORMAL_R, FPFH_R, CELL
        outs, counts, status = h.describe_points_each([c for _, c in cs], [p] * len(cs))
        assert (status == 0).all() and list(counts) == [len(c) for _, c in cs]
        for (name, _), (n_ref, d_ref), (nrm, desc) in zip(cs, refs, outs):
            assert same_bits(nrm, n_ref, nan_equal=True) and same_bits(desc, d_ref), name
