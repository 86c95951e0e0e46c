"""Scratch reuse: every wave reads the live part of its lane's buffers and nothing past it.

A handle keeps its lanes' buffers for its whole life, and waves of every kind and size reuse them.  Each test here first fills the
slots of one lane to capacity ("soil": raw pairs at max_voxel_points voxels, complete graphs and correspondence and inlier sets at
max_corr, caller features with non-finite bins, describe and voxelize waves, the single-pair calls), then runs a smaller wave of
another kind on the same slots ("probe") at the sizes where a read past the live part lands on stale data: L = 0, 1, 2, 31, 32, 33,
63, 64, 65 (32-bit adjacency words), cliques of 0, 1 and 2 members (no inlier masks), words_per_row above ceil(L / 32), keypoint
counts around the 64-column tiles and 128-row stripes.  Each probe's outputs must equal the oracle's and, byte for byte, the same
probe's outputs on a freshly created handle; entries past each live count keep the 0xA5 sentinel.

The single-pair getters read lane 0's slot 0: after a later wave on lane 0 they refuse instead of handing out another call's
entries."""
import numpy as np
import pytest

from quatro_b200 import synth
from quatro_b200.capi import (FLAG_LISTS_TRUNCATED, GRAPH_LISTS, INLIER_NONE, MATCH_LISTS, MEM_DEVICE, MEM_HOST, PMC_EXACT, PMC_HEU, SET_LISTS,
                              LIST_LAYOUT, GraphBuffers, ListBuffers, QuatroB200Error)
from support import assert_same_record, fpfh_like, make_handle, make_params, same_bits, same_lists, sentinel, sentinel_lists

SLOTS, V, LC, RAW = 4, 1024, 1024, 4096
CFG = dict(max_batch_slots=SLOTS, max_voxel_points=V, max_corr=LC, max_raw_points=RAW)
PROBE_L = (0, 1, 2, 31, 32, 33, 63, 64, 65)
WPR = 5                                      # words per exported or caller row: above ceil(65 / 32) = 3
ROWS, CAP_EDGES, CAP_CLIQUE = max(PROBE_L), 65 * 64 // 2, 8
SENT32 = 0xA5A5A5A5
MATCH_SIZES = ((1, 1), (2, 3), (63, 65), (129, 128), (V - 1, 64))
POSE_IDS = ((33, 0), (1, 1), (2, 2), (65, 31), (65, 33))   # (L of the probe set, inlier ids)


# ---- inputs -------------------------------------------------------------------------------------------------------------------------
def lattice(seed, n, spacing=1.2, jitter=0.1):
    """n points on a jittered cubic lattice: points at least spacing - 2 jitter = 1.0 apart, more than the 0.866 diagonal of a 0.5
    voxel, so every point is its own voxel whatever rigid motion moves the cloud"""
    rng = np.random.default_rng(seed)
    side = int(np.ceil(n ** (1 / 3)))
    g = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing="ij"), -1).reshape(-1, 3)[:n] * spacing
    pts = np.ones((n, 4), np.float32)
    pts[:, :3] = g + rng.uniform(-jitter, jitter, g.shape)
    return pts


def moved(pts, yaw=0.2, t=(1.0, 2.0, 0.0)):
    c, s = np.cos(yaw), np.sin(yaw)
    out = pts.copy()
    out[:, :3] = pts[:, :3] @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]], np.float32).T + np.float32(t)
    return out


FRONT = dict(voxel_size=0.5, normal_radius=2.0, fpfh_radius=3.0)


def corr_set(seed, L, inlier_ratio=0.6):
    a4, b4, _, _ = synth.matched_pairs(seed, max(L, 1), inlier_ratio=inlier_ratio, noise=0.03)
    return np.ascontiguousarray(a4[:L]), np.ascontiguousarray(b4[:L])


def complete_rows(L):
    """adjacency rows of the complete graph on L vertices: every word all ones but the diagonal bit"""
    a = np.full((L, (L + 31) // 32), 0xFFFFFFFF, np.uint32)
    a[np.arange(L), np.arange(L) >> 5] &= ~(np.uint32(1) << (np.arange(L) & 31).astype(np.uint32))
    return a


def hostile_features(seed, n):
    """n keypoints with FPFH-like rows, some bins NaN, +inf or 3e38, and runs of bit-identical rows"""
    rng = np.random.default_rng(seed)
    d = fpfh_like(rng, n)
    d[rng.random(n) < 0.02, rng.integers(0, 33)] = np.nan
    d[rng.random(n) < 0.02, rng.integers(0, 33)] = np.inf
    d[rng.random(n) < 0.02, rng.integers(0, 33)] = 3e38
    for s in range(0, n - 8, 97):
        d[s:s + 8] = d[s]
    pts = np.ones((n, 4), np.float32)
    pts[:, :3] = rng.uniform(-30, 30, (n, 3))
    return pts, d


PROBE_SETS = [corr_set(900 + L, L) for L in PROBE_L]
SOIL_SETS = [corr_set(700 + i, LC, 0.9) for i in range(SLOTS)]


def tim_rows(oracle, a, b, p, wpr=None):
    """the oracle's TIM graph of one set: (adjacency rows, degrees, edge count)"""
    return oracle.build_graph(a, b, p.noise_bound, p.cbar2, wpr)


def probe_graphs(oracle):
    """(graphs, params, oracle adjacency) of the clique probe: the TIM rows of every probe set with all-ones words past
    ceil(L / 32) (columns >= L are ignored), then an empty graph, an edgeless one and one with a single edge (cliques of 0, 0 and 2
    members; one-member cliques come through the pose probe)"""
    p = make_params()
    graphs, params, adj = [], [], []
    for i, (a, b) in enumerate(PROBE_SETS):
        L = len(a)
        rows = tim_rows(oracle, a, b, p)[0] if L else np.zeros((0, 1), np.uint32)
        g = np.full((L, WPR), 0xFFFFFFFF, np.uint32)
        g[:, :rows.shape[1]] = rows
        graphs.append(g), adj.append(rows), params.append(make_params(inlier_selection_mode=PMC_EXACT if i % 2 else PMC_HEU))
    one_edge = np.zeros((40, 2), np.uint32)
    one_edge[3, 0] |= np.uint32(1 << 17)
    one_edge[17, 0] |= np.uint32(1 << 3)
    for rows in (np.zeros((0, WPR), np.uint32), np.zeros((5, WPR), np.uint32), one_edge):
        graphs.append(rows), adj.append(rows), params.append(make_params(inlier_selection_mode=PMC_HEU))
    return graphs, params, adj


def match_pairs():
    rng = np.random.default_rng(5)
    out = []
    for ns, nt in MATCH_SIZES:
        s4, t4 = (np.ones((n, 4), np.float32) for n in (ns, nt))
        s4[:, :3], t4[:, :3] = rng.uniform(-20, 20, (ns, 3)), rng.uniform(-20, 20, (nt, 3))
        s4[:, 3], t4[:, 3] = rng.uniform(0, 1, ns), rng.uniform(0, 1, nt)
        out.append((s4, fpfh_like(rng, ns), t4, fpfh_like(rng, nt)))
    return out


MATCH_PAIRS = match_pairs()


# ---- soils: every slot of the lane filled to capacity by one kind of wave -----------------------------------------------------------
def soil_raw(h):
    pairs = [(lattice(i, V), moved(lattice(i, V))) for i in range(SLOTS - 1)] + [(lattice(9, 1100), lattice(10, V))]
    h.register_batch_each(pairs, [make_params(**FRONT, inlier_selection_mode=PMC_EXACT)] * SLOTS,
                          buffers=ListBuffers(SLOTS, LC))


def soil_features(h):
    pairs = [(*hostile_features(2 * i, V), *hostile_features(2 * i + 1, V)) for i in range(SLOTS)]
    h.register_features_each(pairs, [make_params()] * SLOTS, buffers=ListBuffers(SLOTS, LC))


def soil_graphs(h):
    h.max_clique_batch_each([complete_rows(LC)] * SLOTS, [make_params(inlier_selection_mode=PMC_HEU)] * SLOTS,
                            buffers=ListBuffers(SLOTS, LC, MEM_HOST, GRAPH_LISTS))


def soil_sets(h):
    h.solve_batch_each(SOIL_SETS, [make_params(inlier_selection_mode=INLIER_NONE)] * SLOTS, buffers=ListBuffers(SLOTS, LC, MEM_HOST, SET_LISTS))
    h.build_graph_batch_each(SOIL_SETS, [make_params()] * SLOTS, buffers=GraphBuffers(SLOTS, LC, LC // 32, 1000))


def soil_pose(h):
    params = [make_params(using_rot_inliers_when_estimating_cote=i % 2) for i in range(SLOTS)]
    h.solve_pose_batch_each(SOIL_SETS, [np.arange(LC)[::-1]] * SLOTS, params, buffers=ListBuffers(SLOTS, LC, MEM_HOST, SET_LISTS))


def soil_scans(h):
    p = [make_params(**FRONT)] * (2 * SLOTS)
    h.describe_batch_each([lattice(20 + i, V) for i in range(2 * SLOTS)], p)
    h.voxelize_batch_each([lattice(30 + i, RAW) for i in range(2 * SLOTS)], p)


def soil_single(h):
    p = make_params(**FRONT)
    src, tgt = lattice(40, V), moved(lattice(40, V))
    h.register_pair(src, tgt, p)
    h.match_and_pack(src, tgt, p)
    h.compute_fpfh(src, p.normal_radius, p.fpfh_radius, p.fpfh_radius * 1.001953125)
    h.max_clique(complete_rows(LC), PMC_HEU)
    h.solve_pose(*SOIL_SETS[0], np.arange(LC), make_params())


SOILS = {"raw": soil_raw, "features": soil_features, "graphs": soil_graphs, "sets": soil_sets, "pose": soil_pose, "scans": soil_scans,
         "single": soil_single}


# ---- probes: smaller waves of every kind; each returns its records and raw output arrays, and checks them against the oracle ------
def probe_graph(h):
    """the TIM graphs of the probe sets into host arrays (copied out at collect time) and into device arrays (graph_export_kernel)"""
    out = {}
    for kind, tag in ((MEM_HOST, ""), (MEM_DEVICE, "_dev")):
        gb = GraphBuffers(len(PROBE_SETS), ROWS, WPR, CAP_EDGES, kind, fill=SENT32, device=h.cfg.device)
        out["records" + tag] = h.build_graph_batch_each(PROBE_SETS, [make_params()] * len(PROBE_SETS), buffers=gb)
        out.update({k + tag: gb.host(k).copy() for k in ("adj", "degree", "edges")})
    return out


def check_graph(out, oracle):
    for tag in ("", "_dev"):
        check_graph_kind({k[:len(k) - len(tag)]: v for k, v in out.items() if k.endswith(tag)} if tag else out, oracle)


def check_graph_kind(out, oracle):
    p = make_params()
    for i, (a, b) in enumerate(PROBE_SETS):
        L, r = len(a), out["records"][i]
        adj, deg, ne = tim_rows(oracle, a, b, p, WPR) if L else (np.zeros((0, WPR), np.uint32), np.zeros(0, np.int32), 0)
        assert (r["status"], r["n_corr"], r["n_edges"]) == (0, L, ne), (L, r)
        assert out["adj"][i, :L].tobytes() == adj.tobytes(), L          # words ceil(L / 32) .. WPR - 1 are zero in adj
        assert out["degree"][i, :L].tobytes() == deg.tobytes(), L
        assert (out["adj"][i, L:] == SENT32).all() and (out["degree"][i, L:].view(np.uint32) == SENT32).all(), L
        dense = np.unpackbits(adj.view(np.uint8), axis=1, bitorder="little")[:, :L].astype(bool)
        edges = np.argwhere(np.triu(dense, 1)).astype(np.int32)
        assert out["edges"][i, :ne].tobytes() == edges.tobytes(), L
        assert (out["edges"][i, ne:].view(np.uint32) == SENT32).all(), L


def probe_clique(h, oracle):
    graphs, params, _ = probe_graphs(oracle)
    lb = sentinel_lists(ListBuffers(len(graphs), CAP_CLIQUE, MEM_HOST, GRAPH_LISTS))
    recs, _ = h.max_clique_batch_each(graphs, params, buffers=lb)
    return {"records": recs, "clique": lb.host("clique").copy()}


def check_clique(out, oracle):
    graphs, params, adj = probe_graphs(oracle)
    for i, (rows, p) in enumerate(zip(adj, params)):
        L, r = rows.shape[0], out["records"][i]
        oc, _, _, omc, _ = oracle.max_clique_ex(rows, p.inlier_selection_mode) if L else (np.zeros(0, np.int32), 0, 0, 0, 0)
        n_edges = int(np.unpackbits(rows.view(np.uint8)).sum()) // 2
        assert (r["status"], r["n_corr"], r["n_edges"], r["clique_size"], r["max_core"]) == (0, L, n_edges, len(oc), omc), (i, r)
        m = min(len(oc), CAP_CLIQUE)
        assert out["clique"][i, :m].tobytes() == oc[:m].astype(np.int32).tobytes(), i
        assert (out["clique"][i, m:].view(np.uint32) == SENT32).all(), i
        assert bool(r["flags"] & FLAG_LISTS_TRUNCATED) == (len(oc) > CAP_CLIQUE), i
    assert [int(r["clique_size"]) for r in out["records"][-3:]] == [0, 0, 2]


def probe_solve(h):
    lb = sentinel_lists(ListBuffers(len(PROBE_SETS), LC, MEM_HOST, SET_LISTS))
    params = [make_params(inlier_selection_mode=PMC_EXACT if i % 3 == 0 else PMC_HEU) for i in range(len(PROBE_SETS))]
    recs, _ = h.solve_batch_each(PROBE_SETS, params, buffers=lb)
    return {"records": recs, **{k: lb.host(k).copy() for k in SET_LISTS}, "params": params}


def check_lists_tail(out, i, counts):
    for name, m in counts.items():
        assert (out[name][i, m:].view(np.uint8) == 0xA5).all(), (i, name)


def check_solve(out, oracle):
    for i, ((a, b), p) in enumerate(zip(PROBE_SETS, out["params"])):
        r, L = out["records"][i], len(a)
        nq, nf = int(r["clique_size"]), int(r["n_final_inliers"])
        got = {k: out[k][i, :nq] for k in ("clique", "rot_inlier_mask", "trans_inlier_mask")}
        got["final_inliers"] = out["final_inliers"][i, :nf]
        if L < 2:   # the oracle returns before it fills its sets; a degenerate clique has no solved masks
            assert not got["rot_inlier_mask"].any() and not got["trans_inlier_mask"].any(), L
        else:
            _, _, clique, fin = oracle.solve_correspondences(a, b, p, want_sets=True)
            _, rm, tm, _ = oracle.solve_pose(a, b, clique, p)
            same_lists(got, {"clique": clique, "final_inliers": fin, "rot_inlier_mask": rm, "trans_inlier_mask": tm})
        check_lists_tail(out, i, {"clique": nq, "rot_inlier_mask": nq, "trans_inlier_mask": nq, "final_inliers": nf})


def pose_inputs():
    sets = [PROBE_SETS[PROBE_L.index(L)] for L, _ in POSE_IDS]
    ids = [np.arange(n)[::-1].astype(np.int32) for _, n in POSE_IDS]
    params = [make_params(using_rot_inliers_when_estimating_cote=i % 2) for i in range(len(POSE_IDS))]
    return sets, ids, params


def probe_pose(h):
    sets, ids, params = pose_inputs()
    lb = sentinel_lists(ListBuffers(len(sets), LC, MEM_HOST, SET_LISTS))
    recs, _ = h.solve_pose_batch_each(sets, ids, params, buffers=lb)
    return {"records": recs, **{k: lb.host(k).copy() for k in SET_LISTS}}


def check_pose(out, oracle):
    for i, ((a, b), ids, p) in enumerate(zip(*pose_inputs())):
        r = out["records"][i]
        nq, nf = int(r["clique_size"]), int(r["n_final_inliers"])
        assert nq == len(ids) and out["clique"][i, :nq].tobytes() == ids.tobytes(), i
        rm, tm = out["rot_inlier_mask"][i, :nq], out["trans_inlier_mask"][i, :nq]
        if nq < 2:
            assert not rm.any() and not tm.any(), i
        else:
            _, orm, otm, _, ofin = oracle.solve_pose(a, b, ids, p, want_final=True)
            assert rm.tobytes() == orm.tobytes() and tm.tobytes() == otm.tobytes(), i
            assert out["final_inliers"][i, :nf].tobytes() == ofin.tobytes(), i
        check_lists_tail(out, i, {"clique": nq, "rot_inlier_mask": nq, "trans_inlier_mask": nq, "final_inliers": nf})


def probe_match(h):
    lb = sentinel_lists(ListBuffers(len(MATCH_PAIRS), LC, MEM_HOST, MATCH_LISTS))
    recs, _ = h.match_features_each(MATCH_PAIRS, [make_params()] * len(MATCH_PAIRS), buffers=lb)
    return {"records": recs, **{k: lb.host(k).copy() for k in MATCH_LISTS}}


def check_match(out, oracle):
    for i, (s4, sd, t4, td) in enumerate(MATCH_PAIRS):
        r = out["records"][i]
        corr, nm, _ = oracle.match(s4, sd, t4, td, make_params())
        n = len(corr)
        assert (r["n_src_vox"], r["n_tgt_vox"], r["n_mutual"], r["n_corr"]) == (len(s4), len(t4), nm, n), (i, r)
        # a match record is not solved: every solver field as on a fresh record
        assert (r["n_edges"], r["max_core"], r["clique_size"], r["gnc_iters"], r["n_rot_inliers"], r["n_final_inliers"], r["valid"]) == \
            (0,) * 7, (i, r)
        assert np.array_equal(np.asarray(r["T"]), np.eye(4).reshape(-1)) and r["cost"] == 0.0, i
        assert out["corr"][i, :n].tobytes() == corr.tobytes(), i
        assert out["src_matched4"][i, :n].tobytes() == s4[corr[:, 0]].tobytes(), i
        assert out["tgt_matched4"][i, :n].tobytes() == t4[corr[:, 1]].tobytes(), i
        check_lists_tail(out, i, {k: n for k in MATCH_LISTS})


VOXEL_COUNTS = (1, 2, 63, 64, 65, 127, 128, 129, V - 1)
RAW_SIZES = ((1, 2), (63, 64), (65, 127), (128, 129), (V - 1, V - 1))


def probe_voxelize(h):
    """one point per voxel, so the counts sit on the 64-column tiles and 128-row stripes"""
    vox = sentinel((len(VOXEL_COUNTS), V, 4))
    _, counts, status = h.voxelize_batch_each([lattice(60 + n, n) for n in VOXEL_COUNTS], [make_params(**FRONT)] * len(VOXEL_COUNTS),
                                              arrays={"vox4": vox})
    return {"counts": counts, "status": status, "vox4": vox}


def check_voxelize(out, oracle):
    for i, n in enumerate(VOXEL_COUNTS):
        want, st = oracle.voxelize(lattice(60 + n, n), FRONT["voxel_size"])
        assert (out["counts"][i], out["status"][i], st) == (n, 0, 0), (n, out["counts"][i], out["status"][i])
        assert same_bits(out["vox4"][i, :n], want), n
        assert (out["vox4"][i, n:].view(np.uint32) == SENT32).all(), n


def raw_pairs():
    return [(lattice(70 + a, a), moved(lattice(71 + b, b))) for a, b in RAW_SIZES]


def probe_raw(h):
    lb = sentinel_lists(ListBuffers(len(RAW_SIZES), LC))
    recs, _ = h.register_batch_each(raw_pairs(), [make_params(**FRONT)] * len(RAW_SIZES), buffers=lb)
    return {"records": recs, **{k: lb.host(k).copy() for k in LIST_LAYOUT}}


def check_raw(out, oracle):
    for i, (src, tgt) in enumerate(raw_pairs()):
        r = out["records"][i]
        res, _ = oracle.register_pair(src, tgt, make_params(**FRONT))
        assert_same_record(r, res)
        counts = {k: min(int(r[LIST_LAYOUT[k][2]]), LC) for k in LIST_LAYOUT}
        check_lists_tail(out, i, counts)
        if counts["corr"]:
            c = out["corr"][i, :counts["corr"]]
            assert out["src_matched4"][i, :len(c), :3].tobytes() == oracle.voxelize(src, FRONT["voxel_size"])[0][c[:, 0], :3].tobytes(), i


PROBES = {"graph": (lambda h, o: probe_graph(h), check_graph), "clique": (probe_clique, check_clique),
          "solve": (lambda h, o: probe_solve(h), check_solve), "pose": (lambda h, o: probe_pose(h), check_pose),
          "match": (lambda h, o: probe_match(h), check_match), "voxelize": (lambda h, o: probe_voxelize(h), check_voxelize),
          "raw": (lambda h, o: probe_raw(h), check_raw)}


def same_outputs(got, want, label):
    for k in want:
        if k == "params":
            continue
        assert np.asarray(got[k]).tobytes() == np.asarray(want[k]).tobytes(), (label, k)


# ---- CPU: the constructions reach their targets ---------------------------------------------------------------------------------------
def test_soil_and_probe_inputs_reach_their_targets(oracle):
    for n in (V, 1100):
        vox, st = oracle.voxelize(lattice(3, n), FRONT["voxel_size"])
        assert st == 0 and len(vox) == n                        # one voxel per point: n_vox = V, and V + 76 overflows the handle
        assert len(oracle.voxelize(moved(lattice(3, n)), FRONT["voxel_size"])[0]) == n
    assert len(oracle.voxelize(lattice(30, RAW), FRONT["voxel_size"])[0]) == RAW
    assert [len(a) for a, _ in SOIL_SETS] == [LC] * SLOTS
    adj, _, ne = tim_rows(oracle, *SOIL_SETS[0], make_params())
    assert adj.shape == (LC, LC // 32) and ne > LC * 100          # dense rows across every word of the row
    full = complete_rows(LC)
    assert (full.view(np.uint8) == 0xFF).mean() > 0.99 and not np.any(full[np.arange(LC), np.arange(LC) >> 5] >> (np.arange(LC) & 31) & 1)
    assert [len(a) for a, _ in PROBE_SETS] == list(PROBE_L) and WPR > (max(PROBE_L) + 31) // 32
    graphs, params, adj = probe_graphs(oracle)
    sizes = [len(oracle.max_clique_ex(a, PMC_HEU)[0]) if a.shape[0] else 0 for a in adj[-3:]]
    assert sizes == [0, 0, 2]                                    # an edgeless graph's clique is empty
    assert any(len(oracle.max_clique_ex(a, PMC_HEU)[0]) > CAP_CLIQUE for a in adj[:-3] if a.shape[0])   # cap below and above
    assert [n for _, n in POSE_IDS] == [0, 1, 2, 31, 33]
    d = hostile_features(0, V)[1]
    assert np.isnan(d).any() and np.isposinf(d).any() and (d == np.float32(3e38)).any()
    assert {n % 64 for n, _ in MATCH_SIZES} >= {1, 63} and any(n > 128 for n, _ in MATCH_SIZES)
    assert [len(oracle.voxelize(lattice(60 + n, n), FRONT["voxel_size"])[0]) for n in VOXEL_COUNTS] == list(VOXEL_COUNTS)
    assert [len(a) for a, _ in WIDE_SETS] == list(WIDE_L) and [len(a) for a, _ in SOIL_SETS_B] == [LC_B] * 2
    assert V_B > 17920 and LC_B > 8192 and WPR_B > (max(WIDE_L) + 31) // 32


# ---- GPU: soil x probe on one lane ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def reference(oracle):
    """every probe's outputs on a freshly created handle, checked against the oracle once"""
    out = {}
    for name, (run, check) in PROBES.items():
        with make_handle(1, **CFG) as h:
            out[name] = run(h, oracle)
        check(out[name], oracle)
    return out


@pytest.fixture(scope="module")
def handle_a():
    h = make_handle(1, **CFG)
    yield h
    h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("probe", list(PROBES))
@pytest.mark.parametrize("soil", list(SOILS))
def test_probe_after_soil_equals_a_fresh_handle_and_the_oracle(handle_a, reference, oracle, soil, probe):
    run, check = PROBES[probe]
    SOILS[soil](handle_a)
    got = run(handle_a, oracle)
    same_outputs(got, reference[probe], (soil, probe))
    check(got, oracle)


@pytest.mark.gpu
def test_four_lanes_soiled_then_probed_equal_one_lane(reference, oracle):
    """16 sets or graphs per soil call: one wave on each of the four lanes; the probes' waves land on three of them"""
    with make_handle(4, **CFG) as h:
        h.solve_batch_each(SOIL_SETS * 4, [make_params(inlier_selection_mode=INLIER_NONE)] * 16,
                           buffers=ListBuffers(16, LC, MEM_HOST, SET_LISTS))
        h.max_clique_batch_each([complete_rows(LC)] * 16, [make_params()] * 16)
        h.build_graph_batch_each(SOIL_SETS * 4, [make_params()] * 16, buffers=GraphBuffers(16, LC, LC // 32, 1))
        for name, (run, _) in PROBES.items():
            same_outputs(run(h, oracle), reference[name], name)


# ---- GPU: the single-pair getters after a later wave on lane 0 --------------------------------------------------------------------------
GETTERS = {"clique": lambda h: h.last_clique(), "final_inliers": lambda h: h.last_final_inliers(),
           "correspondences": lambda h: h.last_correspondences(), "features": lambda h: h.last_features(0)}


def getter_state(h):
    out = {}
    for k, g in GETTERS.items():
        got = g(h)
        out[k] = [np.asarray(a).tobytes() for a in (got if isinstance(got, tuple) else (got,))]
    return out


def soil_for_getters(h, soil, p):
    if soil == "voxelize":
        h.voxelize(lattice(51, 900), 0.5)
    elif soil == "two_pairs":
        h.register_batch([(lattice(52, 700), moved(lattice(52, 700)))] * 2, p)
    else:
        SOILS[soil](h)


def refused(call, label):
    """True when call() refuses with QB200_ERR_BAD_ARG and the reuse message; what it handed out otherwise"""
    try:
        got = call()
    except QuatroB200Error as e:
        assert e.code == -1 and "reused" in str(e), (label, str(e))
        return True
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("soil", [s for s in SOILS if s != "single"] + ["voxelize", "two_pairs"])
def test_getters_refuse_once_a_later_wave_reused_slot_0(handle_a, soil):
    p = make_params(**FRONT)
    rng = np.random.default_rng(1)
    a, b = lattice(50, 300), lattice(51, 300)
    handle_a.match(a, fpfh_like(rng, 300), b, fpfh_like(rng, 300), p)
    want_nn = [t.tobytes() for t in handle_a.debug_nn_tables(300, 300)]
    soil_for_getters(handle_a, soil, p)
    stale = {}
    got = refused(lambda: handle_a.debug_nn_tables(300, 300), "nn_tables")
    if got is not True:
        stale["nn_tables"] = [t.tobytes() for t in got] == want_nn

    src, tgt = lattice(50, 600), moved(lattice(50, 600))
    res, _ = handle_a.register_pair(src, tgt, p)
    assert res.clique_size > 1 and res.n_final_inliers > 1
    want = getter_state(handle_a)
    soil_for_getters(handle_a, soil, p)
    for name, g in GETTERS.items():
        got = refused(lambda: g(handle_a), name)
        if got is not True:
            got = [np.asarray(x).tobytes() for x in (got if isinstance(got, tuple) else (got,))]
            stale[name] = got == want[name]
    assert not stale, f"getters handed out slot 0 after a later wave (True: the entries still equal the call's own): {stale}"
    # the next single-pair call makes them hand out its lists again
    handle_a.register_pair(src, tgt, p)
    assert getter_state(handle_a) == want


# Every single-pair call that sets some of the lists, after a batch rewrote slot 0: the lists it produced are its own, and every
# other getter refuses (that call's wave reused the buffers the older lists were in)
PARTIAL = {"compute_fpfh": {"features"}, "match": {"correspondences", "nn_tables"}, "match_and_pack": {"correspondences", "features"},
           "max_clique": {"clique"}, "solve_pose": {"clique", "final_inliers"}, "build_graph": set(), "voxelize": set()}


def partial_call(h, name):
    """run the single-pair call `name`; returns what its own outputs say each list it sets must hold (None: not checked here)"""
    p = make_params(**FRONT)
    src, tgt = lattice(80, 500), moved(lattice(80, 500))
    rng = np.random.default_rng(3)
    if name == "compute_fpfh":
        nrm, desc = h.compute_fpfh(src, p.normal_radius, p.fpfh_radius, p.fpfh_radius * 1.001953125)
        return {"features": [nrm.tobytes(), desc.tobytes()]}
    if name == "match":
        corr, _, _ = h.match(src, fpfh_like(rng, 500), tgt, fpfh_like(rng, 500), p)
        return {"correspondences": corr.tobytes(), "nn_tables": None}
    if name == "match_and_pack":
        corr, sm, tm, _ = h.match_and_pack(src, tgt, p)
        return {"correspondences": [corr.tobytes(), sm.tobytes(), tm.tobytes()], "features": None}
    if name == "max_clique":
        clique, _, _, _ = h.max_clique(complete_rows(40), PMC_HEU)
        return {"clique": clique.tobytes()}
    if name == "solve_pose":
        a, b = PROBE_SETS[-1]
        ids = np.arange(20)[::-1].astype(np.int32)
        res, _, _, _ = h.solve_pose(a, b, ids, make_params())
        return {"clique": ids.tobytes(), "final_inliers": res.n_final_inliers}
    if name == "build_graph":
        h.build_graph(*PROBE_SETS[-1], 0.3, 1.0)
    else:
        h.voxelize(lattice(81, 300), 0.5)
    return {}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PARTIAL))
def test_a_partial_single_pair_call_sets_only_its_own_lists(handle_a, name):
    p = make_params(**FRONT)
    handle_a.register_pair(lattice(50, 600), moved(lattice(50, 600)), p)
    # slot 0's clique, final inliers, masks, correspondences and matched points rewritten by batches of two
    handle_a.max_clique_batch_each([complete_rows(30)] * 2, [make_params()] * 2)
    handle_a.solve_pose_batch_each(PROBE_SETS[-2:], [np.arange(60)] * 2, [make_params()] * 2)
    handle_a.solve_batch_each(PROBE_SETS[-2:], [make_params()] * 2)
    handle_a.register_batch([(lattice(52, 300), moved(lattice(52, 300)))] * 2, p)
    own = partial_call(handle_a, name)
    assert set(own) == PARTIAL[name]
    calls = dict(GETTERS, nn_tables=lambda h: h.debug_nn_tables(500, 500))
    for getter, g in calls.items():
        got = refused(lambda: g(handle_a), getter)
        if getter not in own:
            assert got is True, (name, getter, "handed out a list this call did not produce")
            continue
        assert got is not True, (name, getter, "refused a list this call produced")
        want = own[getter]
        if isinstance(want, int):
            assert len(got) == want, (name, getter)
        elif want is not None:
            got = [np.asarray(x).tobytes() for x in got] if isinstance(want, list) else got[0].tobytes() if isinstance(got, tuple) \
                else np.asarray(got).tobytes()
            assert got == want, (name, getter)


# ---- GPU: a queued stream of soils and probes, one flush ------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_queued_stream_of_soils_and_probes_equals_a_fresh_handle(handle_a, reference, oracle):
    h, keep = handle_a, []
    n_sets, n_pose = len(PROBE_SETS), len(POSE_IDS)
    soil_arr, k1 = h._set_array(SOIL_SETS, MEM_HOST)
    soil_out = np.zeros(SLOTS, capi_result_dtype())
    gb = GraphBuffers(n_sets, ROWS, WPR, CAP_EDGES, fill=SENT32)
    g_arr, k2 = h._set_array(PROBE_SETS, MEM_HOST)
    g_out = np.zeros(n_sets, capi_result_dtype())
    full_arr, k3 = h.graph_array([complete_rows(LC)] * SLOTS)
    full_out = np.zeros(SLOTS, capi_result_dtype())
    sets, ids, params = pose_inputs()
    pose_arr, k4 = h.inlier_array(sets, ids, MEM_HOST)
    pose_out = np.zeros(n_pose, capi_result_dtype())
    pose_lb = sentinel_lists(ListBuffers(n_pose, LC, MEM_HOST, SET_LISTS))
    graphs, gparams, _ = probe_graphs(oracle)
    cl_arr, k5 = h.graph_array(graphs)
    cl_out = np.zeros(len(graphs), capi_result_dtype())
    cl_lb = sentinel_lists(ListBuffers(len(graphs), CAP_CLIQUE, MEM_HOST, GRAPH_LISTS))
    pa = [h.params_array(x) for x in ([make_params(inlier_selection_mode=INLIER_NONE)] * SLOTS, [make_params()] * n_sets,
                                      [make_params()] * SLOTS, params, gparams)]
    soil_lb = ListBuffers(SLOTS, LC, MEM_HOST, SET_LISTS)
    keep += [k1, k2, k3, k4, k5, pa]       # the host inputs and every output must live until the flush returns
    h.solve_batch_enqueue_each_raw(soil_arr, SLOTS, pa[0], MEM_HOST, soil_out, soil_lb)
    h.build_graph_batch_enqueue_each_raw(g_arr, n_sets, pa[1], MEM_HOST, g_out, gb)
    h.max_clique_batch_enqueue_each_raw(full_arr, SLOTS, pa[2], MEM_HOST, full_out)
    h.solve_pose_batch_enqueue_each_raw(pose_arr, n_pose, pa[3], MEM_HOST, pose_out, pose_lb)
    h.max_clique_batch_enqueue_each_raw(cl_arr, len(graphs), pa[4], MEM_HOST, cl_out, cl_lb)
    h.register_batch_flush()
    same_outputs({"records": g_out, **{k: gb.host(k) for k in ("adj", "degree", "edges")}},
                 {k: v for k, v in reference["graph"].items() if not k.endswith("_dev")}, "graph")
    same_outputs({"records": pose_out, **{k: pose_lb.host(k) for k in SET_LISTS}}, reference["pose"], "pose")
    same_outputs({"records": cl_out, "clique": cl_lb.host("clique")}, reference["clique"], "clique")


def capi_result_dtype():
    from quatro_b200.capi import RESULT_DTYPE
    return RESULT_DTYPE


# ---- GPU: a wide handle ------------------------------------------------------------------------------------------------------------
# max_voxel_points 18048 is above the 17920 points the block sort takes, so the lattice and norm sorts run the library radix sort
# through key_a / val_a; max_corr 16384 brings in pose_ws (cliques above 4096 members) and kcore_ws / chain_ws (graphs above 8192
# vertices).  The probes sit on both sides of those switches.
V_B, LC_B = 18048, 16384
CFG_B = dict(max_batch_slots=2, max_voxel_points=V_B, max_corr=LC_B)
WIDE_L = (4095, 4096, 4097, 8191, 8192, 8193)
WPR_B = (max(WIDE_L) + 31) // 32 + 2
WIDE_SETS = [corr_set(960 + i, L, 0.3) for i, L in enumerate(WIDE_L)]
SOIL_SETS_B = [corr_set(980 + i, LC_B, 0.9) for i in range(2)]
_WIDE_ROWS = {}


def wide_rows(oracle):
    """the oracle's TIM rows, degrees and edge counts of the wide sets at WPR_B words per row (computed once)"""
    if not _WIDE_ROWS:
        _WIDE_ROWS["rows"] = [tim_rows(oracle, a, b, make_params(), WPR_B) for a, b in WIDE_SETS]
    return _WIDE_ROWS["rows"]


def soil_b(h):
    h.max_clique_batch_each([complete_rows(LC_B)] * 2, [make_params()] * 2)
    h.solve_batch_each(SOIL_SETS_B, [make_params(inlier_selection_mode=INLIER_NONE)] * 2, buffers=ListBuffers(2, LC_B, MEM_HOST, SET_LISTS))
    h.build_graph_batch_each(SOIL_SETS_B, [make_params()] * 2, buffers=GraphBuffers(2, LC_B, LC_B // 32, 1, arrays=("adj", "degree")))
    h.solve_pose_batch_each(SOIL_SETS_B, [np.arange(LC_B)[::-1]] * 2, [make_params(using_rot_inliers_when_estimating_cote=1)] * 2)
    h.register_features_each([(*hostile_features(90, V_B), *hostile_features(91, V_B))] * 2, [make_params()] * 2)


def probe_wide_graph(h, oracle):
    out = {}
    for kind, tag in ((MEM_HOST, ""), (MEM_DEVICE, "_dev")):
        gb = GraphBuffers(len(WIDE_SETS), max(WIDE_L), WPR_B, 1, kind, ("adj", "degree"), h.cfg.device, fill=SENT32)
        out["records" + tag] = h.build_graph_batch_each(WIDE_SETS, [make_params()] * len(WIDE_SETS), buffers=gb)
        out.update({k + tag: gb.host(k).copy() for k in ("adj", "degree")})
    return out


def check_wide_graph(out, oracle):
    for tag in ("", "_dev"):
        for i, (L, (adj, deg, ne)) in enumerate(zip(WIDE_L, wide_rows(oracle))):
            r = out["records" + tag][i]
            assert (r["status"], r["n_corr"], r["n_edges"]) == (0, L, ne), (tag, L)
            assert out["adj" + tag][i, :L].tobytes() == adj.tobytes() and out["degree" + tag][i, :L].tobytes() == deg.tobytes(), (tag, L)
            assert (out["adj" + tag][i, L:] == SENT32).all(), (tag, L)


def probe_wide_clique(h, oracle):
    graphs = []
    for (adj, _, _), L in zip(wide_rows(oracle), WIDE_L):
        g = adj.copy()
        g[:, (L + 31) // 32:] = 0xFFFFFFFF      # columns >= L are ignored
        graphs.append(g)
    lb = sentinel_lists(ListBuffers(len(graphs), LC_B, MEM_HOST, GRAPH_LISTS))
    recs, _ = h.max_clique_batch_each(graphs, [make_params()] * len(graphs), buffers=lb)
    return {"records": recs, "clique": lb.host("clique").copy()}


def check_wide_clique(out, oracle):
    for i, ((adj, _, ne), L) in enumerate(zip(wide_rows(oracle), WIDE_L)):
        oc, _, _, omc, _ = oracle.max_clique_ex(adj, PMC_HEU)
        r = out["records"][i]
        assert (r["status"], r["n_corr"], r["n_edges"], r["clique_size"], r["max_core"]) == (0, L, ne, len(oc), omc), (L, r)
        assert out["clique"][i, :len(oc)].tobytes() == oc.astype(np.int32).tobytes(), L
        assert (out["clique"][i, len(oc):].view(np.uint32) == SENT32).all(), L


def probe_wide_pose(h, oracle):
    lb = sentinel_lists(ListBuffers(len(WIDE_SETS), LC_B, MEM_HOST, SET_LISTS))
    recs, _ = h.solve_pose_batch_each(WIDE_SETS, [np.arange(L)[::-1] for L in WIDE_L], [make_params()] * len(WIDE_L), buffers=lb)
    return {"records": recs, **{k: lb.host(k).copy() for k in SET_LISTS}}


def check_wide_pose(out, oracle):
    for i, ((a, b), L) in enumerate(zip(WIDE_SETS, WIDE_L)):
        r, ids = out["records"][i], np.arange(L)[::-1].astype(np.int32)
        nf = int(r["n_final_inliers"])
        _, orm, otm, _, ofin = oracle.solve_pose(a, b, ids, make_params(), want_final=True)
        assert int(r["clique_size"]) == L and out["clique"][i, :L].tobytes() == ids.tobytes(), L
        assert out["rot_inlier_mask"][i, :L].tobytes() == orm.tobytes() and out["trans_inlier_mask"][i, :L].tobytes() == otm.tobytes(), L
        assert out["final_inliers"][i, :nf].tobytes() == ofin.tobytes(), L
        check_lists_tail(out, i, {"clique": L, "rot_inlier_mask": L, "trans_inlier_mask": L, "final_inliers": nf})


PROBES_B = {"graph": (probe_wide_graph, check_wide_graph), "clique": (probe_wide_clique, check_wide_clique),
            "pose": (probe_wide_pose, check_wide_pose), "match": (lambda h, o: probe_match(h), check_match)}


@pytest.mark.gpu
def test_wide_handle_probes_after_wide_soils_equal_a_fresh_handle_and_the_oracle(oracle):
    want = {}
    for name, (run, _) in PROBES_B.items():
        with make_handle(1, **CFG_B) as h:
            want[name] = run(h, oracle)
    with make_handle(1, **CFG_B) as h:
        for name, (run, check) in PROBES_B.items():
            soil_b(h)
            got = run(h, oracle)
            same_outputs(got, want[name], ("wide", name))
            check(got, oracle)
