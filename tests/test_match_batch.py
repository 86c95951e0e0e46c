"""Batches of pairs matched and not solved: qb200_match_batch_mixed, qb200_match_cached_mixed, qb200_match_features_each and their
queued forms.  Every source gives the lists and matcher counters of its register call with the "not solved" record; feature and raw
pairs give the single-pair matchers' correspondences and the oracle's; match + qb200_solve_batch_each equals the fused register call
field for field; a mixed wave equals its single-pair calls; edge cases, rejections, one shared stream and the stage times."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import (INLIER_NONE, KCORE_HEU, LIST_LAYOUT, MATCH_LISTS, MEM_DEVICE, MEM_HOST, PMC_EXACT, RESULT_DTYPE, SET_LISTS,
                              FeaturePair, ListBuffers, default_params)
from support import P4, ROOT, device_copies, host_lists, make_handle, make_params, sentinel, sentinel_lists

# new call -> the register call whose arguments it takes
NEW = {"qb200_match_batch_mixed": "qb200_register_batch_mixed", "qb200_match_batch_enqueue_mixed": "qb200_register_batch_enqueue_mixed",
       "qb200_match_cached_mixed": "qb200_register_cached_mixed", "qb200_match_cached_enqueue_mixed": "qb200_register_cached_enqueue_mixed",
       "qb200_match_features_each": "qb200_register_features_each",
       "qb200_match_features_enqueue_each": "qb200_register_features_enqueue_each"}
MATCHER = ("status", "n_src_vox", "n_tgt_vox", "n_mutual", "n_corr")
UNSOLVED = ("valid", "max_core", "clique_size", "gnc_iters", "n_rot_inliers", "n_final_inliers", "n_edges", "cost")
SOLVER = ("valid", "max_core", "clique_size", "gnc_iters", "n_rot_inliers", "n_final_inliers", "n_edges", "cost", "T")
CLIQUE_TRUNCATED = 1


# ---- CPU: symbols, prototypes, null handle -------------------------------------------------------------------------------------------
def test_library_exports_the_match_calls():
    lib = capi.load_library()
    for n, reg in NEW.items():
        assert n in capi.EXPORTED_SYMBOLS and hasattr(lib, n)
        assert getattr(lib, n).argtypes == getattr(lib, reg).argtypes, n


def test_header_prototypes_agree_with_the_binding(tmp_path):
    """Each new prototype, compiled as C11, is the register counterpart's type; the binding has one argtype per parameter."""
    body = "".join(f"  __typeof__(&{reg}) p{i} = {n};\n  (void)p{i};\n" for i, (n, reg) in enumerate(NEW.items()))
    (tmp_path / "proto.c").write_text('#include "quatro_b200.h"\nint main(void) {\n' + body + "  return 0;\n}\n")
    r = subprocess.run(["/usr/bin/gcc", "-std=gnu11", "-Wall", "-Werror", "-Wincompatible-pointer-types", f"-I{ROOT / 'include'}",
                        "-c", str(tmp_path / "proto.c"), "-o", str(tmp_path / "proto.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    header = (ROOT / "include" / "quatro_b200.h").read_text()
    for n in NEW:
        decl = header[header.index(f"int {n}("):]
        decl = decl[:decl.index(");")]
        assert decl.count(",") + 1 == len(capi._SIGNATURES[n][1]), n


def test_a_null_handle_is_refused():
    lib = capi.load_library()
    for n in NEW:
        fn = getattr(lib, n)
        args = [None, None, 0, None] + ([MEM_HOST] if len(fn.argtypes) == 7 else []) + [None, None]
        assert fn(*args) == -1, n


# ---- configurations ----------------------------------------------------------------------------------------------------------------
SLOTS, N = 8, 20   # 20 pairs: three waves of up to 8 pairs
# matcher and solver fields vary; the front end is the default one, which the slots are cached with
PER_PAIR = [make_params(seed=11 + i % 3, use_tuple_test=int(i % 4 != 2), tuple_scale=0.9 if i % 5 == 1 else 0.95,
                        noise_bound=0.35 if i % 3 == 1 else 0.3,
                        inlier_selection_mode=(KCORE_HEU, INLIER_NONE, 1)[i % 3] if i % 7 else PMC_EXACT) for i in range(N)]
# raw pairs: the front end varies as well
RAW = [make_params(voxel_size=(0.3, 0.35, 0.4)[i % 3], normal_radius=(0.5, 0.6)[i % 2], fpfh_radius=(0.75, 0.9)[i % 2],
                   grid_cell=0.95 if i % 4 == 3 else 0.0, seed=40 + i, use_tuple_test=int(i % 3 != 1), tuple_scale=(0.95, 0.9)[i % 2])
       for i in range(N)]
SLOT_PAIRS = [(2 * i, 2 * i + 1) for i in range(N)]


def _device_pairs(pairs):
    """(src, tgt) numpy pairs -> the MEM_DEVICE tuples of the raw calls, and the tensors behind them"""
    keep, out = [], []
    for s, t in pairs:
        _, ts = device_copies([s, t])
        keep.append(ts)
        out.append((ts[0].data_ptr(), len(s), ts[1].data_ptr(), len(t)))
    return out, keep


def _device_feats(feats):
    keep, out = [], []
    for s, sd, t, td in feats:
        _, ts = device_copies([s, sd, t, td])
        keep.append(ts)
        out.append((ts[0].data_ptr(), ts[1].data_ptr(), len(s), ts[2].data_ptr(), ts[3].data_ptr(), len(t)))
    return out, keep


def _lists_bytes(recs, lb):
    return [{k: v.tobytes() for k, v in d.items()} for d in host_lists(lb.trimmed(recs))]


def expected_status(reg):
    """the match call's status of a pair whose register call gave record `reg`"""
    if reg["status"] in (3, -5) or reg["status"] < 0:
        return reg["status"]
    return 2 if reg["n_src_vox"] == 0 or reg["n_tgt_vox"] == 0 else 0


def assert_matches_register(got, reg, label=""):
    """match records `got` against register records `reg`: the matcher's part equal, the solver's part "not solved"."""
    assert len(got) == len(reg)
    for i, (g, r) in enumerate(zip(got, reg)):
        for k in MATCHER[1:]:
            assert g[k] == r[k], (label, i, k, g[k], r[k])
        assert g["status"] == expected_status(r), (label, i, g["status"], r["status"])
        assert g["flags"] == r["flags"] & ~CLIQUE_TRUNCATED, (label, i, g["flags"], r["flags"])
        for k in UNSOLVED:
            assert g[k] == 0, (label, i, k, g[k])
        assert np.array_equal(np.asarray(g["T"]), np.eye(4).reshape(-1)), (label, i)


def _untouched(out, lb):
    return (out.view(np.uint8) == 0xA5).all() and all((a.view(np.uint8) == 0xA5).all() for a in lb.arrays.values())


# ---- GPU fixtures ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def street():
    return [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(1300, 1300 + N)]


def _cached_handle(lanes, street):
    h = make_handle(lanes, max_batch_slots=SLOTS)
    h.cache_reserve(2 * N)
    h.cache_scans([s for pr in street for s in pr], list(range(2 * N)), default_params())
    return h


@pytest.fixture(scope="module")
def h4(street):
    h = _cached_handle(4, street)
    yield h
    h.close()


@pytest.fixture(scope="module")
def h1(street):
    h = _cached_handle(1, street)
    yield h
    h.close()


@pytest.fixture(scope="module")
def feats(h4):
    """every cached pair's (keypoints, descriptors) of both scans, read back from the slots"""
    out = []
    for i in range(N):
        (sv, _, sd), (tv, _, td) = h4.cache_read(2 * i), h4.cache_read(2 * i + 1)
        out.append((sv, sd, tv, td))
    return out


# ---- GPU 1: every source against its register call -----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 4])
def test_three_sources_equal_their_register_calls(h1, h4, street, feats, lanes):
    h = h1 if lanes == 1 else h4
    dev_raw, keep_raw = _device_pairs(street)
    dev_feat, keep_feat = _device_feats(feats)
    sources = {
        "raw": (lambda lb: h.register_batch_mixed(street, RAW, buffers=lb),
                [(f"raw {k}", lambda lb, ps=ps, k=k: h.match_batch_mixed(ps, RAW, k, buffers=lb)) for k, ps in ((MEM_HOST, street),
                                                                                                                (MEM_DEVICE, dev_raw))]),
        "cached": (lambda lb: h.register_cached_mixed(SLOT_PAIRS, PER_PAIR, buffers=lb),
                   [("cached", lambda lb: h.match_cached_mixed(SLOT_PAIRS, PER_PAIR, buffers=lb))]),
        "features": (lambda lb: h.register_features_each(feats, PER_PAIR, buffers=lb),
                     [(f"features {k}", lambda lb, ps=ps, k=k: h.match_features_each(ps, PER_PAIR, k, buffers=lb))
                      for k, ps in ((MEM_HOST, feats), (MEM_DEVICE, dev_feat))]),
    }
    for name, (register, calls) in sources.items():
        lb = ListBuffers(N, h.cfg.max_corr, MEM_HOST, MATCH_LISTS)
        reg = register(lb)[0]
        want = _lists_bytes(reg, lb)
        assert (reg["status"] == 0).sum() >= N - 3 and len(set(reg["n_corr"])) > 5, name
        for label, fn in calls:
            for dest in (MEM_HOST, MEM_DEVICE):
                lb = ListBuffers(N, h.cfg.max_corr, dest, MATCH_LISTS, device=h.cfg.device)
                got = fn(lb)[0]
                assert_matches_register(got, reg, (label, dest))
                assert _lists_bytes(got, lb) == want, (label, dest)


# ---- GPU 2: the per-pair matchers ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_pairs_equal_the_per_pair_matchers(h4, street, feats):
    idx = [0, 3, 7, 12]
    lb = ListBuffers(len(idx), h4.cfg.max_corr, MEM_HOST, MATCH_LISTS)
    recs, lists = h4.match_features_each([feats[i] for i in idx], [PER_PAIR[i] for i in idx], buffers=lb)
    for k, i in enumerate(idx):
        s, sd, t, td = feats[i]
        corr, n_mutual, st = h4.match(s, sd, t, td, PER_PAIR[i], cap=h4.cfg.max_corr)
        assert st == 0 and len(corr) > 10
        assert np.array_equal(lists[k]["corr"], corr) and recs[k]["n_mutual"] == n_mutual, i
    lb = ListBuffers(len(idx), h4.cfg.max_corr, MEM_HOST, MATCH_LISTS)
    recs, lists = h4.match_batch_mixed([street[i] for i in idx], [RAW[i] for i in idx], buffers=lb)
    for k, i in enumerate(idx):   # qb200_match_and_pack takes voxelized clouds
        vs, vt = (h4.voxelize(c, RAW[i].voxel_size, RAW[i].skip_flagged)[0] for c in street[i])
        corr, sm, tm, st = h4.match_and_pack(vs, vt, RAW[i], cap=h4.cfg.max_corr)
        assert st == 0 and len(corr) > 10 and recs[k]["status"] == 0
        assert np.array_equal(lists[k]["corr"], corr), i
        assert lists[k]["src_matched4"].tobytes() == sm.tobytes() and lists[k]["tgt_matched4"].tobytes() == tm.tobytes(), i


# ---- GPU 3: the CPU oracle -----------------------------------------------------------------------------------------------------------
def _independent_features(seed):
    """voxel points of a street pair with float64 PCL normals and FPFH (tests/independent_ref.py), cast to float32"""
    from independent_ref import fpfh_pcl, normals_pcl, voxel_grid
    p = default_params()
    out = []
    for cloud in synth.outdoor_pair(seed, rings=16, azimuths=600)[:2]:
        pts = voxel_grid(cloud[:, :3].astype(np.float64), p.voxel_size)[0]
        nrm, _ = normals_pcl(pts, p.normal_radius)
        desc, _ = fpfh_pcl(pts, nrm, p.fpfh_radius)
        out += [P4(pts), desc.astype(np.float32)]
    return tuple(out)


@pytest.mark.gpu
def test_raw_and_independent_pairs_give_the_oracle_list(h4, oracle):
    for seed in (41, 42):
        s, sd, t, td = _independent_features(seed)
        p = make_params(seed=seed)
        lb = ListBuffers(1, h4.cfg.max_corr, MEM_HOST, MATCH_LISTS)
        recs, lists = h4.match_features_each([(s, sd, t, td)], [p], buffers=lb)
        corr, n_mutual, _ = oracle.match(s, sd, t, td, p, cap=h4.cfg.max_corr)
        assert len(corr) > 10 and np.array_equal(lists[0]["corr"], corr) and recs[0]["n_mutual"] == n_mutual, seed
    src, tgt = synth.outdoor_pair(43, rings=32, azimuths=900)[:2]
    p = make_params()
    lb = ListBuffers(1, h4.cfg.max_corr, MEM_HOST, MATCH_LISTS)
    recs, lists = h4.match_batch_mixed([(src, tgt)], [p], buffers=lb)
    vs, vt = (oracle.voxelize(c, p.voxel_size, p.skip_flagged)[0] for c in (src, tgt))
    corr, sm, tm, st = oracle.match_and_pack(vs, vt, p, cap=h4.cfg.max_corr)
    ref, _ = oracle.register_pair(src, tgt, p)
    assert len(corr) > 10 and np.array_equal(lists[0]["corr"], corr)
    assert lists[0]["src_matched4"].tobytes() == sm.tobytes() and lists[0]["tgt_matched4"].tobytes() == tm.tobytes()
    assert (recs[0]["n_mutual"], recs[0]["n_corr"], recs[0]["n_src_vox"], recs[0]["n_tgt_vox"]) == \
           (ref.n_mutual, ref.n_corr, ref.n_src_vox, ref.n_tgt_vox)


# ---- GPU 4: match, then solve the device lists, equals the fused register call ------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("source", ["raw", "features"])
def test_match_then_solve_equals_register(street, feats, source):
    # rot_noise_bound = 0 everywhere: the latch of the first pair decides, and the match call must not take it
    params = [make_params(rot_noise_bound=0.0, noise_bound=(0.3, 0.4, 0.25)[i % 3], seed=60 + i, use_tuple_test=int(i % 4 != 1),
                          inlier_selection_mode=(PMC_EXACT, PMC_EXACT, KCORE_HEU, INLIER_NONE, 1)[i % 5],
                          using_rot_inliers_when_estimating_cote=i % 2, cote_mode=i % 3 == 2) for i in range(N)]
    inputs = street if source == "raw" else feats
    with make_handle(4, max_batch_slots=SLOTS) as hm:
        cap = hm.cfg.max_corr
        lb = ListBuffers(N, cap, MEM_DEVICE, MATCH_LISTS, device=hm.cfg.device)
        m = (hm.match_batch_mixed if source == "raw" else hm.match_features_each)(inputs, params, buffers=lb)[0]
        assert (m["status"] == 0).sum() >= N - 3
        sm, tm = lb.arrays["src_matched4"], lb.arrays["tgt_matched4"]
        sets = [(sm.data_ptr() + i * cap * 16, tm.data_ptr() + i * cap * 16, int(m["n_corr"][i])) for i in range(N)]
        slb = ListBuffers(N, cap, MEM_HOST, SET_LISTS)
        solved, solved_lists = hm.solve_batch_each(sets, params, MEM_DEVICE, buffers=slb)
    with make_handle(4, max_batch_slots=SLOTS) as hr:
        rlb = ListBuffers(N, cap, MEM_HOST, tuple(LIST_LAYOUT))
        reg, reg_lists = (hr.register_batch_mixed if source == "raw" else hr.register_features_each)(inputs, params, buffers=rlb)
    assert (reg["valid"] == 1).sum() >= N - 3
    for i in range(N):
        assert m["n_corr"][i] == reg["n_corr"][i], i
        for k in SOLVER:
            assert np.asarray(solved[k][i]).tobytes() == np.asarray(reg[k][i]).tobytes(), (source, i, k, solved[k][i], reg[k][i])
        assert solved["flags"][i] & CLIQUE_TRUNCATED == reg["flags"][i] & CLIQUE_TRUNCATED, i
        if reg["status"][i] in (0, 1, 2):
            assert solved["status"][i] == reg["status"][i], i
        for k in SET_LISTS:
            assert solved_lists[i][k].tobytes() == reg_lists[i][k].tobytes(), (source, i, k)


# ---- GPU 5: one mixed wave equals its single-pair calls ------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_mixed_wave_equals_its_single_pair_calls(street):
    pairs = street[:12]
    params = [make_params(voxel_size=(0.3, 0.45, 0.25, 0.5)[i % 4], normal_radius=(0.5, 0.7, 0.45)[i % 3],
                          fpfh_radius=(0.75, 1.0, 0.8)[i % 3], use_tuple_test=i % 2, tuple_scale=(0.95, 0.9, 0.8)[i % 3],
                          tuple_trials_per_corr=(100, 30)[i % 2], seed=100 + i, noise_bound=float("nan") if i == 5 else 0.3)
              for i in range(len(pairs))]
    with make_handle(4, max_batch_slots=5) as h:
        single = []
        for pr, p in zip(pairs, params):
            lb = ListBuffers(1, h.cfg.max_corr, MEM_HOST, MATCH_LISTS)
            recs = h.match_batch_mixed([pr], [p], buffers=lb)[0]
            single.append((recs.tobytes(), _lists_bytes(recs, lb)[0]))
        recs = np.frombuffer(b"".join(s[0] for s in single), RESULT_DTYPE)
        assert len(set(recs["n_src_vox"])) > 6 and (recs["n_corr"] > 10).sum() >= 10
        lb = ListBuffers(len(pairs), h.cfg.max_corr, MEM_HOST, MATCH_LISTS)
        got = h.match_batch_mixed(pairs, params, buffers=lb)[0]
        lists = _lists_bytes(got, lb)
        for i in range(len(pairs)):
            assert got[i].tobytes() == single[i][0] and lists[i] == single[i][1], i


# ---- GPU 6: edge cases ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_edge_cases(h4, street, feats):
    s, sd, t, td = feats[0]
    empty = (np.zeros((0, 4), np.float32), np.zeros((0, 33), np.float32))
    fp = [(*empty, t, td), (s, sd, *empty), (s, sd, t, td), (s[:1], sd[:1], t[:1], td[:1])]
    out, lb = sentinel(max(len(fp), 1), RESULT_DTYPE), sentinel_lists(ListBuffers(max(len(fp), 1), h4.cfg.max_corr, MEM_HOST, MATCH_LISTS))
    arr, keep = h4.feature_array(fp)
    assert h4.lib.qb200_match_features_each(h4.h, arr, len(fp), h4.params_array([PER_PAIR[0]] * len(fp)), MEM_HOST, capi._ptr(out),
                                            C.byref(lb.descriptor())) == 0
    assert list(out["status"]) == [2, 2, 0, 0] and list(out["n_corr"][:2]) == [0, 0] and out["n_corr"][3] <= 1
    for i in (0, 1):   # an empty side writes no entry
        assert all((a[i].view(np.uint8) == 0xA5).all() for a in lb.arrays.values()), i
    raw = [(street[0][0], np.zeros((0, 4), np.float32)), street[0]]
    recs = h4.match_batch_mixed(raw, [RAW[0]] * 2)[0]
    assert list(recs["status"]) == [2, 0] and recs["n_tgt_vox"][0] == 0
    # a cap below n_corr: the first cap entries and the flag
    full_lb = ListBuffers(1, h4.cfg.max_corr, MEM_HOST, MATCH_LISTS)
    full, full_lists = h4.match_features_each([feats[2]], [PER_PAIR[2]], buffers=full_lb)
    cap = int(full["n_corr"][0]) // 2
    small_lb = ListBuffers(1, cap, MEM_HOST, MATCH_LISTS)
    small, small_lists = h4.match_features_each([feats[2]], [PER_PAIR[2]], buffers=small_lb)
    assert full["flags"][0] == 0 and small["flags"][0] == capi.FLAG_LISTS_TRUNCATED and small["n_corr"][0] == full["n_corr"][0]
    for k in MATCH_LISTS:
        assert small_lists[0][k].tobytes() == full_lists[0][k][:cap].tobytes(), k
    # lists == NULL: records only, equal to the records of the call with lists
    bare = h4.match_features_each([feats[2]], [PER_PAIR[2]])[0]
    assert bare.tobytes() == full.tobytes()
    # more correspondences than max_corr
    with make_handle(1, max_batch_slots=2, max_corr=32) as hs:
        lb = ListBuffers(2, 32, MEM_HOST, MATCH_LISTS)
        out, lists = hs.match_features_each([feats[2], (s[:20], sd[:20], t[:20], td[:20])], [PER_PAIR[2]] * 2, buffers=lb)
        assert out["status"][0] == 3 and all(len(v) == 0 for v in lists[0].values())
        assert out["status"][1] == 0 and out["n_corr"][1] <= 20


# ---- GPU 7: rejections -------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_rejected_call_writes_and_queues_nothing(h4, street, feats):
    import torch
    lib, n = h4.lib, 2 * SLOTS + 1
    good, keep_good = h4.feature_array(feats[:n])
    good_params = h4.params_array(PER_PAIR[:n])
    want, _ = h4.match_features_each(feats[:n], PER_PAIR[:n])
    pair_arr, keep_pairs = h4.pair_array(street[:3])
    feat_arr, keep_feats = h4.feature_array(feats[:3])
    s, sd, t, td = feats[1]
    _, dev = device_copies([s, sd, t, td])
    raw = torch.zeros(64, dtype=torch.float32, device="cuda")

    host_buf = np.zeros(64 * 3 * 16, np.uint8)

    def lists_with(name, kind=MEM_HOST, addr=None):
        """a list descriptor with one array, `name`, at addr (default: host memory)"""
        d = capi.PairLists(64, kind)
        setattr(d, name, addr if addr is not None else host_buf.ctypes.data)
        return d

    def call(fn_name, arr, ps=None, kind=MEM_HOST, lists=None):
        out, lb = sentinel(3, RESULT_DTYPE), sentinel_lists(ListBuffers(3, 64, MEM_HOST, MATCH_LISTS))
        d = lists if lists is not None else lb.descriptor()
        args = [h4.h, arr, 3, h4.params_array(ps or PER_PAIR[:3])] + ([kind] if fn_name != "qb200_match_cached_enqueue_mixed" else [])
        st = getattr(lib, fn_name)(*args, capi._ptr(out), C.byref(d))
        return st, out, lb

    fe, ra, ca = "qb200_match_features_enqueue_each", "qb200_match_batch_enqueue_mixed", "qb200_match_cached_enqueue_mixed"
    slots_ok = capi._slot_array(SLOT_PAIRS[:3])
    slots_bad = capi._slot_array([(0, 1), (2, 3), (4, 2 * N)])
    dev_bad = (FeaturePair * 3)()
    for i, e in enumerate([(dev[0].data_ptr(), dev[1].data_ptr(), len(s), dev[2].data_ptr(), dev[3].data_ptr(), len(t))] * 2 +
                          [(raw.data_ptr() + 4, dev[1].data_ptr(), 1, dev[2].data_ptr(), dev[3].data_ptr(), len(t))]):
        dev_bad[i].src, dev_bad[i].src_desc, dev_bad[i].n_src, dev_bad[i].tgt, dev_bad[i].tgt_desc, dev_bad[i].n_tgt = e
    cases = {}
    for name in ("clique", "final_inliers", "rot_inlier_mask", "trans_inlier_mask"):
        cases[f"{name} array"] = (lambda name=name: call(fe, feat_arr, lists=lists_with(name)), -1, "solves nothing")
    cases.update({
        "bad voxel_size": (lambda: call(ra, pair_arr, ps=[RAW[0], make_params(voxel_size=-1.0), RAW[0]]), -1, "entry 1"),
        "bad radii": (lambda: call(ra, pair_arr, ps=[RAW[0], RAW[1], make_params(normal_radius=2.0)]), -1, "entry 2"),
        "bad tuple trials": (lambda: call(fe, feat_arr, ps=[PER_PAIR[0], make_params(tuple_trials_per_corr=-1), PER_PAIR[0]]), -1, "entry 1"),
        "crosscheck off": (lambda: call(fe, feat_arr, ps=[PER_PAIR[0], PER_PAIR[1], make_params(use_crosscheck=0)]), -4, "entry 2"),
        "host memory as device features": (lambda: call(fe, feat_arr, kind=MEM_DEVICE), -1, "feature pair 0"),
        "misaligned device keypoints": (lambda: call(fe, dev_bad, kind=MEM_DEVICE), -1, "feature pair 2"),
        "foreign device list": (lambda: call(fe, feat_arr, lists=lists_with("corr", MEM_DEVICE)), -1, "device list array"),
        "misaligned device list": (lambda: call(fe, feat_arr, lists=lists_with("src_matched4", MEM_DEVICE, raw.data_ptr() + 4)), -1,
                                   "device list array"),
        "slot outside the cache": (lambda: call(ca, capi._ptr(slots_bad)), -1, "slot outside"),
        "slot signature": (lambda: call(ca, capi._ptr(slots_ok), ps=[PER_PAIR[0], make_params(voxel_size=0.35), PER_PAIR[0]]), -1,
                           "pair 1"),
    })
    for name, (fn, code, names) in cases.items():
        out1 = np.zeros(n, RESULT_DTYPE)
        assert lib.qb200_match_features_enqueue_each(h4.h, good, n, good_params, MEM_HOST, capi._ptr(out1), None) == 0
        st, out, lb = fn()
        err = lib.qb200_last_error(h4.h).decode()
        assert st == code, (name, st, err)
        if names:
            assert names in err, (name, err)
        h4.register_batch_flush()
        assert _untouched(out, lb), name
        assert out1.tobytes() == want.tobytes(), name
    # a NaN solver field is neither checked nor read
    nan = [make_params(noise_bound=float("nan"), cbar2=float("nan"), cote_noise_bound=-1.0, inlier_selection_mode=9,
                       rotation_max_iterations=-3, cote_mode=7, max_clique_node_limit=-1) for _ in range(3)]
    for q, p in zip(nan, PER_PAIR[:3]):
        q.seed, q.use_tuple_test, q.tuple_scale = p.seed, p.use_tuple_test, p.tuple_scale
    assert h4.match_features_each(feats[:3], nan)[0].tobytes() == want[:3].tobytes()


# ---- GPU 8: one stream of raw, cache-write, cached, feature and set batches ---------------------------------------------------------------
@pytest.mark.gpu
def test_one_stream_of_match_and_register_batches(street, feats):
    sets = [tuple(a[:L] for a in synth.matched_pairs(800 + i, L, inlier_ratio=0.35, noise=0.03)[:2]) for i, L in enumerate([40, 300, 900] * 3)]
    new_scan = synth.outdoor_pair(1999, rings=32, azimuths=900)[0]
    with make_handle(4, max_batch_slots=SLOTS) as h:
        h.cache_reserve(2 * N)
        h.cache_scans([s for pr in street for s in pr], list(range(2 * N)), default_params())
        before = h.match_cached_mixed(SLOT_PAIRS, PER_PAIR)[0]
        pair_arr, keep_pairs = h.pair_array(street)
        feat_arr, keep_feats = h.feature_array(feats)
        set_arr, keep_sets = h._set_array(sets, MEM_HOST)
        slot_arr = capi._slot_array(SLOT_PAIRS)
        scan_ptrs, counts, keep_scan = capi._scan_arrays([new_scan], MEM_HOST)
        slot_ids = (C.c_int32 * 1)(0)
        outs = [np.zeros(len(x), RESULT_DTYPE) for x in (street, SLOT_PAIRS, feats, sets)]
        bufs = [ListBuffers(N, h.cfg.max_corr, MEM_HOST, MATCH_LISTS), ListBuffers(N, h.cfg.max_corr, MEM_DEVICE, MATCH_LISTS, device=h.cfg.device),
                ListBuffers(N, h.cfg.max_corr, MEM_HOST, MATCH_LISTS), ListBuffers(len(sets), h.cfg.max_corr, MEM_HOST, SET_LISTS)]
        pas = [h.params_array(ps) for ps in (RAW, PER_PAIR, PER_PAIR, [make_params()] * len(sets), [default_params()])]
        h.match_batch_enqueue_mixed_raw(pair_arr, N, pas[0], MEM_HOST, outs[0], bufs[0])
        h.cache_scans_enqueue_each_raw(scan_ptrs, counts, slot_ids, 1, pas[4], MEM_HOST)
        h.match_cached_enqueue_mixed_raw(slot_arr, N, pas[1], outs[1], bufs[1])
        h.match_features_enqueue_each_raw(feat_arr, N, pas[2], MEM_HOST, outs[2], bufs[2])
        h.solve_batch_enqueue_each_raw(set_arr, len(sets), pas[3], MEM_HOST, outs[3], bufs[3])
        h.register_batch_flush()
        got = [(o.tobytes(), _lists_bytes(o, b)) for o, b in zip(outs, bufs)]
        want = []
        for k, fn in enumerate((lambda lb: h.match_batch_mixed(street, RAW, buffers=lb),
                                lambda lb: h.match_cached_mixed(SLOT_PAIRS, PER_PAIR, buffers=lb),
                                lambda lb: h.match_features_each(feats, PER_PAIR, buffers=lb),
                                lambda lb: h.solve_batch_each(sets, [make_params()] * len(sets), buffers=lb))):
            lb = ListBuffers(len(outs[k]), h.cfg.max_corr, MEM_HOST, SET_LISTS if k == 3 else MATCH_LISTS)
            recs = fn(lb)[0]
            want.append((recs.tobytes(), _lists_bytes(recs, lb)))
        for k in range(4):
            assert got[k] == want[k], k
        # the cached match saw the new scan in slot 0, and only pair 0 reads it
        assert outs[1][0]["n_src_vox"] != before[0]["n_src_vox"] and outs[1][1:].tobytes() == before[1:].tobytes()


# ---- GPU 9: stage times -------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_stage_times_of_a_match_call(h4, street, feats):
    h4.match_batch_mixed(street, RAW)
    ms = h4.stage_ms()
    assert ms[0] > 0 and ms[1] > 0 and ms[2] > 0 and ms[3] > 0 and ms[7] > 0, ms
    assert ms[4] == 0 and ms[5] == 0 and ms[6] == 0, ms
    h4.match_features_each(feats, PER_PAIR)
    ms = h4.stage_ms()
    assert ms[0] > 0 and ms[3] > 0 and ms[1] == ms[2] == ms[4] == ms[5] == ms[6] == 0, ms
    h4.match_cached_mixed(SLOT_PAIRS, PER_PAIR)
    ms = h4.stage_ms()
    assert ms[3] > 0 and ms[0] == ms[1] == ms[4] == ms[5] == ms[6] == 0, ms
