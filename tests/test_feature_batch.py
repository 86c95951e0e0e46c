"""Batches of caller keypoints and FPFH-33 descriptors: qb200_register_features_each and qb200_register_features_enqueue_each.
Features read back from the scan cache register byte-identically to the cached pairs; a pair's correspondences equal qb200_match's;
descriptors this library did not compute (the float64 PCL restatement, adversarial sets) give the oracle's correspondence list and
solve; a mixed wave equals its single-pair calls; a rejected call writes and queues nothing; and feature batches share one stream
with raw, cached and correspondence-set batches."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import (INLIER_NONE, KCORE_HEU, LIST_LAYOUT, MEM_DEVICE, MEM_HOST, PMC_EXACT, RESULT_DTYPE, SET_LISTS, FeaturePair,
                              ListBuffers, default_params)
from support import P4, ROOT, device_copies, fpfh_like, host_lists, make_handle, make_params, sentinel, sentinel_lists

NEW = ("qb200_register_features_each", "qb200_register_features_enqueue_each")


# ---- CPU: the POD, the header, the symbols -----------------------------------------------------------------------------------------
def test_feature_pair_mirror_matches_the_c_layout(tmp_path):
    """sizeof and every offsetof of qb200_feature_pair from a C compiler (the header compiles as C11), against the ctypes mirror."""
    body = f'  printf("size %zu\\n", sizeof(qb200_feature_pair));\n' + "".join(
        f'  printf("{f} %zu\\n", offsetof(qb200_feature_pair, {f}));\n' for f, _ in FeaturePair._fields_)
    (tmp_path / "pod.c").write_text('#include <stddef.h>\n#include <stdio.h>\n#include "quatro_b200.h"\nint main(void) {\n' + body +
                                    "  return 0;\n}\n")
    r = subprocess.run(["/usr/bin/gcc", "-std=c11", "-Wall", "-Werror", "-pedantic", f"-I{ROOT / 'include'}", str(tmp_path / "pod.c"), "-o",
                        str(tmp_path / "pod")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    probe = dict(ln.split() for ln in subprocess.run([str(tmp_path / "pod")], capture_output=True, text=True, check=True).stdout.splitlines())
    assert C.sizeof(FeaturePair) == int(probe["size"]) == 40
    for f, _ in FeaturePair._fields_:
        assert getattr(FeaturePair, f).offset == int(probe[f]), f


def test_library_exports_the_feature_calls():
    lib = capi.load_library()
    for n in NEW:
        assert n in capi.EXPORTED_SYMBOLS and hasattr(lib, n)
        assert getattr(lib, n).argtypes == lib.qb200_solve_batch_enqueue_each.argtypes
    assert lib.qb200_register_features_each(None, None, 0, None, MEM_HOST, None, None) == -1
    assert lib.qb200_register_features_enqueue_each(None, None, 0, None, MEM_HOST, None, None) == -1


# ---- configurations ----------------------------------------------------------------------------------------------------------------
SLOTS, N = 8, 20   # 20 pairs: three waves of up to 8 pairs
# matcher and solver fields vary; the front end is the default one, which the slots are cached with
PER_PAIR = [make_params(seed=11 + i % 3, use_tuple_test=int(i % 4 != 2), tuple_scale=0.9 if i % 5 == 1 else 0.95,
                        noise_bound=0.35 if i % 3 == 1 else 0.3,
                        inlier_selection_mode=(KCORE_HEU, INLIER_NONE, 1)[i % 3] if i % 7 else PMC_EXACT) for i in range(N)]


def _flat(recs, lb):
    return recs.tobytes(), [{k: v.tobytes() for k, v in d.items()} for d in host_lists(lb.trimmed(recs))]


def _device_pairs(feats):
    """(src, sdesc, tgt, tdesc) numpy tuples -> the MEM_DEVICE tuples of register_features_each, and the tensors behind them"""
    keep, out = [], []
    for s, sd, t, td in feats:
        _, ts = device_copies([s, sd, t, td])
        keep.append(ts)
        out.append((ts[0].data_ptr(), ts[1].data_ptr(), len(s), ts[2].data_ptr(), ts[3].data_ptr(), len(t)))
    return out, keep


def _untouched(out, lb):
    return (out.view(np.uint8) == 0xA5).all() and all((a.view(np.uint8) == 0xA5).all() for a in lb.arrays.values())


# ---- GPU fixtures ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def street():
    return [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(900, 900 + N)]


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


SLOT_PAIRS = [(2 * i, 2 * i + 1) for i in range(N)]


# ---- GPU 1: features read back from the cache register like the cached pairs ---------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 4])
def test_features_equal_the_cached_path(h1, h4, feats, lanes):
    h = h1 if lanes == 1 else h4
    lb = ListBuffers(N, h.cfg.max_corr, MEM_HOST)
    want = _flat(h.register_cached_mixed(SLOT_PAIRS, PER_PAIR, buffers=lb)[0], lb)
    recs = np.frombuffer(want[0], RESULT_DTYPE)
    assert (recs["status"] == 0).sum() >= N - 3 and len(set(recs["n_corr"])) > 5 and (recs["clique_size"] > 3).sum() >= N - 3
    dev, keep = _device_pairs(feats)
    for kind, pairs in ((MEM_HOST, feats), (MEM_DEVICE, dev)):
        for dest in (MEM_HOST, MEM_DEVICE):
            lb = ListBuffers(N, h.cfg.max_corr, dest, device=h.cfg.device)
            got = _flat(h.register_features_each(pairs, PER_PAIR, kind, buffers=lb)[0], lb)
            assert got == want, (kind, dest)
    ms = h.stage_ms()
    assert ms[0] > 0 and ms[1] == 0 and ms[2] == 0 and ms[3] > 0, ms   # the import under h2d; no voxel or FPFH stage


# ---- GPU 2: the correspondences of the single-pair matcher -----------------------------------------------------------------------------
@pytest.mark.gpu
def test_features_equal_the_single_pair_matcher(h4, feats):
    idx = [0, 3, 7, 12]
    lb = ListBuffers(len(idx), h4.cfg.max_corr, MEM_HOST, ("corr", "src_matched4", "tgt_matched4"))
    recs, lists = h4.register_features_each([feats[i] for i in idx], [PER_PAIR[i] for i in idx], buffers=lb)
    for k, i in enumerate(idx):
        s, sd, t, td = feats[i]
        corr, n_mutual, st = h4.match(s, sd, t, td, PER_PAIR[i], cap=h4.cfg.max_corr)
        assert st == 0 and len(corr) > 10
        assert np.array_equal(lists[k]["corr"], corr) and recs[k]["n_mutual"] == n_mutual, i
        assert (recs[k]["n_src_vox"], recs[k]["n_tgt_vox"]) == (len(s), len(t))
        assert np.array_equal(lists[k]["src_matched4"], s[corr[:, 0]]) and np.array_equal(lists[k]["tgt_matched4"], t[corr[:, 1]])


# ---- GPU 3: features this library did not compute, against the oracle --------------------------------------------------------------------
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


def _oracle_case(h, oracle, s, sd, t, td, p, label, solve=True):
    lb = ListBuffers(1, h.cfg.max_corr, MEM_HOST)
    recs, lists = h.register_features_each([(s, sd, t, td)], [p], buffers=lb)
    corr, n_mutual, _ = oracle.match(s, sd, t, td, p, cap=h.cfg.max_corr)
    assert np.array_equal(lists[0]["corr"], corr), f"{label}: correspondence list differs"
    assert recs[0]["n_mutual"] == n_mutual, label
    if solve:
        ref, st = oracle.solve_correspondences(s[corr[:, 0]], t[corr[:, 1]], p)
        for k in ("valid", "status", "n_corr", "n_edges", "max_core", "clique_size", "gnc_iters", "n_rot_inliers", "n_final_inliers"):
            assert recs[0][k] == getattr(ref, k), (label, k, recs[0][k], getattr(ref, k))
        assert np.allclose(np.asarray(recs[0]["T"]).reshape(4, 4).T, ref.matrix(), atol=1e-9, rtol=0), label
    return recs[0]


@pytest.mark.gpu
def test_independent_features_against_the_oracle(h4, oracle):
    for seed in (31, 32):
        s, sd, t, td = _independent_features(seed)
        rec = _oracle_case(h4, oracle, s, sd, t, td, make_params(), f"seed {seed}")
        assert rec["valid"] == 1 and rec["clique_size"] > 5


def _adversarial(rng):
    """(label, source descriptors, target descriptors): the matcher's hard cases"""
    A, B = fpfh_like(rng, 900), fpfh_like(rng, 700)
    same = np.repeat(fpfh_like(rng, 1), 3000, axis=0)
    zeros_a, zeros_b = A.copy(), B.copy()
    zeros_a[::3] = 0.0
    zeros_b[::4] = 0.0
    bad_a, bad_b = A.copy(), B.copy()
    bad_a[5, 3], bad_a[9, :] = np.nan, np.inf
    bad_a[11, 7], bad_b[2, 0], bad_b[17, 32] = -np.inf, np.nan, np.inf
    bad_b[30, :] = 3e38
    out = [("identical rows", np.concatenate([same, A[:100]]), np.concatenate([same[:2000], B[:50]])),
           ("all-zero rows", zeros_a, zeros_b), ("NaN and inf", bad_a, bad_b),
           ("src larger than tgt", A, B), ("src smaller than tgt", B, A)]
    for k in (-20, 8, 40):
        out.append((f"x 2^{k}", A * np.float32(2.0 ** k), B * np.float32(2.0 ** k)))
    return out


@pytest.mark.gpu
def test_adversarial_descriptors_give_the_oracle_list(h4, oracle):
    rng = np.random.default_rng(77)
    p = make_params(use_tuple_test=0)
    for label, A, B in _adversarial(rng):
        a4, b4 = P4(rng.uniform(-30, 30, (len(A), 3))), P4(rng.uniform(-30, 30, (len(B), 3)))
        _oracle_case(h4, oracle, a4, A, b4, B, p, label, solve=False)


# ---- GPU 4: one mixed wave equals its single-pair calls ------------------------------------------------------------------------------------
def _feature_pair(rng, ns, nt):
    """ns source keypoints and descriptors; the target holds the first min(ns, nt) of them moved and perturbed, then random ones"""
    src, desc = P4(rng.uniform(-20, 20, (ns, 3))), fpfh_like(rng, ns)
    m = min(ns, nt)
    c, s_ = np.cos(0.3), np.sin(0.3)
    R = np.array([[c, -s_, 0], [s_, c, 0], [0, 0, 1]])
    tgt_xyz = np.concatenate([src[:m, :3] @ R.T + [1.0, -2.0, 0.5] + rng.normal(0, 0.02, (m, 3)), rng.uniform(-20, 20, (nt - m, 3))])
    tdesc = np.concatenate([desc[:m] + rng.normal(0, 0.5, (m, 33)).astype(np.float32), fpfh_like(rng, nt - m)])
    tgt = P4(tgt_xyz, w=0.5)     # w is handed back in the matched points
    return src, desc, tgt, tdesc.astype(np.float32)


@pytest.mark.gpu
def test_a_mixed_wave_equals_its_single_pair_calls():
    V = 2048
    sizes = [(0, 40), (40, 0), (1, 1), (2, 2), (63, 64), (64, 65), (65, 63), (127, 128), (128, 129), (129, 127), (V, V), (300, V)]
    rng = np.random.default_rng(5)
    pairs = [_feature_pair(rng, ns, nt) for ns, nt in sizes]
    params = [make_params(use_tuple_test=i % 2, seed=100 + i, tuple_scale=(0.95, 0.9, 0.8)[i % 3],
                          inlier_selection_mode=(PMC_EXACT, INLIER_NONE, 1, KCORE_HEU)[i % 4]) for i in range(len(sizes))]
    with make_handle(4, max_batch_slots=16, max_voxel_points=V) as h:
        dev, keep = _device_pairs(pairs)
        single = []
        for pr, p in zip(pairs, params):
            lb = ListBuffers(1, h.cfg.max_corr, MEM_HOST)
            single.append(_flat(h.register_features_each([pr], [p], buffers=lb)[0], lb))
        recs = np.frombuffer(b"".join(s[0] for s in single), RESULT_DTYPE)
        assert (recs["status"][:2] == 2).all() and (recs["n_src_vox"] == [s for s, _ in sizes]).all()
        assert (recs["clique_size"] > 3).sum() >= 5
        for kind, ps in ((MEM_HOST, pairs), (MEM_DEVICE, dev)):
            lb = ListBuffers(len(pairs), h.cfg.max_corr, MEM_HOST)
            got = _flat(h.register_features_each(ps, params, kind, buffers=lb)[0], lb)
            for i in range(len(pairs)):
                assert got[0][i * RESULT_DTYPE.itemsize:(i + 1) * RESULT_DTYPE.itemsize] == single[i][0], (kind, sizes[i])
                assert got[1][i] == single[i][1][0], (kind, sizes[i])


# ---- GPU 5: refusals -------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_rejected_call_writes_and_queues_nothing(h4, feats):
    import torch
    lib, n = h4.lib, 2 * SLOTS + 1
    good, keep_good = h4.feature_array(feats[:n])
    good_params = h4.params_array(PER_PAIR[:n])
    want, _ = h4.register_features_each(feats[:n], PER_PAIR[:n])
    s, sd, t, td = feats[1]
    _, dev = device_copies([s, sd, t, td])
    raw = torch.zeros(4 * len(s) + 8, dtype=torch.float32, device="cuda")
    V = h4.cfg.max_voxel_points
    big = (np.zeros((V + 1, 4), np.float32), np.zeros((V + 1, 33), np.float32))

    def call(entries, kind=MEM_HOST, ps=None, n_=None):
        """entries: per pair (src, src_desc, n_src, tgt, tgt_desc, n_tgt) raw addresses"""
        arr = (FeaturePair * len(entries))()
        for i, e in enumerate(entries):
            arr[i].src, arr[i].src_desc, arr[i].n_src, arr[i].tgt, arr[i].tgt_desc, arr[i].n_tgt = e
        out, lb = sentinel(max(len(entries), 1), RESULT_DTYPE), sentinel_lists(ListBuffers(max(len(entries), 1), 64))
        st = lib.qb200_register_features_enqueue_each(h4.h, arr, len(entries) if n_ is None else n_, h4.params_array(ps or [PER_PAIR[0]] * 3),
                                                      kind, capi._ptr(out), C.byref(lb.descriptor()))
        return st, out, lb

    ok = (s.ctypes.data, sd.ctypes.data, len(s), t.ctypes.data, td.ctypes.data, len(t))
    okd = (dev[0].data_ptr(), dev[1].data_ptr(), len(s), dev[2].data_ptr(), dev[3].data_ptr(), len(t))
    cases = {
        "n < 0": (lambda: call([ok] * 3, n_=-1), -1, None),
        "n_src < 0": (lambda: call([ok, ok[:2] + (-1,) + ok[3:], ok]), -1, "feature pair 1"),
        "n_tgt > max_voxel_points": (lambda: call([ok, ok, ok[:3] + (big[0].ctypes.data, big[1].ctypes.data, V + 1)]), -1, "feature pair 2"),
        "null keypoints": (lambda: call([ok, (0,) + ok[1:], ok]), -1, "feature pair 1"),
        "null descriptors": (lambda: call([ok, ok[:4] + (0, len(t)), ok]), -1, "feature pair 1"),
        "host memory as device kind": (lambda: call([okd, ok, okd], MEM_DEVICE), -1, "feature pair 1"),
        "misaligned device keypoints": (lambda: call([okd, okd, (raw.data_ptr() + 4,) + okd[1:]], MEM_DEVICE), -1, "feature pair 2"),
        "misaligned device descriptors": (lambda: call([okd, okd[:4] + (dev[3].data_ptr() + 2, len(t)), okd], MEM_DEVICE), -1,
                                          "feature pair 1"),
        "bad params entry": (lambda: call([ok] * 3, ps=[PER_PAIR[0], make_params(noise_bound=-1.0), PER_PAIR[0]]), -1, "entry 1"),
        "crosscheck off": (lambda: call([ok] * 3, ps=[PER_PAIR[0], PER_PAIR[1], make_params(use_crosscheck=0)]), -4, "entry 2"),
    }
    for name, (fn, code, names) in cases.items():
        out1 = np.zeros(n, RESULT_DTYPE)
        assert lib.qb200_register_features_enqueue_each(h4.h, good, n, good_params, MEM_HOST, capi._ptr(out1), None) == 0
        st, out, lb = fn()
        err = lib.qb200_last_error(h4.h).decode()
        assert st == code, (name, st, err)
        if names:
            assert names in err, (name, err)
        h4.register_batch_flush()
        assert _untouched(out, lb), name
        assert out1.tobytes() == want.tobytes(), name


# ---- GPU 6: one stream of raw, cached, feature and set batches --------------------------------------------------------------------------
@pytest.mark.gpu
def test_one_stream_of_feature_raw_cached_and_set_batches(h4, street, feats):
    sets = [tuple(a[:L] for a in synth.matched_pairs(700 + i, L, inlier_ratio=0.35, noise=0.03)[:2]) for i, L in enumerate([40, 300, 1200] * 4)]
    fp = [make_params(seed=31 + i, noise_bound=0.45 if i % 4 == 1 else 0.3, rot_noise_bound=0.0 if i % 4 == 1 else 0.6) for i in range(N)]
    dev, keep = _device_pairs(feats)
    feat_host, keep_host = h4.feature_array(feats)
    feat_dev, _ = h4.feature_array(dev, MEM_DEVICE)
    pair_arr, keep_pairs = h4.pair_array(street)
    set_arr, keep_sets = h4._set_array(sets, MEM_HOST)
    slot_arr = capi._slot_array(SLOT_PAIRS)
    outs = [np.zeros(len(x), RESULT_DTYPE) for x in (feats, street, SLOT_PAIRS, sets, feats)]
    bufs = [ListBuffers(N, h4.cfg.max_corr, MEM_HOST), ListBuffers(N, h4.cfg.max_corr, MEM_HOST),
            ListBuffers(N, h4.cfg.max_corr, MEM_DEVICE, device=h4.cfg.device), ListBuffers(len(sets), h4.cfg.max_corr, MEM_HOST, SET_LISTS),
            ListBuffers(N, h4.cfg.max_corr, MEM_DEVICE, device=h4.cfg.device)]
    pas = [h4.params_array(ps) for ps in (fp, PER_PAIR, PER_PAIR, [make_params()] * len(sets), fp)]
    h4.register_features_enqueue_each_raw(feat_host, N, pas[0], MEM_HOST, outs[0], bufs[0])
    h4.register_batch_enqueue_mixed_raw(pair_arr, N, pas[1], MEM_HOST, outs[1], bufs[1])
    h4.register_cached_enqueue_mixed_raw(slot_arr, N, pas[2], outs[2], bufs[2])
    h4.solve_batch_enqueue_each_raw(set_arr, len(sets), pas[3], MEM_HOST, outs[3], bufs[3])
    h4.register_features_enqueue_each_raw(feat_dev, N, pas[4], MEM_DEVICE, outs[4], bufs[4])
    h4.register_batch_flush()
    got = [_flat(o, b) for o, b in zip(outs, bufs)]
    # the blocking calls, every zero rotation noise bound replaced by the latch of the first one enqueued (every other entry of this
    # module is explicit, so the handle latches here)
    latched = [capi.Params.from_buffer_copy(p) for p in fp]
    for q in latched:
        q.rot_noise_bound = q.rot_noise_bound or 2 * fp[1].noise_bound
    want = []
    for k, fn in enumerate((lambda lb: h4.register_features_each(feats, latched, MEM_HOST, buffers=lb),
                            lambda lb: h4.register_batch_mixed(street, PER_PAIR, buffers=lb),
                            lambda lb: h4.register_cached_mixed(SLOT_PAIRS, PER_PAIR, buffers=lb),
                            lambda lb: h4.solve_batch_each(sets, [make_params()] * len(sets), buffers=lb),
                            lambda lb: h4.register_features_each(dev, latched, MEM_DEVICE, buffers=lb))):
        lb = ListBuffers(len(outs[k]), h4.cfg.max_corr, MEM_HOST, SET_LISTS if k == 3 else tuple(LIST_LAYOUT))
        want.append(_flat(fn(lb)[0], lb))
    for k in range(5):
        assert got[k] == want[k], k
    assert got[0] == got[4]

