"""FPFH of caller keypoint clouds in batches: qb200_describe_points_each and qb200_describe_points_enqueue_each.
Every cloud's normals and FPFH-33 rows are byte-identical to qb200_compute_fpfh on that cloud alone with the resolved radii and cell,
for host and device clouds and outputs on one lane and on four, on a handle whose lattice sort takes the library path; a subset
equals the oracle; the voxel keypoints of qb200_describe_batch_each described again reproduce its features; described keypoints
register like per-cloud features; a cloud's output does not depend on its batch; every refusal writes and queues nothing; and
describe-points calls share one stream with every other batch kind."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import (FEATURE_ARRAYS, LIST_LAYOUT, MEM_DEVICE, MEM_HOST, POINT_ARRAYS, RESULT_DTYPE, SET_LISTS, FeatureOut,
                              ListBuffers)
from support import P4, ROOT, _host, device_copies, host_lists, make_handle, make_params, same_bits, sentinel

NEW = ("qb200_describe_points_each", "qb200_describe_points_enqueue_each")
OK = 0


# ---- CPU: the POD, the header, the symbols -----------------------------------------------------------------------------------------
def test_header_compiles_as_c11_and_feature_out_matches(tmp_path):
    """The header compiles as C11 with the new prototypes called as the header declares them, and the ctypes mirror of
    qb200_feature_out still has the C layout."""
    body = '  printf("size %zu\\n", sizeof(qb200_feature_out));\n' + "".join(
        f'  printf("{f} %zu\\n", offsetof(qb200_feature_out, {f}));\n' for f, _ in FeatureOut._fields_)
    calls = ("  int (*each)(qb200_handle*, const float* const*, const int32_t*, int32_t, const qb200_params*, qb200_mem_kind,\n"
             "              const qb200_feature_out*) = qb200_describe_points_each;\n"
             "  int (*enq)(qb200_handle*, const float* const*, const int32_t*, int32_t, const qb200_params*, qb200_mem_kind,\n"
             "             const qb200_feature_out*) = qb200_describe_points_enqueue_each;\n"
             '  printf("fns %d\\n", each != 0 && enq != 0);\n')
    (tmp_path / "pod.c").write_text('#include <stddef.h>\n#include <stdio.h>\n#include "quatro_b200.h"\nint main(void) {\n' + body +
                                    "  return 0;\n}\n")
    (tmp_path / "fns.c").write_text('#include <stdio.h>\n#include "quatro_b200.h"\nint main(void) {\n' + calls + "  return 0;\n}\n")
    for name in ("pod.c", "fns.c"):
        r = subprocess.run(["/usr/bin/gcc", "-std=c11", "-Wall", "-Werror", "-pedantic", f"-I{ROOT / 'include'}", "-c", str(tmp_path / name),
                            "-o", str(tmp_path / (name + ".o"))], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    r = subprocess.run(["/usr/bin/gcc", "-std=c11", f"-I{ROOT / 'include'}", str(tmp_path / "pod.c"), "-o", str(tmp_path / "pod")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    probe = dict(ln.split() for ln in subprocess.run([str(tmp_path / "pod")], capture_output=True, text=True, check=True).stdout.splitlines())
    assert C.sizeof(FeatureOut) == int(probe["size"]) == 48
    for f, _ in FeatureOut._fields_:
        assert getattr(FeatureOut, f).offset == int(probe[f]), f


def test_library_exports_the_describe_points_calls():
    lib = capi.load_library()
    want = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int32), C.c_int32, C.POINTER(capi.Params), C.c_int32, C.POINTER(FeatureOut)]
    for n in NEW:
        assert n in capi.EXPORTED_SYMBOLS and hasattr(lib, n)
        assert getattr(lib, n).argtypes == want and getattr(lib, n).restype == C.c_int32
    assert set(POINT_ARRAYS) < set(FEATURE_ARRAYS) and "vox4" not in POINT_ARRAYS


def test_a_null_handle_is_refused():
    """Without a handle there is nothing to check against: both forms refuse before reading any other argument."""
    lib = capi.load_library()
    out = FeatureOut(16, MEM_HOST)
    for n in NEW:
        assert getattr(lib, n)(None, None, None, 0, None, MEM_HOST, None) == -1
        assert getattr(lib, n)(None, None, None, 3, None, MEM_HOST, C.byref(out)) == -1


# ---- configurations ----------------------------------------------------------------------------------------------------------------
SLOTS, RAW_CAP, BIG_V = 2, 65536, 32768   # a wave holds 2 * SLOTS = 4 clouds; above 17920 voxel points the lattice sort is the library's
CFG = dict(max_batch_slots=SLOTS, max_raw_points=RAW_CAP)
STREET = make_params()                                                         # 0.5 / 0.75, cell resolved
EQUAL = make_params(normal_radius=0.75, fpfh_radius=0.75)                     # normal_radius == fpfh_radius
COARSE = make_params(grid_cell=0.4)                                           # cell below the radius: a reach of two cells
WIDE = make_params(normal_radius=0.6, fpfh_radius=0.9, grid_cell=1.0)
INDOOR = make_params(normal_radius=0.16, fpfh_radius=0.24)
IGNORED = make_params(voxel_size=-1.0, noise_bound=0.0, cbar2=0.0, use_crosscheck=0, inlier_selection_mode=9)   # only the lattice is read


def resolved_cell(p):
    return float(p.grid_cell) if p.grid_cell > 0 else float(np.float32(p.fpfh_radius) * np.float32(1.001953125))


def _bytes(per_cloud):
    return [tuple(None if a is None else _host(a).tobytes() for a in row) for row in per_cloud]


def _stage_ref(h, clouds, params):
    """per cloud: (normals, desc) bytes of qb200_compute_fpfh on that cloud alone with the resolved radii and cell"""
    out = []
    for c, p in zip(clouds, params):
        nrm, desc = h.compute_fpfh(c, p.normal_radius, p.fpfh_radius, resolved_cell(p))
        out.append((nrm.tobytes(), desc.tobytes()))
    return out


def _lists(buffers, records):
    return [{k: v.tobytes() for k, v in d.items()} for d in host_lists(buffers.trimmed(records))]


def dense_patch(rng, n=2500):
    """A non-voxelized patch: every point has several hundred neighbours within 0.75 m, far above the 80 of the neighbour list."""
    return P4(rng.uniform(-0.6, 0.6, (n, 3)) * np.array([1.0, 1.0, 0.2]))


def mixed_clouds():
    """(label, cloud, entry): voxel keypoints of street, dense and indoor scans, the same shuffled, duplicates with NaN / inf rows,
    points outside the lattice, a dense patch, an empty cloud and a cloud of exactly BIG_V points.  Built on the CPU from the oracle-free
    generator, voxelized by a handle."""
    rng = np.random.default_rng(11)
    street = [synth.outdoor_pair(s, rings=32, azimuths=900)[0] for s in (40, 41)]
    indoor = synth.indoor_pair(3, n_rays=60000)[0]
    with make_handle(1, max_voxel_points=BIG_V, **CFG) as h:
        sv = h.voxelize(street[0], 0.3, 1, cap=BIG_V)[0]
        dv = h.voxelize(street[1], 0.22, 1, cap=BIG_V)[0]
        iv = h.voxelize(indoor, 0.08, 1, cap=BIG_V)[0]
    dup = np.concatenate([sv[:3000], sv[:3000:4], sv[10:15]])
    dup[[7, 500, 2900]] = np.array([np.nan, 0.0, 0.0, 1.0], np.float32)
    dup[1200, 1] = np.inf
    dup[1600, 2] = -np.inf
    dup[2222, 3] = -1.0                                                      # a flagged w is kept: there is no voxel filter
    far = sv[:2500].copy()
    far[::3, 0] += np.float32(120000.0)                                      # a third of the points lie beyond the lattice
    big = P4(rng.uniform([-60, -60, -2], [60, 60, 2], (BIG_V, 3)))
    return [("street", sv, STREET), ("dense", dv, COARSE), ("indoor", iv, INDOOR),
            ("street shuffled", sv[rng.permutation(len(sv))], WIDE), ("dense shuffled", dv[rng.permutation(len(dv))], EQUAL),
            ("indoor shuffled", iv[rng.permutation(len(iv))], INDOOR), ("duplicates nan inf", dup, STREET),
            ("outside the lattice", far, EQUAL), ("dense patch", dense_patch(rng), STREET), ("empty", np.zeros((0, 4), np.float32), WIDE),
            ("max_voxel_points", big, IGNORED)]


def test_dense_patch_exceeds_the_neighbour_list():
    """Every point of the dense patch has more than the 80 listed neighbours within fpfh_radius, so its SPFH and FPFH walk the lattice."""
    pts = dense_patch(np.random.default_rng(11))[:, :3].astype(np.float64)
    d2 = ((pts[:, None, :] - pts[None, ::1, :]) ** 2).sum(-1)
    assert ((d2 < 0.75 ** 2).sum(1) > 80).all()


# ---- GPU fixtures ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mixed():
    return mixed_clouds()


@pytest.fixture(scope="module")
def h1():
    h = make_handle(1, max_voxel_points=BIG_V, **CFG)
    yield h
    h.close()


@pytest.fixture(scope="module")
def h4():
    h = make_handle(4, max_voxel_points=BIG_V, **CFG)
    yield h
    h.close()


@pytest.fixture(scope="module")
def ref(mixed):
    with make_handle(1, max_voxel_points=BIG_V, **CFG) as h:
        return _stage_ref(h, [c for _, c, _ in mixed], [p for _, _, p in mixed])


# ---- GPU 1: every cloud equals qb200_compute_fpfh on it alone -----------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 4])
def test_every_cloud_equals_compute_fpfh_alone(h1, h4, mixed, ref, lanes):
    h = h1 if lanes == 1 else h4
    labels, clouds, params = zip(*mixed)
    n = len(clouds)
    assert n > 2 * SLOTS * 2 and len(clouds[-1]) == BIG_V == h.cfg.max_voxel_points
    dev, keep = device_copies(clouds)
    for kind, cs in ((MEM_HOST, clouds), (MEM_DEVICE, dev)):
        for dest in (MEM_HOST, MEM_DEVICE):
            per_cloud, counts, status = h.describe_points_each(cs, params, kind, dest)
            assert (status == OK).all() and list(counts) == [len(c) for c in clouds], (kind, dest)
            got = _bytes(per_cloud)
            for i in range(n):
                assert got[i] == ref[i], (labels[i], kind, dest)
            assert not h.stage_ms().any() and not h.kernel_ms()[0].any()   # a call that registers nothing reports zeros
    # the clouds reach what they were built for: points the lattice drops get NaN normals, the others do not
    nrm = {lab: np.frombuffer(r[0], np.float32).reshape(-1, 4) for lab, r in zip(labels, ref)}
    assert np.isnan(nrm["outside the lattice"][::3]).all() and not np.isnan(nrm["outside the lattice"][1::3]).all()
    assert np.isnan(nrm["duplicates nan inf"][[7, 1200, 1600]]).all() and not np.isnan(nrm["duplicates nan inf"][3000:]).all()


# ---- GPU 2: the oracle ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_subset_equals_the_oracle(h4, mixed, oracle):
    sel = [m for m in mixed if m[0] in ("street", "indoor shuffled", "duplicates nan inf", "outside the lattice", "dense patch")]
    per_cloud, _, status = h4.describe_points_each([c for _, c, _ in sel], [p for _, _, p in sel])
    assert (status == OK).all()
    for (label, c, p), (nrm, desc) in zip(sel, per_cloud):
        n_ref, d_ref = oracle.compute_fpfh(c, p.normal_radius, p.fpfh_radius, resolved_cell(p))
        assert same_bits(nrm, n_ref, nan_equal=True) and same_bits(desc, d_ref), label


# ---- GPU 3: the voxel keypoints of qb200_describe_batch_each, described again --------------------------------------------------------
@pytest.mark.gpu
def test_describe_batch_keypoints_round_trip(h4):
    scans = [c for s in range(50, 53) for c in synth.outdoor_pair(s, rings=32, azimuths=900)[:2]] + list(synth.indoor_pair(4, n_rays=60000)[:1])
    params = [make_params(voxel_size=0.3), make_params(voxel_size=0.22, grid_cell=0.4), make_params(voxel_size=0.25, normal_radius=0.6,
              fpfh_radius=0.9, grid_cell=1.0), make_params(voxel_size=0.3, normal_radius=0.75), make_params(voxel_size=0.3),
              make_params(voxel_size=0.35), make_params(voxel_size=0.08, normal_radius=0.16, fpfh_radius=0.24)]
    for dest in (MEM_HOST, MEM_DEVICE):
        described, counts, status = h4.describe_batch_each(scans, params, MEM_HOST, dest)
        assert (status == OK).all() and counts.min() > 1000
        vox = [row[0] for row in described]
        clouds = vox if dest == MEM_HOST else [(v.data_ptr(), len(v)) for v in vox]
        again, counts2, _ = h4.describe_points_each(clouds, params, dest, dest)
        assert list(counts2) == list(counts)
        assert _bytes(again) == [b[1:] for b in _bytes(described)], dest


# ---- GPU 4: described keypoints feed qb200_register_features_each ---------------------------------------------------------------------
@pytest.mark.gpu
def test_described_keypoints_register_like_per_cloud_features(h1, h4):
    rng = np.random.default_rng(5)
    pairs = [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(60, 65)]
    pp = [make_params(grid_cell=0.8 if i % 2 else 0.0, seed=5 + i, normal_radius=(0.5, 0.75)[i % 2]) for i in range(len(pairs))]
    kps = []
    for i, (s, t) in enumerate(pairs):   # the caller's own keypoints: voxel centroids, then every point or a random 70 %
        sv, tv = (h1.voxelize(c, 0.3, 1, cap=BIG_V)[0] for c in (s, t))
        if i % 2:
            sv, tv = (v[np.sort(rng.permutation(len(v))[:int(0.7 * len(v))])] for v in (sv, tv))
        kps += [sv, tv]
    dev, keep = device_copies(kps)
    per_cloud, _, status = h4.describe_points_each(dev, [p for p in pp for _ in (0, 1)], MEM_DEVICE, MEM_DEVICE)
    assert (status == OK).all()
    feats_dev = [(dev[2 * i][0], per_cloud[2 * i][1].data_ptr(), dev[2 * i][1], dev[2 * i + 1][0], per_cloud[2 * i + 1][1].data_ptr(),
                  dev[2 * i + 1][1]) for i in range(len(pairs))]
    feats_ref = []
    for i, p in enumerate(pp):
        s, t = kps[2 * i], kps[2 * i + 1]
        feats_ref.append((s, h1.compute_fpfh(s, p.normal_radius, p.fpfh_radius, resolved_cell(p))[1], t,
                          h1.compute_fpfh(t, p.normal_radius, p.fpfh_radius, resolved_cell(p))[1]))
    lb_d, lb_r = ListBuffers(len(pairs), h1.cfg.max_corr), ListBuffers(len(pairs), h1.cfg.max_corr)
    got, _ = h4.register_features_each(feats_dev, pp, MEM_DEVICE, buffers=lb_d)
    want, _ = h1.register_features_each(feats_ref, pp, MEM_HOST, buffers=lb_r)
    assert (want["status"] == OK).sum() >= len(pairs) - 1 and (want["clique_size"] > 3).sum() >= len(pairs) - 1
    assert got.tobytes() == want.tobytes()
    assert _lists(lb_d, got) == _lists(lb_r, want)


# ---- GPU 5: a cloud alone and inside a batch that spans waves and lanes ---------------------------------------------------------------
@pytest.mark.gpu
def test_a_cloud_alone_equals_the_cloud_in_a_batch(h4, mixed):
    sel = [m for m in mixed if m[0] != "max_voxel_points"]
    batch = (sel * 2)[:2 * SLOTS + 1]
    assert len(batch) == 2 * SLOTS + 1                                 # two waves, on two lanes
    clouds, params = [c for _, c, _ in batch], [p for _, _, p in batch]
    whole, _, _ = h4.describe_points_each(clouds, params, dest=MEM_DEVICE)
    whole = _bytes(whole)
    for i, (label, c, p) in enumerate(batch):
        alone, _, _ = h4.describe_points_each([c], [p], dest=MEM_DEVICE)
        assert _bytes(alone)[0] == whole[i], (i, label)


# ---- GPU 6: refusals -------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_rejected_call_writes_and_queues_nothing(h4, mixed, ref):
    lib = h4.lib
    sel = list(range(6))
    clouds, params = [mixed[i][1] for i in sel], [mixed[i][2] for i in sel]
    n, cap = len(clouds), BIG_V
    ptrs, cnts, keep = capi._scan_arrays(clouds, MEM_HOST)
    dev, keep_d = device_copies(clouds)
    dptrs, dcnts, _ = capi._scan_arrays(dev, MEM_DEVICE)
    pa = h4.params_array(params)
    # a feature batch queued before every refused call: its records must come out as a blocking call gives them
    feats = [(clouds[0], np.frombuffer(ref[0][1], np.float32).reshape(-1, 33), clouds[3], np.frombuffer(ref[3][1], np.float32).reshape(-1, 33))]
    fp = [make_params()]
    want_rec, _ = h4.register_features_each(feats, fp)

    def call(dest=MEM_HOST, cap_=cap, arrays=None, counts=True, ps=None, shift=None, kind_as=None, kind=MEM_HOST, edit=None, vox=False):
        names = FEATURE_ARRAYS if vox else POINT_ARRAYS
        arrays = arrays if arrays is not None else {k: sentinel((n + 1, max(cap_, 1), FEATURE_ARRAYS[k]), kind=dest) for k in names}
        c, s = np.full(n, -7, np.int32), np.full(n, -7, np.int32)
        out = h4.feature_out(cap_, dest, arrays, c, s)
        if kind_as is not None:
            out.kind = kind_as
        if not counts:
            out.counts = None
        for k, d in (shift or {}).items():
            setattr(out, k, getattr(out, k) + d)
        p_, c_ = (ptrs, cnts) if kind == MEM_HOST else (dptrs, dcnts)
        p2, c2 = (C.c_void_p * n)(*p_), (C.c_int32 * n)(*c_)
        if edit:
            edit(p2, c2)
        st = lib.qb200_describe_points_enqueue_each(h4.h, p2, c2, n, ps if ps is not None else pa, kind, C.byref(out))
        return st, arrays, c, s

    def bad_entry(i, **kw):
        ps = [capi.Params.from_buffer_copy(p) for p in params]
        for k, v in kw.items():
            setattr(ps[i], k, v)
        return h4.params_array(ps)

    def set_(i, ptr=None, count=None):
        def f(p2, c2):
            if ptr is not None:
                p2[i] = ptr(p2[i])
            if count is not None:
                c2[i] = count
        return f

    ddev = {k: sentinel((n + 1, cap, FEATURE_ARRAYS[k]), kind=MEM_DEVICE) for k in POINT_ARRAYS}
    cases = {
        "negative count": (lambda: call(edit=set_(3, count=-1)), "cloud 3"),
        "count above max_voxel_points": (lambda: call(edit=set_(2, count=BIG_V + 1)), "cloud 2"),
        "null cloud": (lambda: call(edit=set_(4, ptr=lambda p: None)), "cloud 4"),
        "misaligned device cloud": (lambda: call(kind=MEM_DEVICE, edit=set_(1, ptr=lambda p: p + 4)), "cloud 1"),
        "host cloud as device kind": (lambda: call(kind=MEM_DEVICE, edit=set_(5, ptr=lambda p: ptrs[5])), "cloud 5"),
        "normal above fpfh radius": (lambda: call(ps=bad_entry(4, normal_radius=0.8, fpfh_radius=0.75)), "entry 4"),
        "zero radius": (lambda: call(ps=bad_entry(1, normal_radius=0.0)), "entry 1"),
        "infinite radius": (lambda: call(ps=bad_entry(2, fpfh_radius=float("inf"))), "entry 2"),
        "nan grid_cell": (lambda: call(ps=bad_entry(5, grid_cell=float("nan"))), "entry 5"),
        "vox4 given": (lambda: call(vox=True), "vox4"),
        "misaligned device normals4": (lambda: call(MEM_DEVICE, arrays=ddev, shift={"normals4": 8}), "normals4"),
        "misaligned device desc33": (lambda: call(MEM_DEVICE, arrays=ddev, shift={"desc33": 2}), "desc33"),
        "host memory as device kind": (lambda: call(MEM_HOST, kind_as=MEM_DEVICE), "normals4"),
        "null counts": (lambda: call(counts=False), "counts"),
        "cap_per_scan 0": (lambda: call(cap_=0), "cap_per_scan"),
    }
    for name, (fn, culprit) in cases.items():
        arrays0 = {k: sentinel((n + 1, cap, FEATURE_ARRAYS[k]), kind=MEM_HOST) for k in POINT_ARRAYS}
        c0, s0 = np.zeros(n, np.int32), np.zeros(n, np.int32)
        out0 = h4.feature_out(cap, MEM_HOST, arrays0, c0, s0)
        assert lib.qb200_describe_points_enqueue_each(h4.h, ptrs, cnts, n, pa, MEM_HOST, C.byref(out0)) == 0
        rec = np.zeros(1, RESULT_DTYPE)
        farr, kf = h4.feature_array(feats)
        h4.register_features_enqueue_each_raw(farr, 1, h4.params_array(fp), MEM_HOST, rec)
        st, arrays, c, s = fn()
        err = lib.qb200_last_error(h4.h).decode()
        assert st == -1, (name, st, err)
        assert culprit in err, (name, err)
        h4.register_batch_flush()
        assert (c == -7).all() and (s == -7).all(), name
        for k, a in arrays.items():
            assert (_host(a).view(np.uint8) == 0xA5).all(), (name, k)
        assert list(c0) == [len(x) for x in clouds] and (s0 == OK).all(), name
        assert [tuple(arrays0[k][i, :c0[i]].tobytes() for k in POINT_ARRAYS) for i in range(n)] == ref[:n], name
        assert rec.tobytes() == want_rec.tobytes(), name


# ---- GPU 7: one stream of describe-points and every other batch kind -------------------------------------------------------------------
@pytest.mark.gpu
def test_one_stream_of_describe_points_and_every_other_batch(mixed, ref):
    clouds, params = [c for _, c, _ in mixed], [p for _, _, p in mixed]
    n = len(clouds)
    pairs = [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(90, 94)]
    pp = [make_params(seed=3 + i, voxel_size=(0.3, 0.25)[i % 2]) for i in range(len(pairs))]
    sets = [tuple(a[:L] for a in synth.matched_pairs(700 + i, L, inlier_ratio=0.35, noise=0.03)[:2]) for i, L in enumerate([40, 300, 1200])]
    sp = [make_params()] * len(sets)
    slot_pairs = [(0, 1), (2, 3)]
    cache_scans = [c for pr in pairs[:2] for c in pr]
    cache_pp = [p for p in pp[:2] for _ in (0, 1)]
    with make_handle(4, max_voxel_points=BIG_V, **CFG) as h:
        h.cache_reserve(4)
        feats = [(clouds[0], np.frombuffer(ref[0][1], np.float32).reshape(-1, 33), clouds[3], np.frombuffer(ref[3][1], np.float32).reshape(-1, 33))]
        dev, keep = device_copies(clouds)
        cap = h.cfg.max_voxel_points

        def run(queued):
            a_host, a_dev = h.feature_buffers(n, cap, MEM_HOST, POINT_ARRAYS), h.feature_buffers(n, cap, MEM_DEVICE, POINT_ARRAYS)
            a_scan = h.feature_buffers(len(pairs), cap, MEM_HOST)
            cnt = [np.zeros(max(n, len(pairs)), np.int32) for _ in range(6)]
            o_host, o_dev = h.feature_out(cap, MEM_HOST, a_host, cnt[0], cnt[1]), h.feature_out(cap, MEM_DEVICE, a_dev, cnt[2], cnt[3])
            o_scan = h.feature_out(cap, MEM_HOST, a_scan, cnt[4], cnt[5])
            recs = [np.zeros(k, RESULT_DTYPE) for k in (len(pairs), len(slot_pairs), len(feats), len(sets))]
            bufs = [ListBuffers(len(r), h.cfg.max_corr, MEM_HOST, SET_LISTS if k == 3 else tuple(LIST_LAYOUT)) for k, r in enumerate(recs)]
            sh, ch, kh = capi._scan_arrays(clouds, MEM_HOST)
            sd, cd, _ = capi._scan_arrays(dev, MEM_DEVICE)
            wp, wc, wk = capi._scan_arrays(cache_scans, MEM_HOST)
            rp, rc, rk = capi._scan_arrays([pr[0] for pr in pairs], MEM_HOST)
            ids = (C.c_int32 * 4)(*range(4))
            pair_arr, kp = h.pair_array(pairs)
            feat_arr, kf = h.feature_array(feats)
            set_arr, ks = h._set_array(sets, MEM_HOST)
            slot_arr = capi._slot_array(slot_pairs)
            pa = [h.params_array(x) for x in (params, pp, cache_pp, pp[:2], [make_params()], sp)]
            steps = [
                lambda: h.describe_points_enqueue_each_raw(sh, ch, n, pa[0], MEM_HOST, o_host),
                lambda: h.register_batch_enqueue_mixed_raw(pair_arr, len(pairs), pa[1], MEM_HOST, recs[0], bufs[0]),
                lambda: h.cache_scans_enqueue_each_raw(wp, wc, ids, 4, pa[2], MEM_HOST),
                lambda: h.register_cached_enqueue_mixed_raw(slot_arr, len(slot_pairs), pa[3], recs[1], bufs[1]),
                lambda: h.describe_points_enqueue_each_raw(sd, cd, n, pa[0], MEM_DEVICE, o_dev),
                lambda: h.register_features_enqueue_each_raw(feat_arr, len(feats), pa[4], MEM_HOST, recs[2], bufs[2]),
                lambda: h.describe_batch_enqueue_each_raw(rp, rc, len(pairs), pa[1], MEM_HOST, o_scan),
                lambda: h.solve_batch_enqueue_each_raw(set_arr, len(sets), pa[5], MEM_HOST, recs[3], bufs[3]),
            ]
            for step in steps:
                step()
                if not queued:
                    h.register_batch_flush()
            h.register_batch_flush()
            outs = {"records": [r.tobytes() for r in recs], "lists": [_lists(b, r) for b, r in zip(bufs, recs)],
                    "counts": [c.tobytes() for c in cnt]}
            outs["described"] = [[tuple(_host(arr[k])[i, :cnt[2 * j][i]].tobytes() for k in POINT_ARRAYS) for i in range(n)]
                                 for j, arr in enumerate((a_host, a_dev))]
            outs["scans"] = [tuple(a_scan[k][i, :cnt[4][i]].tobytes() for k in FEATURE_ARRAYS) for i in range(len(pairs))]
            return outs

        got, want = run(True), run(False)
        assert got == want
        assert got["described"][0] == got["described"][1] == ref
        recs = np.frombuffer(got["records"][0], RESULT_DTYPE)
        assert (recs["status"] == OK).sum() >= len(pairs) - 1
