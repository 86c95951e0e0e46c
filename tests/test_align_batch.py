"""Aligned scans, transformed matches and good matches of registered pairs: qb200_align_batch_each and its queued form.  A float64
restatement of the example's step after computeTransformation (the transform of pcl_compat.hpp's transformPointCloud, PCL's
pass-through of non-finite points, the good-match loop with pow(d, 2) as d * d) is pinned against that code compiled from the
header; the device must equal it byte for byte on adversarial clouds, at the threshold, with refused sets, empty sets and clipping,
across waves, memory kinds, lane counts and used handles, on street pairs registered end to end, and queued beside feature batches."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest

from quatro_b200 import capi, synth
from quatro_b200.capi import (MEM_DEVICE, MEM_HOST, AlignOut, AlignSet, ListBuffers, default_params)
from support import ROOT, build_against_lib, device_copy, make_handle, sentinel

NEW = ("qb200_align_batch_each", "qb200_align_batch_enqueue_each")
BAD_ARG = -1
OK = 0
NAMES = ("aligned4", "matched4", "good_ids", "good4")


# ---- the restatement --------------------------------------------------------------------------------------------------------------------
def transform(pts4, T):
    """pcl::transformPointCloud with a Matrix4d: (float)(T(r,0)*x + T(r,1)*y + T(r,2)*z + T(r,3)) in float64, left to right, w copied;
    a point with a non-finite x, y or z passes through unchanged."""
    p = np.asarray(pts4, np.float32).reshape(-1, 4)
    x, y, z = (p[:, i].astype(np.float64) for i in range(3))
    out = p.copy()
    with np.errstate(all="ignore"):
        for r in range(3):
            out[:, r] = (((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3]).astype(np.float32)
    keep = ~(np.isfinite(p[:, 0]) & np.isfinite(p[:, 1]) & np.isfinite(p[:, 2]))
    out[keep] = p[keep]
    return out


def distances(m4, t4):
    """sqrt(dx*dx + dy*dy + dz*dz) of float32 points widened to float64, the squares summed in that order"""
    with np.errstate(all="ignore"):
        d = [m4[:, i].astype(np.float64) - t4[:, i].astype(np.float64) for i in range(3)]
        return np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])


def threshold(voxel_size):
    return 3.0 * float(np.float32(voxel_size))


def restate(st, voxel_size):
    """what the call must write for one set: (aligned4, matched4, good_ids, good4), or None when a correspondence index is out of
    range (the set is refused)"""
    T = np.asarray(st["T"], np.float64).reshape(4, 4)
    src = np.asarray(st.get("src_kp", np.zeros((0, 4))), np.float32).reshape(-1, 4)
    tgt = np.asarray(st.get("tgt_kp", np.zeros((0, 4))), np.float32).reshape(-1, 4)
    corr = np.asarray(st.get("corr", np.zeros((0, 2))), np.int32).reshape(-1, 2)
    if ((corr[:, 0] < 0) | (corr[:, 0] >= len(src)) | (corr[:, 1] < 0) | (corr[:, 1] >= len(tgt))).any():
        return None
    cloud = st.get("cloud")
    aligned = transform(np.zeros((0, 4)) if cloud is None else cloud, T)
    matched = transform(src[corr[:, 0]], T)
    with np.errstate(invalid="ignore"):
        good = distances(matched, tgt[corr[:, 1]]) < threshold(voxel_size)
    ids = np.flatnonzero(good).astype(np.int32)
    return aligned, matched, ids, matched[ids]


def pose(yaw, t, neg_zero=False):
    c, s = np.cos(yaw), np.sin(yaw)
    T = np.eye(4)
    T[:2, :2] = [[c, -s], [s, c]]
    T[:3, 3] = t
    if neg_zero:
        T[np.abs(T) == 0] = -0.0
    return T


def random_set(rng, n_points, n_src, n_tgt, n_corr, T=None, spread=30.0):
    src = rng.uniform(-spread, spread, (n_src, 4)).astype(np.float32)
    src[:, 3] = rng.choice([1.0, -1.0], n_src)
    T = pose(rng.uniform(-np.pi, np.pi), rng.uniform(-5, 5, 3)) if T is None else T
    tgt = rng.uniform(-spread, spread, (n_tgt, 4)).astype(np.float32)
    corr = np.stack([rng.integers(0, max(n_src, 1), n_corr), rng.integers(0, max(n_tgt, 1), n_corr)], 1).astype(np.int32)
    # about half the correspondences land near their transformed source point
    near = rng.random(n_corr) < 0.5
    if n_src and n_tgt:
        moved = transform(src[corr[near, 0]], T)
        tgt[corr[near, 1], :3] = moved[:, :3] + rng.normal(0, 0.5, (near.sum(), 3)).astype(np.float32)
    cloud = rng.normal(0, spread, (n_points, 4)).astype(np.float32)
    return {"cloud": cloud, "src_kp": src, "tgt_kp": tgt, "corr": corr, "T": T}


def adversarial_sets():
    """(name, set) of the adversarial cloud families; the keypoints carry the same values so matched4 and the test see them too"""
    rng = np.random.default_rng(7)
    fam = {}
    base = rng.uniform(-50, 50, (700, 4)).astype(np.float32)
    bad = base.copy()
    bad[::7, 0] = np.nan
    bad[1::7, 1] = np.inf
    bad[2::7, 2] = -np.inf
    bad[3::7, 3] = np.nan   # w alone is not a coordinate: the point is transformed, w copied
    fam["non_finite"] = (bad, pose(0.3, [1, 2, 3]))
    big = rng.uniform(-3.4e38, 3.4e38, (700, 4)).astype(np.float32)
    fam["near_float_max"] = (big, pose(0.7, [0, 0, 0]))
    den = (rng.integers(1, 2 ** 23, (700, 4)).astype(np.uint32) | (rng.integers(0, 2, (700, 4)).astype(np.uint32) << 31)).view(np.float32)
    fam["denormals"] = (den, pose(1.1, [0, 0, 0]))
    fam["denormals_translated"] = (den, pose(0.0, [1e-40, -1e-41, 3e-39]))
    fam["far_translation"] = (base, pose(-2.0, [1e6, -1e6, 2.5e5]))
    fam["identity"] = (bad, np.eye(4))
    fam["negative_zero"] = (np.concatenate([base, -np.zeros((5, 4), np.float32)]), pose(0.0, [0, 0, 0], neg_zero=True))
    out = []
    for name, (pts, T) in fam.items():
        n = len(pts)
        corr = np.stack([rng.integers(0, n, 900), rng.integers(0, n, 900)], 1).astype(np.int32)
        tgt = transform(pts, T)
        tgt[::3] = pts[::3]
        out.append((name, {"cloud": pts, "src_kp": pts, "tgt_kp": tgt, "corr": corr, "T": T}))
    return out


def threshold_sets(voxel_size=0.3):
    """three sets whose one correspondence lies at exactly 3 * voxel_size, one float64 ulp below and one above (identity pose):
    src (c, 0, 0), tgt (t, dy, 0) with t - c and dy chosen so that the restated distance is exactly the target"""
    tau = threshold(voxel_size)
    out = []
    for target in (np.nextafter(tau, 0.0), tau, np.nextafter(tau, np.inf)):
        t = np.float32(tau)
        t = t if float(t) > target else np.nextafter(t, np.float32(np.inf))
        c = np.float32(float(t) - target)
        while float(t) - float(c) > target:
            c = np.nextafter(c, np.float32(np.inf))
        dx = float(t) - float(c)
        found = None
        if dx == target:
            found = np.float32(0.0)
        else:
            dy0 = np.float32(np.sqrt((target - dx) * (target + dx)))
            for k in range(-4096, 4097):
                dy = np.float32(dy0 + np.float32(k) * np.spacing(dy0))
                m, q = np.array([[c, 0, 0, 1]], np.float32), np.array([[t, dy, 0, 1]], np.float32)
                if distances(m, q)[0] == target:
                    found = dy
                    break
        assert found is not None
        src = np.array([[c, 0, 0, 1]], np.float32)
        tgt = np.array([[t, found, 0, 1]], np.float32)
        assert distances(src, tgt)[0] == target
        out.append((target, {"cloud": src, "src_kp": src, "tgt_kp": tgt, "corr": np.array([[0, 0]], np.int32), "T": np.eye(4)}))
    return out


# ---- CPU: layouts, prototypes, the restatement against the example's code ------------------------------------------------------------
@pytest.mark.parametrize("struct,fields", [
    ("qb200_align_set", ("cloud", "src_kp", "tgt_kp", "corr", "n_points", "n_src", "n_tgt", "n_corr", "T")),
    ("qb200_align_out", ("cap_points", "cap_corr", "kind", "reserved", "aligned4", "matched4", "good_ids", "good4", "counts", "status")),
])
def test_align_mirrors_match_the_c_layout(tmp_path, struct, fields):
    mirror = AlignSet if struct == "qb200_align_set" else AlignOut
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "quatro_b200.h"\nint main(void) {\n'
                   '  printf("%zu' + " %zu" * len(fields) + f'\\n", sizeof({struct})' +
                   "".join(f", offsetof({struct}, {f})" for f in fields) + ");\n  return 0;\n}\n")
    exe = tmp_path / "layout"
    r = subprocess.run(["/usr/bin/gcc", "-std=c11", "-Wall", "-Werror", f"-I{ROOT / 'include'}", str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(mirror)] + [getattr(mirror, f).offset for f in fields]


def test_header_declares_both_entry_points_and_documents_the_structs(tmp_path):
    header = (ROOT / "include" / "quatro_b200.h").read_text()
    for n in NEW:
        decl = header[header.index(f"int {n}("):]
        decl = decl[:decl.index(");")]
        assert decl.count(",") + 1 == len(capi._SIGNATURES[n][1]), n
    for s in ("qb200_align_set", "qb200_align_out"):
        assert f"}} {s};" in header
    assert "qb200_align_batch_*" in header[:header.index("Conventions")]
    assert "pow(d, 2)" in header and "d*d" in header
    body = "".join(f"  __typeof__(&{NEW[0]}) p{i} = {n};\n  (void)p{i};\n" for i, n in enumerate(NEW))
    (tmp_path / "proto.c").write_text('#include "quatro_b200.h"\nint main(void) {\n' + body + "  return 0;\n}\n")
    r = subprocess.run(["/usr/bin/gcc", "-std=gnu11", "-Wall", "-Werror", "-Wincompatible-pointer-types", f"-I{ROOT / 'include'}", "-c",
                        str(tmp_path / "proto.c"), "-o", str(tmp_path / "proto.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = capi.load_library()
    for n in NEW:
        assert n in capi.EXPORTED_SYMBOLS and hasattr(lib, n)


def test_a_null_handle_is_refused():
    lib = capi.load_library()
    out = AlignOut(1, 1, MEM_HOST)
    for n in NEW:
        assert getattr(lib, n)(None, None, 0, None, MEM_HOST, C.byref(out)) == BAD_ARG, n


def test_the_integration_snippet_compiles(tmp_path):
    """The describe -> match -> solve -> align loop-closure example of INTEGRATION.md, with the names it takes from the steps before
    it as parameters, compiles as C++ against the header."""
    text = (ROOT / "INTEGRATION.md").read_text()
    blocks = [b for b in re.findall(r"```cpp\n(.*?)```", text, re.S) if "qb200_align_batch_each" in b]
    assert len(blocks) == 1
    src = ("#include <vector>\n#include \"quatro_b200.h\"\n"
           "int close_loops(qb200_handle* h, const std::vector<qb200_feature_pair>& feats, const std::vector<qb200_params>& ps,\n"
           "                const float* const* d_scans, const int32_t* n_points, int32_t max_points, int32_t max_corr,\n"
           "                int32_t* d_corr, float* d_aligned, int32_t* d_good_ids) {\n"
           + blocks[0] + "}\n")
    (tmp_path / "loop.cpp").write_text(src)
    r = subprocess.run(["/usr/bin/g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", f"-I{ROOT / 'include'}", "-fsyntax-only",
                        str(tmp_path / "loop.cpp")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def run_example(exe, tmp_path, st, voxel_size):
    src, tgt, corr = (np.asarray(st[k]) for k in ("src_kp", "tgt_kp", "corr"))
    blob = (np.array([len(src), len(tgt), len(corr)], np.int32).tobytes() + np.asarray(st["T"], np.float64).T.ravel().tobytes()
            + np.array([float(np.float32(voxel_size))], np.float64).tobytes() + np.ascontiguousarray(src[:, :3], np.float32).tobytes()
            + np.ascontiguousarray(tgt[:, :3], np.float32).tobytes() + np.ascontiguousarray(corr, np.int32).tobytes())
    (tmp_path / "in.bin").write_bytes(blob)
    subprocess.run([str(exe), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], check=True)
    raw = (tmp_path / "out.bin").read_bytes()
    f = np.frombuffer(raw, np.float32, 3 * (len(src) + len(corr)))
    n_good = int(np.frombuffer(raw, np.int32, 1, 4 * f.size)[0])
    ids = np.frombuffer(raw, np.int32, n_good, 4 * (f.size + 1))
    good = np.frombuffer(raw, np.float32, 3 * n_good, 4 * (f.size + 1 + n_good)).reshape(-1, 3)
    return f[:3 * len(src)].reshape(-1, 3), f[3 * len(src):].reshape(-1, 3), ids, good


def test_restatement_equals_the_example_through_pcl_compat(tmp_path):
    """On finite keypoints (the example's transformPointCloud has no pass-through), the restatement gives the bytes of the example's
    code: the transformed keypoints, the matched ones, the good ids and good_matched_pcl; the threshold cases included."""
    exe = build_against_lib(tmp_path, "tests/fixtures/align_example.cpp")
    rng = np.random.default_rng(3)
    cases = [(0.3, random_set(rng, 0, 400, 300, 1000)), (0.05, random_set(rng, 0, 50, 60, 200, spread=1.0)),
             (1.0, random_set(rng, 0, 10, 10, 0))]
    for name, st in adversarial_sets():
        if name not in ("non_finite", "identity"):
            cases.append((0.3, st))
    cases += [(0.3, st) for _, st in threshold_sets()]
    for voxel, st in cases:
        src = np.asarray(st["src_kp"], np.float32)
        a, m, ids, good = run_example(exe, tmp_path, st, voxel)
        _, matched, want_ids, want_good = restate(dict(st, cloud=None), voxel)
        assert a.tobytes() == np.ascontiguousarray(transform(src, np.asarray(st["T"]))[:, :3]).tobytes()
        assert m.tobytes() == np.ascontiguousarray(matched[:, :3]).tobytes()
        assert ids.tobytes() == want_ids.tobytes()
        assert good.tobytes() == np.ascontiguousarray(want_good[:, :3]).tobytes()
    # exactly at the threshold is not a good match; one ulp below is, one above is not
    got = [len(restate(st, 0.3)[2]) for _, st in threshold_sets()]
    assert got == [1, 0, 0]


# ---- GPU helpers ------------------------------------------------------------------------------------------------------------------------
def on_device(sets):
    """the sets with every array in device memory: (sets as the call takes them, the tensors that hold them)"""
    keep, out = [], []
    for st in sets:
        d = {"T": st["T"]}
        for k in ("cloud", "src_kp", "tgt_kp", "corr"):
            a = st.get(k)
            if a is None or len(a) == 0:
                d[k] = None
                continue
            t = device_copy(np.ascontiguousarray(a, np.int32 if k == "corr" else np.float32))
            keep.append(t)
            d[k] = (t.data_ptr(), len(a))
        out.append(d)
    return out, keep


def run(h, sets, voxels, kind=MEM_HOST, dest=MEM_HOST, cap_points=None, cap_corr=None, fill=True):
    """align_batch_each with 0xA5-filled outputs (fill) -> (per set dict trimmed, counts, status, the full arrays on the host)"""
    n = len(sets)
    cp = cap_points or max([len(s.get("cloud") if s.get("cloud") is not None else ()) for s in sets] + [1])
    cc = cap_corr or max([len(s.get("corr", ())) for s in sets] + [1])
    arrays = {k: sentinel((max(n, 1), cp if k == "aligned4" else cc) + ((4,) if k != "good_ids" else ()),
                          np.int32 if k == "good_ids" else np.float32, dest) for k in NAMES} if fill else None
    call_sets, keep = on_device(sets) if kind == MEM_DEVICE else (sets, None)
    params = [capi.default_params() for _ in range(n)]
    for p, v in zip(params, voxels):
        p.voxel_size = v
    per, counts, status = h.align_batch_each(call_sets, params, kind, dest, cp, cc, arrays)
    full = {k: (a if dest == MEM_HOST else a.cpu().numpy()) for k, a in arrays.items()} if fill else None
    return per, counts, status, full


def check(per_set, counts, status, st, voxel, label, full=None, i=None, cp=None, cc=None):
    """one set's outputs against the restatement, byte for byte; with full (sentinel-filled arrays), nothing past the counts"""
    want = restate(st, voxel)
    if want is None:
        assert status == BAD_ARG, label
        if full is not None:
            assert all((full[k][i].view(np.uint8) == 0xA5).all() for k in NAMES), label
        return
    assert status == OK, label
    aligned, matched, ids, good = want
    assert list(counts) == [len(aligned), len(matched), len(ids)], (label, counts)
    got = {k: np.asarray(v if isinstance(v, np.ndarray) else v.cpu().numpy()) for k, v in per_set.items()}
    for k, w in zip(NAMES, (aligned, matched, ids, good)):
        g, cap = got[k], cp if k == "aligned4" else cc
        assert g.tobytes() == w[:len(g)].tobytes(), (label, k)
        assert len(g) == (len(w) if cap is None else min(len(w), cap)), (label, k)
    if full is not None:
        for k in NAMES:
            rest = full[k][i][len(got[k]):]
            assert (rest.view(np.uint8) == 0xA5).all(), (label, k)


# ---- GPU: adversarial clouds and the threshold ------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_adversarial_clouds_equal_the_restatement_and_the_set_alone(handle):
    named = adversarial_sets()
    sets = [s for _, s in named]
    voxels = [0.3] * len(sets)
    per, counts, status, full = run(handle, sets, voxels)
    for i, (name, st) in enumerate(named):
        check(per[i], counts[i], status[i], st, 0.3, name, full, i)
        alone = run(handle, [st], [0.3])
        for k in NAMES:
            assert alone[0][0][k].tobytes() == per[i][k].tobytes(), (name, k)


@pytest.mark.gpu
def test_threshold_at_and_one_ulp_either_side(handle):
    cases = threshold_sets()
    per, counts, status, _ = run(handle, [s for _, s in cases], [0.3] * 3)
    assert [int(c[2]) for c in counts] == [1, 0, 0]
    for i, (_, st) in enumerate(cases):
        check(per[i], counts[i], status[i], st, 0.3, f"threshold {i}")


# ---- GPU: refusals, empty sets, clipping ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", [MEM_HOST, MEM_DEVICE])
def test_bad_indices_refuse_their_set_alone(handle, kind):
    rng = np.random.default_rng(11)
    sets = [random_set(rng, 300, 40, 50, 120) for _ in range(6)]
    sets[0]["corr"] = np.concatenate([sets[0]["corr"], sets[0]["corr"][:10]])   # duplicates are taken as they are
    sets[1]["corr"][17, 0] = 40            # n_src
    sets[3]["corr"][119, 1] = -1
    sets[4]["corr"][0, 1] = 2 ** 31 - 1
    per, counts, status, full = run(handle, sets, [0.5] * 6, kind, kind)
    assert list(status) == [OK, BAD_ARG, OK, BAD_ARG, BAD_ARG, OK]
    for i, st in enumerate(sets):
        check(per[i], counts[i], status[i], st, 0.5, f"set {i}", full, i)
    for i in (1, 3, 4):
        assert list(counts[i]) == [0, 0, 0]   # left as the wrapper zeroed them: the call writes no counts for a refused set


@pytest.mark.gpu
def test_empty_sets_null_cloud_and_clipping(handle):
    rng = np.random.default_rng(12)
    sets = [random_set(rng, 0, 10, 10, 0), dict(random_set(rng, 0, 10, 10, 30), cloud=None), random_set(rng, 5000, 100, 80, 600),
            random_set(rng, 17, 0, 0, 0), random_set(rng, 2500, 300, 300, 1000)]
    for cp, cc in ((1, 1), (64, 100), (3000, 700), (5000, 1000)):
        per, counts, status, full = run(handle, sets, [0.7] * len(sets), cap_points=cp, cap_corr=cc)
        for i, st in enumerate(sets):
            check(per[i], counts[i], status[i], st, 0.7, f"set {i} caps {cp}/{cc}", full, i, cp, cc)


# ---- GPU: batch independence ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def wave_sets():
    rng = np.random.default_rng(21)
    sizes = rng.integers(0, 9000, 37)
    sets = [random_set(rng, int(n), int(rng.integers(1, 500)), int(rng.integers(1, 500)), int(rng.integers(0, 1500))) for n in sizes]
    sets[5]["corr"][:1, 0] = -5
    voxels = list(rng.choice([0.1, 0.3, 1.0, 2.5], len(sets)))
    return sets, voxels


@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, None])
def test_waves_kinds_lanes_and_used_handles_give_the_same_bytes(wave_sets, lanes):
    sets, voxels = wave_sets
    rng = np.random.default_rng(22)
    with make_handle(lanes, max_batch_slots=4, max_raw_points=12000, max_voxel_points=1024, max_corr=2048) as h:
        # earlier, larger waves on the same handle: every lane's staging and tables hold their data
        big = [random_set(rng, 12000, 1024, 1024, 2048) for _ in range(12)]
        run(h, big, [0.4] * len(big), MEM_HOST, MEM_HOST)
        run(h, big, [0.4] * len(big), MEM_DEVICE, MEM_DEVICE)
        ref = None
        for kind in (MEM_HOST, MEM_DEVICE):
            for dest in (MEM_HOST, MEM_DEVICE):
                per, counts, status, full = run(h, sets, voxels, kind, dest, cap_points=9000, cap_corr=1500)
                for i, st in enumerate(sets):
                    check(per[i], counts[i], status[i], st, voxels[i], f"set {i} kind {kind} dest {dest}", full, i, 9000, 1500)
                if ref is None:
                    ref = (full, counts, status)
                assert all(full[k].tobytes() == ref[0][k].tobytes() for k in NAMES)
                assert counts.tobytes() == ref[1].tobytes() and status.tobytes() == ref[2].tobytes()
        for i in (0, 5, 36):
            alone = run(h, [sets[i]], [voxels[i]], cap_points=9000, cap_corr=1500)
            assert all(alone[3][k][0].tobytes() == ref[0][k][i].tobytes() for k in NAMES), i


# ---- GPU: rejections ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rejections_write_nothing_and_name_the_set(handle):
    rng = np.random.default_rng(31)
    good = [random_set(rng, 50, 20, 20, 30) for _ in range(3)]
    lib = handle.lib
    V, R, Lc = handle.cfg.max_voxel_points, handle.cfg.max_raw_points, handle.cfg.max_corr

    def attempt(mutate, voxel=0.3, out_mut=None, kind=MEM_HOST):
        arr, keep = handle.align_array(good, MEM_HOST)
        mutate(arr)
        params = [capi.default_params() for _ in good]
        params[2].voxel_size = voxel
        arrays = handle.align_buffers(3, 64, 64, MEM_HOST)
        for a in arrays.values():
            a.view(np.uint8)[...] = 0xA5
        counts, status = np.full((3, 3), -7, np.int32), np.full(3, -7, np.int32)
        out = handle.align_out(64, 64, MEM_HOST, arrays, counts, status)
        if out_mut:
            out_mut(out)
        rc = lib.qb200_align_batch_each(handle.h, arr, 3, handle.params_array(params), kind, C.byref(out))
        assert (counts == -7).all() and (status == -7).all()
        assert all((a.view(np.uint8) == 0xA5).all() for a in arrays.values())
        return rc, lib.qb200_last_error(handle.h).decode()

    def setf(field, value):
        return lambda arr: setattr(arr[2], field, value)

    def set_t(arr):
        arr[2].T[5] = float("nan")

    for mut, words in ((setf("n_points", -1), "set 2"), (setf("n_points", R + 1), "set 2"), (setf("n_src", V + 1), "set 2"),
                       (setf("n_tgt", -3), "set 2"), (setf("n_corr", Lc + 1), "set 2"), (setf("corr", None), "set 2"),
                       (setf("cloud", None), "set 2"), (set_t, "set 2")):
        rc, msg = attempt(mut)
        assert rc == BAD_ARG and words in msg, msg
    for v in (0.0, -1.0, float("nan")):
        rc, msg = attempt(lambda arr: None, voxel=v)
        assert rc == BAD_ARG and "entry 2" in msg, msg
    for out_mut in (lambda o: setattr(o, "kind", 7), lambda o: setattr(o, "cap_points", 0), lambda o: setattr(o, "cap_corr", -1)):
        rc, msg = attempt(lambda arr: None, out_mut=out_mut)
        assert rc == BAD_ARG, msg
    # host memory passed as device kind
    rc, msg = attempt(lambda arr: None, kind=MEM_DEVICE)
    assert rc == BAD_ARG and "set 0" in msg, msg
    rc, msg = attempt(lambda arr: None, out_mut=lambda o: setattr(o, "kind", MEM_DEVICE))
    assert rc == BAD_ARG and "device" in msg, msg
    assert lib.qb200_align_batch_each(handle.h, None, 1, None, MEM_HOST, None) == BAD_ARG


# ---- GPU: end to end on street pairs ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_registered_street_pairs_equal_the_example_and_the_oracle(oracle):
    seeds = range(4100, 4106)
    pairs = [synth.outdoor_pair(s)[:2] for s in seeds]
    params = []
    for i in range(len(pairs)):
        p = default_params()
        p.rot_noise_bound = 2 * p.noise_bound
        p.voxel_size = (0.3, 0.35, 0.25)[i % 3]
        params.append(p)
    with make_handle(None, max_batch_slots=4) as h:
        lb = ListBuffers(len(pairs), h.cfg.max_corr, MEM_HOST, capi.MATCH_LISTS)
        recs, lists = h.register_batch_mixed(pairs, params, buffers=lb)
        src_desc = h.describe_batch_each([s for s, _ in pairs], params, arrays=None)[0]
        tgt_desc = h.describe_batch_each([t for _, t in pairs], params, arrays=None)[0]
        sets = []
        for i, (src, _) in enumerate(pairs):
            corr = lists[i]["corr"]
            sk, tk = src_desc[i][0], tgt_desc[i][0]
            # the lists index the keypoints describe_batch_each writes
            assert sk[corr[:, 0], :3].tobytes() == lists[i]["src_matched4"][:, :3].tobytes()
            assert tk[corr[:, 1], :3].tobytes() == lists[i]["tgt_matched4"][:, :3].tobytes()
            sets.append({"cloud": src, "src_kp": sk, "tgt_kp": tk, "corr": corr, "T": np.asarray(recs["T"][i]).reshape(4, 4).T})
        per, counts, status, full = run(h, sets, [p.voxel_size for p in params], cap_points=h.cfg.max_raw_points,
                                        cap_corr=h.cfg.max_corr)
    for i, ((src, tgt), p) in enumerate(zip(pairs, params)):
        check(per[i], counts[i], status[i], sets[i], p.voxel_size, f"pair {i}")
        assert counts[i][2] > 0, counts[i]   # a registered street pair has good matches
        ref, st = oracle.register_pair(src, tgt, p)
        assert np.allclose(ref.matrix(), sets[i]["T"], atol=1e-9, rtol=0), i


# ---- GPU: one stream with feature batches ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_enqueue_interleaved_with_feature_batches_and_one_flush(handle):
    from support import fpfh_like
    rng = np.random.default_rng(41)
    sets = [random_set(rng, int(rng.integers(0, 3000)), 200, 200, 400) for _ in range(20)]
    voxels = [0.3] * len(sets)
    ref = run(handle, sets, voxels, cap_points=3000, cap_corr=400)
    feats = []
    for _ in range(10):
        a = rng.uniform(-20, 20, (300, 4)).astype(np.float32)
        feats.append((a, fpfh_like(rng, 300), a + np.float32(0.5), fpfh_like(rng, 300)))
    fp = [default_params() for _ in feats]
    for p in fp:
        p.rot_noise_bound = 0.6
    want = handle.register_features_each(feats, fp)[0]
    keep = []
    outs = []
    for part in (slice(0, 9), slice(9, 20)):
        fa, fk = handle.feature_array(feats)
        rec = np.zeros(len(feats), capi.RESULT_DTYPE)
        handle.register_features_enqueue_each_raw(fa, len(feats), handle.params_array(fp), MEM_HOST, rec)
        aa, ak = handle.align_array(sets[part], MEM_HOST)
        arrays = handle.align_buffers(len(sets[part]), 3000, 400, MEM_HOST)
        counts, status = np.zeros((len(sets[part]), 3), np.int32), np.zeros(len(sets[part]), np.int32)
        out = handle.align_out(3000, 400, MEM_HOST, arrays, counts, status)
        pa = handle.params_array([default_params() for _ in sets[part]])
        handle.align_batch_enqueue_each_raw(aa, len(sets[part]), pa, MEM_HOST, out)
        keep += [fa, fk, aa, ak, out, pa]
        outs.append((part, rec, arrays, counts, status))
    handle.register_batch_flush()
    for part, rec, arrays, counts, status in outs:
        idx = range(len(sets))[part]
        assert counts.tobytes() == ref[1][part].tobytes() and status.tobytes() == ref[2][part].tobytes()
        for j, i in enumerate(idx):
            m = {"aligned4": counts[j, 0], "matched4": counts[j, 1], "good_ids": counts[j, 2], "good4": counts[j, 2]}
            for k in NAMES:
                assert arrays[k][j, :m[k]].tobytes() == ref[0][i][k].tobytes(), (i, k)
        assert rec.tobytes() == want.tobytes()
