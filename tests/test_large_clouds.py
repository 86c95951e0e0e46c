"""Clouds of more than 65536 voxel points (max_voxel_points up to QB200_MAX_VOXEL_POINTS = 262144).

The dense indoor hall pair (synth.indoor_pair(0, extent=9.0): 500 k rays per scan, 134 k / 101 k voxel points at a 0.05 m voxel) runs
through every stage and must match the CPU oracle bit for bit, like the smaller clouds of test_gpu_parity.py.  The oracle needs ~15 s
per hall pair on 8 cores, so its results are computed once per module."""
import re
import subprocess

import numpy as np
import pytest

from quatro_b200 import synth
from quatro_b200.capi import RESULT_DTYPE, Handle, QuatroB200Error, default_params
from support import ROOT, assert_same_record, build_against_lib, same_bits

MAX_V = 262144
HALL = dict(extent=9.0)
HANDLE_CFG = dict(max_batch_slots=1, max_raw_points=524288, max_voxel_points=MAX_V, max_corr=8192)


def indoor_params():
    """The indoor parameters of test_gpu_parity.py::test_dense_indoor_pair_50k_voxels."""
    p = default_params()
    p.voxel_size, p.normal_radius, p.fpfh_radius, p.noise_bound, p.cote_noise_bound, p.skip_flagged = 0.05, 0.10, 0.15, 0.05, 0.05, 0
    return p


def default_cell(fpfh_radius):
    """The lattice cell the pipeline uses when qb200_params.grid_cell = 0: (1 + 2^-9) fpfh_radius in float arithmetic."""
    return float(np.float32(fpfh_radius) * np.float32(1.001953125))


# ---- argument validation (no GPU needed) ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("v", [MAX_V + 128, 131072 + 1])
def test_voxel_capacity_beyond_the_limit_or_off_the_tile_grid_is_refused(v):
    with pytest.raises(QuatroB200Error) as e:
        Handle(max_batch_slots=1, max_voxel_points=v)
    assert e.value.code == -1  # QB200_ERR_BAD_ARG, decided before any device is probed


def test_largest_voxel_capacity_passes_validation():
    """262144 is accepted: without a device qb200_create gets as far as the device probe (NO_DEVICE); with one the handle opens."""
    try:
        h = Handle(max_batch_slots=1, max_voxel_points=MAX_V)
    except QuatroB200Error as e:
        assert e.code == -2, e  # QB200_ERR_NO_DEVICE
    else:
        h.close()


def test_header_documents_the_limit():
    txt = (ROOT / "include" / "quatro_b200.h").read_text()
    assert re.search(r"#define\s+QB200_MAX_VOXEL_POINTS\s+262144\b", txt)


# ---- the hall pair on the GPU ------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def hall():
    src, tgt, T = synth.indoor_pair(0, **HALL)
    return src, tgt, T


@pytest.fixture(scope="module")
def hall_ref(hall, oracle):
    """Oracle results on the seed-0 hall pair: voxel clouds, production-radius features and the whole-pipeline record."""
    src, tgt, _ = hall
    p = indoor_params()
    sv, _ = oracle.voxelize(src, p.voxel_size, 0)
    tv, _ = oracle.voxelize(tgt, p.voxel_size, 0)
    rec, st = oracle.register_pair(src, tgt, p)
    return dict(sv=sv, tv=tv, rec=rec, st=st)


@pytest.fixture(scope="module")
def gpu(hall):
    with Handle(**HANDLE_CFG) as h:
        yield h


@pytest.mark.gpu
def test_voxelize_hall_scan_bit_exact(gpu, hall, hall_ref):
    src, tgt, _ = hall
    for raw, ref in ((src, hall_ref["sv"]), (tgt, hall_ref["tv"])):
        got, st = gpu.voxelize(raw, 0.05, 0, cap=MAX_V)
        assert st == 0
        assert got.shape == ref.shape and got.tobytes() == ref.tobytes()
    assert len(hall_ref["sv"]) > 2 * 65536  # the new range: indices above 65535 in every per-point stage
    assert len(hall_ref["tv"]) > 65536


@pytest.mark.gpu
@pytest.mark.parametrize("radii", [(0.10, 0.15), (0.15, 0.30)], ids=["production", "wide"])
def test_fpfh_hall_cloud_bit_exact(gpu, hall_ref, oracle, radii):
    """Normals and FPFH-33 of the 134 k-point cloud.  The wide radius gives most points more neighbours than the K2c list holds
    (80), so the lattice-walking kernels (spfh_kernel<true>, fpfh_rare_kernel) handle points with indices above 65535."""
    pts = hall_ref["sv"]
    rn, rf = radii
    if rf > 0.2:
        from scipy.spatial import cKDTree
        cnt = np.array([len(x) for x in cKDTree(pts[:, :3].astype(np.float64)).query_ball_point(pts[65536:, :3], rf)])
        assert (cnt > 80).sum() > 20000, (cnt > 80).sum()
    n_got, d_got = gpu.compute_fpfh(pts, rn, rf, default_cell(rf))
    n_ref, d_ref = oracle.compute_fpfh(pts, rn, rf, default_cell(rf))
    assert same_bits(n_got, n_ref)
    assert same_bits(d_got, d_ref)


@pytest.fixture(scope="module")
def hall_features(hall_ref, oracle):
    p = indoor_params()
    _, sd = oracle.compute_fpfh(hall_ref["sv"], p.normal_radius, p.fpfh_radius, default_cell(p.fpfh_radius))
    _, td = oracle.compute_fpfh(hall_ref["tv"], p.normal_radius, p.fpfh_radius, default_cell(p.fpfh_radius))
    corr, nm, st = oracle.match(hall_ref["sv"], sd, hall_ref["tv"], td, p, cap=8192)
    return dict(sd=sd, td=td, corr=corr, nm=nm, st=st)


@pytest.mark.gpu
def test_match_hall_descriptors_tensor_core_path(gpu, hall_ref, hall_features):
    f = hall_features
    p = indoor_params()
    gpu.debug_match_stats()
    corr, nm, st = gpu.match(hall_ref["sv"], f["sd"], hall_ref["tv"], f["td"], p, cap=8192)
    stats = gpu.debug_match_stats()
    assert st == f["st"] and nm == f["nm"]
    assert np.array_equal(corr, f["corr"])
    assert stats["tiles"] > 0


@pytest.mark.gpu
def test_match_hall_descriptors_exact_kernel(hall_ref, hall_features, monkeypatch):
    """QB200_MATCH_EXACT=1: the CUDA-core kernel alone, its column minima folded with atomicMin into one [V] row per pair."""
    f = hall_features
    monkeypatch.setenv("QB200_MATCH_EXACT", "1")
    with Handle(**HANDLE_CFG) as h:
        corr, nm, st = h.match(hall_ref["sv"], f["sd"], hall_ref["tv"], f["td"], indoor_params(), cap=8192)
        stats = h.debug_match_stats()
    assert (nm, st) == (f["nm"], f["st"]) and stats["tiles"] == 0  # no tensor-core tile ran
    assert np.array_equal(corr, f["corr"])


@pytest.mark.gpu
def test_register_hall_pair_matches_the_oracle(gpu, hall, hall_ref):
    src, tgt, T = hall
    ref, st_ref = hall_ref["rec"], hall_ref["st"]
    got, st = gpu.register_pair(src, tgt, indoor_params())
    assert st == st_ref == 0 and got.valid == 1 == ref.valid
    assert_same_record(got, ref)
    assert got.n_src_vox > 65536 and got.n_tgt_vox > 65536 and got.n_corr > 4096
    rot, tr = synth.pose_error(got.matrix(), T)
    assert rot < 2.0 and tr < 0.3


@pytest.mark.gpu
def test_batch_and_cache_records_equal_single_calls(gpu, hall):
    """register_batch (two waves on a one-slot handle) and the scan cache reproduce the single-pair records byte for byte."""
    p = indoor_params()
    pairs = [hall[:2], synth.indoor_pair(2, **HALL)[:2]]
    single = np.frombuffer(b"".join(bytes(gpu.register_pair(s, t, p)[0]) for s, t in pairs), RESULT_DTYPE)
    assert (single["n_src_vox"] > 65536).all() and single["valid"][0] == 1
    batch = gpu.register_batch(pairs, p)
    assert batch.tobytes() == single.tobytes()
    gpu.cache_reserve(4)
    gpu.cache_scans([pairs[0][0], pairs[0][1], pairs[1][0], pairs[1][1]], [0, 1, 2, 3], p)
    cached = gpu.register_cached([[0, 1], [2, 3]], p)
    gpu.cache_reserve(0)
    assert cached.tobytes() == single.tobytes()


FIXTURE = "tests/fixtures/large_cloud_shim.cpp"


def test_large_cloud_shim_driver_compiles(tmp_path):
    build_against_lib(tmp_path, FIXTURE)


@pytest.mark.gpu
def test_cpp_shim_registers_the_hall_pair(tmp_path, hall, hall_ref):
    """voxelize / FPFHManager / Quatro grow their handles (500 k raw points, > 65536 voxel points, > 4096 correspondences)."""
    exe = build_against_lib(tmp_path, FIXTURE)
    src, tgt, T = hall
    (tmp_path / "src.bin").write_bytes(np.ascontiguousarray(src, np.float32).tobytes())
    (tmp_path / "tgt.bin").write_bytes(np.ascontiguousarray(tgt, np.float32).tobytes())
    r = subprocess.run([str(exe), str(tmp_path / "src.bin"), str(tmp_path / "tgt.bin")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "LARGE_CLOUD_SHIM_OK" in r.stdout, r.stdout + r.stderr
    out = {ln.split()[0]: ln.split()[1:] for ln in r.stdout.splitlines() if ln and not ln.startswith("T ")}
    T_cpp = np.array([list(map(float, ln.split()[1:])) for ln in r.stdout.splitlines() if ln.startswith("T ")])
    ref = hall_ref["rec"]
    assert list(map(int, out["raw"])) == [len(src), len(tgt)]
    assert list(map(int, out["voxels"])) == [ref.n_src_vox, ref.n_tgt_vox]
    assert int(out["corr"][0]) == ref.n_corr and int(out["clique"][0]) == ref.clique_size
    assert np.allclose(T_cpp, ref.matrix(), atol=1e-6)
    rot, tr = synth.pose_error(T_cpp, T)
    assert rot < 2.0 and tr < 0.3
