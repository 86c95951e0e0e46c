"""The C++ drop-in layer (include/quatro_b200/quatro.hpp, fpfh_manager.hpp) and the ROS-free mirror of the
reference's example: compiles and links on the CPU box; on the GPU box it runs and must reproduce the oracle."""
import re
import subprocess

import numpy as np
import pytest

from support import ROOT, build_against_lib

EXAMPLE = "examples/run_global_registration.cpp"


def test_example_compiles_against_the_shim(tmp_path):
    exe = build_against_lib(tmp_path, EXAMPLE)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr


def test_shim_keeps_the_reference_surface():
    """Names the reference's caller relies on (examples/run_global_registration.cpp:103-108,206-221,243-246,290-292)."""
    q = (ROOT / "include" / "quatro_b200" / "quatro.hpp").read_text()
    f = (ROOT / "include" / "quatro_b200" / "fpfh_manager.hpp").read_text()
    for name in ["class Quatro", "struct Params", "void reset(const Params", "setInputSource", "setInputTarget",
                 "void computeTransformation(Eigen::Matrix4d& output)", "getMaxCliques", "getFinalInliers", "getFinalInliersIndices",
                 "getNumRotaionInliers", "getNumMaxCliqueInliers", "setPreEstaimatedRyRx", "INLIER_SELECTION_MODE", "PMC_HEU",
                 "rotation_gnc_factor", "rotation_cost_threshold", "noise_bound_", "void voxelize("]:
        assert name in q, name
    for name in ["class FPFHManager", "flushAllFeatures", "setFeaturePair", "getSrcKps", "getTgtKps", "getSrcMatched", "getCorrespondences",
                 "getObjDescriptor", "getSceneDescriptor", "getTgtNormals", "swapTgt2Src", "saveFeaturePair", "loadFeaturePair", "setLoadDir",
                 "setSaveDir", "clearInputs", "setParams"]:
        assert name in f, name


def test_preprocessing_shims_keep_the_reference_surface():
    """examples/run_global_registration.cpp:124-162 of the reference: PatchWork<PointT>::estimate_ground, ImageProjection."""
    pw = (ROOT / "include" / "quatro_b200" / "patchwork.hpp").read_text()
    ip = (ROOT / "include" / "quatro_b200" / "imageProjection.hpp").read_text()
    for name in ["class PatchWork", "void estimate_ground(const pcl::PointCloud<PointT>& cloud_in, pcl::PointCloud<PointT>& cloud_out",
                 "check_input_parameters_are_correct"]:
        assert name in pw, name
    for name in ["class ImageProjection", "void segmentCloud(", "getValidSegments", "getOutliers", "Velodyne-64-HDE", "VLP-16", "HDL-32E",
                 "Ouster-OS1-16", "Ouster-OS1-64", "4CrossNeighbor", "N_SCAN", "Horizon_SCAN"]:
        assert name in ip, name


@pytest.mark.gpu
def test_example_with_preprocessing_reproduces_the_oracle(tmp_path, oracle):
    """--preprocess: PatchWork + ImageProjection through the C++ shim in front of the path, against the oracle's chain."""
    from quatro_b200 import synth
    from quatro_b200.capi import default_params, default_patchwork_params, default_segment_params
    exe = build_against_lib(tmp_path, EXAMPLE)
    src, tgt, T = synth.outdoor_pair(2)
    src[:, 3] = 1.0; tgt[:, 3] = 1.0                  # the .bin loader drops the 4th channel anyway
    (tmp_path / "src.bin").write_bytes(src.astype(np.float32).tobytes())
    (tmp_path / "tgt.bin").write_bytes(tgt.astype(np.float32).tobytes())
    r = subprocess.run([str(exe), str(tmp_path / "src.bin"), str(tmp_path / "tgt.bin"), "--preprocess"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    T_cpp = np.array([list(map(float, ln.split()[1:])) for ln in r.stdout.splitlines() if re.match(r"^T ", ln)])
    pp, sp = default_patchwork_params(), default_segment_params()
    chain = lambda c: oracle.segment_cloud(oracle.patchwork(c, pp)[1], sp)[0]
    cs, ct = chain(src), chain(tgt)
    m = re.search(r"# of valid segments\s+\| (\d+) \| (\d+)", r.stdout)
    assert m and (int(m.group(1)), int(m.group(2))) == (len(cs), len(ct))
    p = default_params()
    sv, _ = oracle.voxelize(cs, 0.3, 0)
    tv, _ = oracle.voxelize(ct, 0.3, 0)
    corr, sm, tm, _ = oracle.match_and_pack(sv, tv, p)
    ref, st = oracle.solve_correspondences(sm, tm, p)
    assert st == 0 and f"# after voxelization | {len(sv)} | {len(tv)}" in r.stdout
    assert np.allclose(T_cpp, ref.matrix(), atol=1e-6)


@pytest.mark.gpu
def test_example_reproduces_the_oracle(tmp_path, oracle):
    from quatro_b200 import synth
    from quatro_b200.capi import default_params
    exe = build_against_lib(tmp_path, EXAMPLE)
    src, tgt, T = synth.outdoor_pair(1)
    src, tgt = src[src[:, 3] > 0], tgt[tgt[:, 3] > 0]      # the example has no ground filter: hand it the non-ground returns
    (tmp_path / "src.bin").write_bytes(src.astype(np.float32).tobytes())
    (tmp_path / "tgt.bin").write_bytes(tgt.astype(np.float32).tobytes())
    r = subprocess.run([str(exe), str(tmp_path / "src.bin"), str(tmp_path / "tgt.bin")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    rows = [list(map(float, ln.split()[1:])) for ln in r.stdout.splitlines() if re.match(r"^T ", ln)]
    T_cpp = np.array(rows)
    p = default_params()
    sv, _ = oracle.voxelize(src, 0.3, 0)
    tv, _ = oracle.voxelize(tgt, 0.3, 0)
    corr, sm, tm, _ = oracle.match_and_pack(sv, tv, p)
    ref, st = oracle.solve_correspondences(sm, tm, p)
    assert st == 0
    assert f"# after voxelization | {len(sv)} | {len(tv)}" in r.stdout and f"# after matching     | {len(corr)} | {len(corr)}" in r.stdout
    assert np.allclose(T_cpp, ref.matrix(), atol=1e-6)
    rot, tr = synth.pose_error(T_cpp, T)
    assert rot < 2.0 and tr < 0.5


def test_shim_extras_compile(tmp_path):
    build_against_lib(tmp_path, "tests/fixtures/shim_extras.cpp")


@pytest.mark.gpu
def test_fpfh_manager_getters_odometry_and_pcd_cache(tmp_path):
    from quatro_b200 import synth
    exe = build_against_lib(tmp_path, "tests/fixtures/shim_extras.cpp")
    a, b, _ = synth.outdoor_pair(11, rings=32, azimuths=900)
    c, _, _ = synth.outdoor_pair(12, rings=32, azimuths=900)
    names = []
    for i, sc in enumerate((a, b, c)):
        sc = sc[sc[:, 3] > 0]
        f = tmp_path / f"s{i}.bin"
        f.write_bytes(sc.astype(np.float32).tobytes())
        names.append(str(f))
    r = subprocess.run([str(exe), *names, str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "SHIM_EXTRAS_OK" in r.stdout, r.stdout + r.stderr
    assert (tmp_path / "000540_to_001319.pcd").exists()
