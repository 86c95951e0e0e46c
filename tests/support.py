"""Helpers several test modules share: point and descriptor builders, bit-exact float comparison, result-record comparison and the
C++ build against libquatro_b200.  A plain module (test files import it as `from support import ...`); fixtures live in conftest.py."""
import subprocess
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent


def P4(xyz, w=1.0):
    """n x {x, y, z, w} float32 records from n x 3 coordinates."""
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    out = np.full((len(xyz), 4), w, np.float32)
    out[:, :3] = xyz
    return out


def fpfh_like(rng, n):
    """n x 33 descriptors shaped like FPFH-33: three 11-bin histograms of sparse (gamma 0.3) mass, each summing to 100."""
    d = rng.gamma(0.3, 1.0, (n, 33)).astype(np.float32)
    for t in range(3):
        d[:, 11 * t:11 * t + 11] *= 100.0 / np.maximum(d[:, 11 * t:11 * t + 11].sum(1, keepdims=True), 1e-6)
    return d.astype(np.float32)


def same_bits(a, b, nan_equal=False):
    """Same shape and bit-identical float32 values.  nan_equal: any NaN matches any NaN (the normals of points with too few
    neighbours are NaN, and their payload is not part of the result)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    if a.shape != b.shape:
        return False
    eq = a.view(np.uint32) == b.view(np.uint32)
    if nan_equal:
        eq |= np.isnan(a) & np.isnan(b)
    return bool(eq.all())


RECORD_FIELDS = ("valid", "status", "n_src_vox", "n_tgt_vox", "n_mutual", "n_corr", "n_edges", "max_core", "clique_size", "gnc_iters",
                 "n_rot_inliers", "n_final_inliers", "flags")


def assert_same_record(got, ref):
    """Two result records of one pair (capi.Result or a row of a RESULT_DTYPE array): every counter equal, poses within 1e-9."""
    def field(r, k):
        return r[k] if isinstance(r, np.void) else getattr(r, k)

    def pose(r):
        return np.asarray(r["T"]).reshape(4, 4).T if isinstance(r, np.void) else r.matrix()

    for k in RECORD_FIELDS:
        assert field(got, k) == field(ref, k), (k, field(got, k), field(ref, k))
    assert np.allclose(pose(got), pose(ref), atol=1e-9, rtol=0)


def same_lists(got: dict, want: dict):
    """One pair's lists (dicts of arrays by list name): every list of `want` has the same shape and bytes in `got`."""
    for name in want:
        g, w = np.asarray(got[name]), np.asarray(want[name])
        assert g.shape == w.shape and g.tobytes() == w.tobytes(), (name, g.shape, w.shape)


def host_lists(lists):
    """Per-pair lists with every CUDA tensor copied to a numpy array."""
    return [{k: (v if isinstance(v, np.ndarray) else v.cpu().numpy()) for k, v in d.items()} for d in lists]


def build_against_lib(tmp_path, source):
    """Compile the C++ file `source` (relative to the repository root) against include/ and link it to libquatro_b200, warnings as
    errors; returns the executable."""
    from quatro_b200 import _build
    lib = _build.build_cuda()
    exe = tmp_path / Path(source).stem
    cmd = ["/usr/bin/g++", "-std=c++17", "-Wall", "-Werror", f"-I{ROOT / 'include'}", str(ROOT / source),
           f"-L{lib.parent}", "-lquatro_b200", f"-Wl,-rpath,{lib.parent}", "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe
