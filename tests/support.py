"""Helpers several test modules share: point and descriptor builders, bit-exact float comparison, result-record comparison, the
params, handles, device copies and 0xA5-filled outputs of the batch tests, and the C++ build against libquatro_b200.  A plain module
(test files import it as `from support import ...`); fixtures live in conftest.py."""
import subprocess
from pathlib import Path

import numpy as np
import pytest

from quatro_b200.capi import MEM_HOST, Handle, default_params

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


def _host(a):
    """a numpy array as it is, a CUDA tensor copied to one."""
    return a if isinstance(a, np.ndarray) else a.cpu().numpy()


def host_lists(lists):
    """Per-pair lists with every CUDA tensor copied to a numpy array."""
    return [{k: _host(v) for k, v in d.items()} for d in lists]


def make_params(**kw):
    """capi.default_params() with the fields in kw set.  rot_noise_bound is 2 * noise_bound unless kw sets it: explicit, as the
    oracle has no latch; a test of the latch asks for it with rot_noise_bound=0."""
    p = default_params()
    p.rot_noise_bound = 2 * kw.get("noise_bound", p.noise_bound)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def make_handle(lanes, **cfg):
    """A Handle of config `cfg` with QB200_LANES=lanes, or unset (the default lane count) for lanes=None; the variable is read when
    the handle is created and restored after."""
    with pytest.MonkeyPatch.context() as mp:
        if lanes is None:
            mp.delenv("QB200_LANES", raising=False)
        else:
            mp.setenv("QB200_LANES", str(lanes))
        return Handle(**cfg)


def device_copy(a):
    """A CUDA copy of the host array a, in its own dtype, the copy finished."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    torch.cuda.synchronize()
    return t


def device_copies(arrays):
    """CUDA float32 copies of host point or descriptor arrays: their (pointer, count) tuples, and the tensors, which must outlive
    the pointers."""
    keep = [device_copy(np.asarray(a, np.float32)) for a in arrays]
    return [(t.data_ptr(), len(t)) for t in keep], keep


def sentinel(shape, dtype=np.float32, kind=MEM_HOST):
    """An output array of `shape` filled with 0xA5 bytes, which entries a call does not write keep: numpy for MEM_HOST, a CUDA
    tensor for MEM_DEVICE."""
    a = np.zeros(shape, dtype)
    a.view(np.uint8)[...] = 0xA5
    return a if kind == MEM_HOST else device_copy(a)


def sentinel_lists(lb):
    """ListBuffers lb with every byte of every array, host or device, set to 0xA5; returns lb."""
    for a in lb.arrays.values():
        if isinstance(a, np.ndarray):
            a.view(np.uint8)[...] = 0xA5
        else:
            import torch
            a.view(torch.uint8).fill_(0xA5)
    return lb


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
