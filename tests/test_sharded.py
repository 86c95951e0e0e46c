"""N > 1 path: shard assignment + result gather.  CPU: world_size-2 gloo run of the host logic.
GPU (needs >= 2 devices): the same pairs registered on 2 ranks must be bit-identical to 1 rank."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


def test_shard_indices_partition():
    from quatro_b200.sharded import shard_indices
    for n in (0, 1, 7, 8, 2048):
        for w in (1, 2, 3, 8):
            parts = [shard_indices(n, r, w) for r in range(w)]
            assert sorted(np.concatenate(parts).tolist()) == list(range(n))
            assert max(map(len, parts)) - min(map(len, parts)) <= 1


def _torchrun(nproc, args, port):
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(ROOT / "tools" / "sharded_check.py"), *args]
    return subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)


def test_gather_with_gloo_world2():
    r = _torchrun(2, ["7", "gloo"], 29611)
    assert r.returncode == 0 and "IDENTICAL" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_two_gpus_match_one_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = _torchrun(2, ["6", "nccl"], 29612)
    assert r.returncode == 0 and "IDENTICAL" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_two_gpus_c_abi_gather_matches_one_gpu():
    """qb200_comm_init_rank + qb200_register_batch_rank (ncclAllGather inside the C++ library, deferred) on 2 ranks."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = _torchrun(2, ["6", "nccl", "cabi"], 29613)
    assert r.returncode == 0 and "IDENTICAL" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_c_abi_comm_on_every_visible_gpu():
    """(A) single process: qb200_comm_init_all + qb200_register_batch_sharded over all visible devices (1 on the driver's box: the
    all-gather degenerates but the whole code path -- dlopen of libnccl, staging, grouped collective, reorder -- runs);
    (B) world = 1: qb200_comm_unique_id + qb200_comm_init_rank + deferred qb200_register_batch_rank.  Records must be byte-identical
    to qb200_register_batch on one handle."""
    import torch
    from quatro_b200 import synth
    from quatro_b200.capi import Handle, Pair, default_params, comm_init_all, register_batch_sharded, MEM_HOST, RESULT_DTYPE
    n_dev = min(torch.cuda.device_count(), 4)
    p = default_params()
    pairs = [synth.outdoor_pair(60 + i, rings=32, azimuths=900)[:2] for i in range(5)]
    with Handle(max_batch_slots=4) as h0:
        ref = h0.register_batch(pairs, p)
        # (B) world 1
        h0.comm_init_rank(1, 0, Handle.comm_unique_id())
        arr = (Pair * len(pairs))()
        for k, (s, t) in enumerate(pairs):
            arr[k].src, arr[k].n_src, arr[k].tgt, arr[k].n_tgt = s.ctypes.data, len(s), t.ctypes.data, len(t)
        out = np.zeros(len(pairs), RESULT_DTYPE)
        h0.register_batch_rank_raw(arr, len(pairs), p, MEM_HOST, out, defer=True)
        h0.comm_wait()
        assert out.tobytes() == ref.tobytes()
        # pipelined stream of batches (defer = 2): three batches in flight, separate record arrays, one comm_wait at the end
        outs = [np.zeros(len(pairs), RESULT_DTYPE) for _ in range(3)]
        for o in outs:
            h0.register_batch_rank_raw(arr, len(pairs), p, MEM_HOST, o, defer=2)
        h0.comm_wait()
        for o in outs:
            assert o.tobytes() == ref.tobytes()
        out[:] = 0
        h0.register_batch_rank_raw(arr, len(pairs), p, MEM_HOST, out, defer=2)   # a single queued batch, then the blocking form
        out2 = np.zeros(len(pairs), RESULT_DTYPE)
        h0.register_batch_rank_raw(arr, len(pairs), p, MEM_HOST, out2, defer=0)
        assert out.tobytes() == ref.tobytes() and out2.tobytes() == ref.tobytes()
    hs = [Handle(device=d, max_batch_slots=4) for d in range(n_dev)]
    try:
        comm_init_all(hs)
        got = register_batch_sharded(hs, pairs, p, MEM_HOST)
        assert got.tobytes() == ref.tobytes()
        got2 = register_batch_sharded(hs, pairs[:3], p, MEM_HOST)     # uneven shards, staging reuse
        assert got2.tobytes() == ref[:3].tobytes()
    finally:
        for h in hs:
            h.close()
