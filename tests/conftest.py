import os
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: pytest -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import Oracle
    return Oracle()


@pytest.fixture(scope="session")
def params():
    from quatro_b200.capi import default_params
    return default_params()


@pytest.fixture(scope="session")
def handle():
    """CUDA handle through the C-ABI.  Fails loudly (no CPU fallback) if the library or device is missing."""
    from quatro_b200.capi import Handle
    h = Handle(max_batch_slots=8)
    yield h
    h.close()


def adj_to_dense(adj, L):
    bits = np.unpackbits(adj.view(np.uint8), axis=1, bitorder="little")[:, :L]
    return bits.astype(bool)


def dense_to_adj(A):
    L = A.shape[0]
    wpr = (L + 31) // 32
    pad = np.zeros((L, wpr * 32), np.uint8)
    pad[:, :L] = A
    return np.packbits(pad, axis=1, bitorder="little").view(np.uint32).reshape(L, wpr).copy()
