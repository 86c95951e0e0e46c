#!/usr/bin/env python3
"""Probe of the tensor-core distance tile (qb200_debug_tc_distances): structured inputs that reveal row/column/K mapping."""
import sys
from pathlib import Path
import numpy as np
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from quatro_b200.capi import Handle

np.set_printoptions(linewidth=220, precision=3, suppress=True)
h = Handle(max_batch_slots=2)


def dots(a, b):
    got = h.debug_tc_distances(a, b).astype(np.float64)
    na = (a.astype(np.float64) ** 2).sum(1)[:, None]
    nb = (b.astype(np.float64) ** 2).sum(1)[None, :]
    return (na + nb - got) / 2.0, got


# probe 1: row / column mapping.  a_i = (i+1) e_0,  b_j = (j+1) e_0  ->  dot = (i+1)(j+1)
a = np.zeros((128, 33), np.float32); b = np.zeros((128, 33), np.float32)
a[:, 0] = np.arange(1, 129); b[:, 0] = np.arange(1, 129)
d, got = dots(a, b)
ref = np.outer(np.arange(1, 129), np.arange(1, 129)).astype(np.float64)
print("probe1 max|dot-ref| =", np.abs(d - ref).max())
print("dot[:6,:6]=\n", d[:6, :6]); print("ref[:6,:6]=\n", ref[:6, :6])
print("dot[30:36,30:36]=\n", d[30:36, 30:36])
print("dot[0, ::16] =", d[0, ::16], " dot[::16, 0] =", d[::16, 0])
# probe 2: K mapping.  a_i = e_{i % 33},  b_j[d] = d + 1  ->  dot(i,j) = (i % 33) + 1
a = np.zeros((128, 33), np.float32); a[np.arange(128), np.arange(128) % 33] = 1.0
b = np.tile(np.arange(1, 34, dtype=np.float32), (128, 1))
d, got = dots(a, b)
print("probe2 dot[:40, 0] =", d[:40, 0])
# probe 3: random
rng = np.random.default_rng(0)
a = rng.uniform(0, 30, (128, 33)).astype(np.float32); b = rng.uniform(0, 30, (128, 33)).astype(np.float32)
d, got = dots(a, b)
ref = a.astype(np.float64) @ b.astype(np.float64).T
print("probe3 max|dot-ref| =", np.abs(d - ref).max(), " rel to |ref|max", np.abs(d - ref).max() / np.abs(ref).max())
print("probe3 corrcoef", np.corrcoef(d.ravel(), ref.ravel())[0, 1], " vs transposed", np.corrcoef(d.ravel(), ref.T.ravel())[0, 1])
