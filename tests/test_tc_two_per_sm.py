"""The tensor-core nearest-neighbour kernel (tc_nn_kernel, csrc/tc_match.cu) is sized so that two CTAs share an SM:
one CTA's wgmma runs while the other filters and evaluates.  That needs <= 96 registers per thread at 320 threads, no
local memory, and at most about 112 KB of shared memory per CTA.  The CPU test reads the compiled resource usage; the
GPU tests check the occupancy the runtime reports and the results at the 64-column tile boundaries."""
import re
import subprocess

import numpy as np
import pytest

from quatro_b200 import _build
from support import P4, fpfh_like

DYN_SMEM = 100 * 1024        # A block (60 KB) + one operand stage (20 KB) + two exact-image stages (2 x 10 KB)
SM_SMEM = 228 * 1024         # shared memory of an H100 SM
CTA_RESERVED = 1024          # shared memory the system reserves per CTA


def _res_usage(kernel_prefix):
    lib = _build.CUDA_LIB
    assert lib.exists(), f"{lib} is missing: run __graft_entry__.build() first"
    out = subprocess.run([_build.cuda_tool("cuobjdump"), "-res-usage", str(lib)], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    for i, line in enumerate(lines):
        if line.strip().startswith("Function " + kernel_prefix):
            fields = dict(re.findall(r"(\w+(?:\[\d+\])?):(\d+)", lines[i + 1]))
            return {k: int(v) for k, v in fields.items()}
    raise AssertionError(f"{kernel_prefix} not found in cuobjdump -res-usage of {lib}")


def test_tc_nn_kernel_fits_two_ctas_per_sm():
    # tc_nn_kernel<false, false>: the production instance
    use = _res_usage("_ZN2qb12tc_nn_kernelILb0ELb0E")
    assert use["REG"] <= 96, use
    assert use["LOCAL"] == 0 and use["STACK"] == 0, use       # no spills
    assert 2 * (DYN_SMEM + use["SHARED"] + CTA_RESERVED) <= SM_SMEM, use


@pytest.mark.gpu
def test_tc_footprint_two_ctas_per_sm(handle):
    fp = handle.debug_tc_footprint()
    assert fp["threads"] == 320 and fp["dyn_smem"] == DYN_SMEM, fp
    assert fp["regs"] <= 96, fp
    assert fp["ctas_per_sm"] == 2, fp


@pytest.mark.gpu
@pytest.mark.parametrize("na", [1, 63, 64, 65, 127, 128, 129])
def test_match_at_tile_boundaries(handle, oracle, na):
    """Column counts around the 64-column tile edge and row counts that leave the second warpgroup of the last stripe
    empty or half filled: the padding must never compete and every real entry must be found."""
    from quatro_b200.capi import default_params
    p = default_params()
    p.use_tuple_test = 0
    rng = np.random.default_rng(1000 + na)
    for nb in (1, 63, 64, 65, 127, 128, 129, 191):
        a, b = P4(rng.uniform(-20, 20, (na, 3))), P4(rng.uniform(-20, 20, (nb, 3)))
        ad, bd = fpfh_like(rng, na), fpfh_like(rng, nb)
        k = min(na, nb) // 3
        bd[:k] = ad[:k]                                   # exact duplicates -> zero distances and lowest-index ties
        ad[na - 1] = 0.0                                  # an isolated point: looks like the zero padding
        ref = oracle.match(a, ad, b, bd, p)
        got = handle.match(a, ad, b, bd, p)
        assert np.array_equal(got[0], ref[0]) and got[1] == ref[1], (na, nb)
