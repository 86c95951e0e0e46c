"""The tuple test (match.cu tuple_test_kernel) draws r % ncorr through qb_fastmod (qb_math.cuh) and tests side 0 of both triangles
before sides 1 and 2.  The CPU test checks the reduction against % for edge and random values; the GPU tests check the marks, through
the correspondences they leave, against the CPU oracle (which draws with %) around the shared-memory staging limit of 4096
mutual pairs, with per-pair scales and seeds, and with the test switched off."""
import subprocess

import numpy as np
import pytest

from quatro_b200 import synth
from quatro_b200.capi import ListBuffers, default_params
from support import P4, ROOT, assert_same_record, fpfh_like

DIVISORS = [1, 2, 3, 5, 7, 1535, 1536, 1537, 4095, 4096, 4097, 32767, 32768, 65535, 65536, 262144, 1000003, (1 << 31) - 1, 1 << 31, (1 << 31) + 1,
            (1 << 32) - 2, (1 << 32) - 1]


def test_fastmod_equals_remainder(tmp_path):
    rng = np.random.default_rng(17)
    divisors = DIVISORS + [int(d) for d in rng.integers(1, 1 << 32, 40, dtype=np.uint64)] + [(1 << k) + o for k in range(1, 32) for o in (-1, 1)]
    src = tmp_path / "fastmod.cpp"
    src.write_text(f"""
#define QB_HD
#include <stdio.h>
#include "qb_math.cuh"
static uint64_t s = 0x9E3779B97F4A7C15ull;
static uint32_t next() {{ s ^= s << 13; s ^= s >> 7; s ^= s << 17; return (uint32_t)(s >> 32); }}
int main() {{
  const uint64_t ds[] = {{{", ".join(f"{d}ull" for d in divisors)}}};
  long long checked = 0, bad = 0;
  for (uint64_t dd : ds) {{
    const uint32_t d = (uint32_t)dd;
    const uint64_t m = qb_fastmod_magic(d);
    auto check = [&](uint32_t r) {{ ++checked; if (qb_fastmod(r, m, d) != r % d) {{ if (bad < 5) printf("r=%u d=%u\\n", r, d); ++bad; }} }};
    for (uint32_t r = 0; r < 4096; ++r) {{ check(r); check(0xFFFFFFFFu - r); }}
    for (uint64_t k = 1; k * d <= 0xFFFFFFFFull && k < 4096; ++k) {{ check((uint32_t)(k * d - 1)); check((uint32_t)(k * d)); check((uint32_t)(k * d + 1)); }}
    const uint64_t top = 0xFFFFFFFFull / d * d;
    for (int o = -2; o <= 2; ++o) check((uint32_t)(top + o));
    for (int i = 0; i < 200000; ++i) check(next());
  }}
  printf("%lld %lld\\n", checked, bad);
  return 0;
}}
""")
    exe = tmp_path / "fastmod"
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", f"-I{ROOT / 'quatro_b200' / 'csrc'}", "-o", str(exe), str(src)], check=True)
    checked, bad = map(int, subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()[-2:])
    assert bad == 0 and checked > 200000 * len(divisors)


def _matched_scene(n, seed):
    """n points and a moved copy (every 7th point displaced) with the same, distinct descriptors: exactly n mutual pairs."""
    rng = np.random.default_rng(seed)
    src = rng.uniform(-25, 25, (n, 3))
    yaw = 0.4
    R = np.array([[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]])
    tgt = src @ R.T + [2.0, -1.0, 0.3] + rng.normal(0, 0.02, (n, 3))
    tgt[::7] += rng.uniform(-6, 6, (len(tgt[::7]), 3))
    perm = rng.permutation(n)
    desc = fpfh_like(rng, n)
    return P4(src), desc, P4(tgt[perm]), desc[perm].copy()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 3, 1536, 4095, 4096, 4097])
def test_tuple_marks_equal_oracle_around_the_staging_limit(oracle, n):
    from quatro_b200.capi import Handle
    a, ad, b, bd = _matched_scene(n, 500 + n)
    handle = Handle(max_batch_slots=2, max_corr=8192)      # room for every mutual pair of the largest scene
    params = [default_params()]
    p = default_params(); p.tuple_scale = 0.8; p.seed = 99; params.append(p)
    p = default_params(); p.tuple_scale = 0.97; p.tuple_trials_per_corr = 7; p.seed = 3; params.append(p)
    p = default_params(); p.use_tuple_test = 0; params.append(p)
    for k, prm in enumerate(params):
        for x, xd, y, yd in ((a, ad, b, bd), (b, bd, a, ad)):
            c_ref, nm_ref, _ = oracle.match(x, xd, y, yd, prm)
            c_got, nm_got, st = handle.match(x, xd, y, yd, prm)
            assert st == 0 and nm_got == nm_ref == n, (k, nm_got, nm_ref)
            assert np.array_equal(c_got, c_ref), (k, len(c_got), len(c_ref))
        if prm.use_tuple_test and prm.tuple_scale >= 0.95 and n > 3:
            assert 0 < len(c_ref) < n, k      # the test really rejects some pairs and keeps others
    handle.close()


@pytest.mark.gpu
def test_mixed_tuple_parameters_in_one_wave(oracle):
    from quatro_b200.capi import Handle
    pairs = [synth.outdoor_pair(s, rings=32, azimuths=900)[:2] for s in range(40, 46)]
    params = []
    for scale, seed, use in ((0.95, 1, 1), (0.9, 2, 1), (0.97, 3, 1), (0.95, 4, 0), (0.85, 5, 1), (0.95, 6, 1)):
        p = default_params()
        p.tuple_scale, p.seed, p.use_tuple_test = scale, seed, use
        p.rot_noise_bound = 2 * p.noise_bound
        params.append(p)
    with Handle(max_batch_slots=len(pairs)) as h:
        recs, _ = h.register_batch_mixed(pairs, params, buffers=ListBuffers(len(pairs), h.cfg.max_corr))
    for (src, tgt), r, p in zip(pairs, recs, params):
        ref, st = oracle.register_pair(src, tgt, p)
        assert r["status"] == st
        assert_same_record(r, ref)
