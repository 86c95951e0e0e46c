"""tc_nn_kernel starts every unique row and column from a seed: the exact distance to its nearest-norm candidates of the other
cloud (tc_seed_kernel, csrc/tc_match.cu).  A seed is only an upper bound, so both nearest-neighbour tables must still equal the
oracle's bit for bit when a seed ties the answer with a higher index, when it already is the answer, when every descriptor is
the same, at column counts around the 64-column tile, in a pair the exact kernel takes over, and at a large descriptor scale."""
import numpy as np
import pytest

from support import fpfh_like
from test_nn_tables import MU, _both_paths, _unit, fam_scaled, handles  # noqa: F401  (handles: the module's two matchers)

SEED_W = 16     # kSeedW: candidates on either side of a descriptor's norm


def fam_tie_beyond_seeds(rng, n=48, fill=40):
    """Row a has two columns at exactly distance 1: b_far = a + e_j (a'_j = 40, norm |a'|^2 + 81, LOWER index) and b_near = a + e_i
    (a'_i = 0, norm |a'|^2 + 1, the next column in norm order).  `fill` columns of norms in between, far from a, keep b_far out of
    the seed window: the seed is (1, b_near) and only the kernel's own evaluation finds the lowest-index answer (1, b_far)."""
    assert fill > SEED_W
    rows, far, near, fillers = [], [], [], []
    for k in range(n):
        a = MU.astype(np.float64).copy()
        a[0] = 40.0                                          # a'_0 = 40 (bin 0 is not centred)
        a[[1 + (k % 3), 7 + (k % 5)]] += rng.integers(1, 30, 2)  # distinct norms per row, integers keep every difference exact
        a[20 + (k % 4)] += 1.0 + k
        nrm = ((a - MU) ** 2).sum()
        bf, bn = a.copy(), a.copy()
        bf[0] += 1.0                                         # |b'|^2 = nrm + 2 * 40 + 1
        bn[33 - 1 - (k % 2) * 2] += 1.0                      # bins 32 / 30 of a' are 0: |b'|^2 = nrm + 1
        rows.append(a); far.append(bf); near.append(bn)
        t = np.sort(rng.uniform(2.0, 80.0, fill))
        fillers.append(MU + np.sqrt(nrm + t)[:, None] * _unit(rng, fill))
    A = np.array(rows, np.float32)
    B = np.concatenate([np.array(far), np.array(near), *fillers]).astype(np.float32)   # every b_far before every b_near
    return A, B


def fam_twins(rng, n=3000):
    """Every row has a column twin 1e-3 away, the nearest norm by far: the seed of almost every row and column is the answer."""
    A = fpfh_like(rng, n)
    B = (A[rng.permutation(n)] + rng.normal(0, 1e-3, (n, 33))).astype(np.float32)
    return A, B


@pytest.mark.gpu
def test_seed_ties_answer_with_higher_index(handles, oracle):
    A, B = fam_tie_beyond_seeds(np.random.default_rng(900))
    _both_paths(handles, oracle, A, B, "seed ties with a higher index (rows)")
    _both_paths(handles, oracle, B, A, "seed ties with a higher index (columns)")


@pytest.mark.gpu
def test_seed_is_the_answer(handles, oracle):
    A, B = fam_twins(np.random.default_rng(901))
    _both_paths(handles, oracle, A, B, "seeds are the answers")


@pytest.mark.gpu
def test_seed_every_descriptor_identical(handles, oracle):
    x = fpfh_like(np.random.default_rng(902), 2)
    for A, B, label in ((np.tile(x[0], (700, 1)), np.tile(x[0], (900, 1)), "one descriptor on both sides"),
                        (np.tile(x[0], (700, 1)), np.tile(x[1], (900, 1)), "one descriptor per side")):
        _both_paths(handles, oracle, A.astype(np.float32), B.astype(np.float32), label)


@pytest.mark.gpu
@pytest.mark.parametrize("nb", [1, 63, 64, 65])
def test_seed_column_counts(handles, oracle, nb):
    rng = np.random.default_rng(903 + nb)
    A, B = fpfh_like(rng, 700), fpfh_like(rng, nb)
    A[:nb] = (B + rng.normal(0, 0.05, B.shape)).astype(np.float32)
    _both_paths(handles, oracle, A, B, f"700 x {nb}")


@pytest.mark.gpu
def test_seed_pair_flagged_for_exact_kernel(handles, oracle):
    """A finite descriptor whose centred squared norm exceeds the tensor-core range: the pair is left unseeded and redone exactly."""
    rng = np.random.default_rng(904)
    A, B = fpfh_like(rng, 900), fpfh_like(rng, 1100)
    A[17] = 0
    A[17, 2] = 5e18
    B[40] = A[17]
    B[40, 12] = 2.0
    _both_paths(handles, oracle, A, B, "flagged pair")


@pytest.mark.gpu
def test_seed_fpfh_scale_2_8(handles, oracle):
    A, B = fam_scaled(np.random.default_rng(905), 8, 3000, 3500)
    _both_paths(handles, oracle, A, B, "fpfh x 2^8")
