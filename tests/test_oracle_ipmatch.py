"""The matching oracle (oracle/vw_ipmatch_oracle.c) pinned by the reference's TestMatcher.cxx known answers and checked bit
for bit against the numpy restatement in ipmatch_reference.py: random sets, ties and duplicates, polarity mixes, every
threshold class, non-finite values, the Hamming byte chunking and remove_duplicates."""
import numpy as np
import pytest

import ipmatch_reference as ref
from oracle import ipmatch as om

THRESHOLDS = (0.0, 0.5, 0.8, 1.0, np.inf, np.nan)


def same(a, b):
    return a[0].tolist() == b[0].tolist() and np.array_equal(a[1], b[1], equal_nan=True) and np.array_equal(a[2], b[2], equal_nan=True)


def test_known_answers():
    """TestMatcher.cxx: DistanceMetric (L2 16, Hamming 4 and 20) and the Matcher case through the Simple matcher"""
    assert om.l2([0, 1, 0], [0, 5, 0]) == 16
    assert om.hamming([1, 2, 3], [0, 0, 0]) == 4
    assert om.hamming([1, 2, 3] * 5, [0] * 15) == 20
    idx, f, s = om.match([[0, 7.7, 0]], [0], [[0, 5, 0], [0, 6, 0], [0, 7, 0], [0, 8, 0], [0, 9, 0]], [0] * 5, 0.5)
    assert idx.tolist() == [3]
    assert f[0] == float(np.float32(np.float32(7.7) - 8) ** 2) and s[0] == float(np.float32(np.float32(7.7) - 7) ** 2)


def sets(seed, n1, n2, dim, dup=False, pol="mix"):
    rng = np.random.default_rng(seed)
    d1 = rng.normal(0, 1, (n1, dim)).astype(np.float32)
    d2 = rng.normal(0, 1, (n2, dim)).astype(np.float32)
    if dup and n2 > 2:
        d2[1::3] = d2[0::3][: len(d2[1::3])]                       # equal candidates: ties and first == second
        d1[: min(n1, n2)] = d2[: min(n1, n2)]                      # zero distances
    p1 = rng.random(n1) < 0.5 if pol == "mix" else np.zeros(n1, bool)
    p2 = rng.random(n2) < 0.5 if pol == "mix" else np.zeros(n2, bool)
    return d1, p1, d2, p2


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("thr", THRESHOLDS)
def test_l2_random_matches_reference(seed, thr):
    d1, p1, d2, p2 = sets(seed, 12, 17, (1, 3, 15, 20)[seed], dup=seed % 2 == 1, pol=("mix", "one")[seed % 2])
    assert same(om.match(d1, p1, d2, p2, thr), ref.match(d1, p1, d2, p2, thr))


@pytest.mark.parametrize("case", ["inf", "nan", "overflow", "neg_inf_pair"])
def test_l2_non_finite_matches_reference(case):
    d1, p1, d2, p2 = sets(9, 10, 14, 6)
    if case == "inf":
        d2[2, 1] = np.inf
        d1[3, 0] = -np.inf
    elif case == "nan":
        d2[4, 5] = np.nan
        d1[0, 2] = np.nan
    elif case == "overflow":
        d2[5, 0] = 3e38                                            # finite, but the square overflows to inf
        d1[1, :] = 2e19
    else:
        d1[2, 0], d2[6, 0] = np.inf, np.inf                        # inf - inf = NaN after the first term
        d2[6, 3] = np.nan
    assert same(om.match(d1, p1, d2, p2, 0.8), ref.match(d1, p1, d2, p2, 0.8))
    assert same(om.match(d1, p1, d2, p2, 1.0), ref.match(d1, p1, d2, p2, 1.0))


def test_l2_break_freezes_at_inf():
    """the break: once dist is inf a later NaN term is not added"""
    assert om.l2([3e38, np.nan], [-3e38, 0]) == np.inf
    assert ref.l2([3e38, np.nan], [-3e38, 0]) == np.inf
    assert np.isnan(om.l2([np.nan, 3e38], [0, -3e38]))


@pytest.mark.parametrize("dim", [1, 3, 4, 7, 8, 13, 32, 33])
def test_hamming_matches_reference(dim):
    rng = np.random.default_rng(dim)
    d1 = rng.uniform(-0.99, 255.99, (9, dim)).astype(np.float32)
    d2 = rng.integers(0, 256, (11, dim)).astype(np.float32)
    d1[0, 0], d2[1, -1] = 255.9, -0.5
    p1, p2 = rng.random(9) < 0.3, rng.random(11) < 0.3
    for thr in (0.5, 1.0):
        assert same(om.match(d1, p1, d2, p2, thr, om.HAMMING), ref.match(d1, p1, d2, p2, thr, "hamming"))
    for i in range(9):
        for j in range(11):
            assert om.hamming(d1[i], d2[j]) == ref.hamming(d1[i], d2[j])


def test_hamming_rejects_non_byte_values():
    d = np.zeros((3, 5), np.float32)
    for v, where in ((256.0, (1, 2, 3)), (-1.0, (0, 1, 4)), (np.nan, (0, 0, 0))):
        a, b = d.copy(), d.copy()
        (a if where[0] == 0 else b)[where[1], where[2]] = v
        with pytest.raises(om.BadByteValue) as e:
            om.match(a, [0] * 3, b, [0] * 3, 0.5, om.HAMMING)
        assert e.value.where == where


def test_edge_cases():
    z = np.zeros((0, 4), np.float32)
    one = np.ones((1, 4), np.float32)
    assert om.match(z, [], one, [0])[0].size == 0
    idx, f, s = om.match(one, [0], z, [])
    assert idx.tolist() == [-1] and f[0] == s[0] == 1e100
    idx, f, s = om.match(np.zeros((2, 0)), [0, 0], np.zeros((3, 0)), [0, 1, 0])          # D = 0: every distance 0
    assert idx.tolist() == [0, 0] and f.tolist() == [0.0, 0.0] and s.tolist() == [0.0, 0.0]
    idx, f, s = om.match(one, [1], one * 2, [1])                                         # a single candidate
    assert idx.tolist() == [0] and f[0] == 4.0 and s[0] == 1e100
    idx, _, _ = om.match(one, [1], one * 2, [0])                                         # no candidate of its polarity
    assert idx.tolist() == [-1]


@pytest.mark.parametrize("seed", range(3))
def test_remove_duplicates_matches_reference(seed):
    rng = np.random.default_rng(seed)
    xy1 = rng.integers(0, 6, (200, 2)).astype(np.float32)
    xy2 = rng.integers(0, 9, (200, 2)).astype(np.float32)
    xy1[rng.random(200) < 0.2] *= -1                                                     # -0.0 beside 0.0
    assert om.remove_duplicates(xy1, xy2).tolist() == ref.remove_duplicates(xy1, xy2).tolist()
    with pytest.raises(om.OracleError):
        xy1[7, 1] = np.nan
        om.remove_duplicates(xy1, xy2)
