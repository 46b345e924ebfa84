"""The oracle's calc_disparity (oracle/vw_oracle.c, the reference's sliding double box sums) against a plain float64
brute force on the imagery of tests/test_gpu_value_domain.py: signed rasters holding -0.0, binary textures at the range
limits (Sq window sums above 2^31, zone-int keys just below 2^32), magnitudes near 1e6 and 3e7, NCC.  The GPU tests compare
with the oracle bit for bit; this pins the oracle itself on inputs its known-answer tests do not reach."""
import numpy as np
import pytest

from bm_reference import brute_calc_disparity
from test_gpu_value_domain import make_pair


A1 = dict(lo=0, hi=2047, halves=True, negzero=True)
A1_LOW = dict(lo=0, hi=3, halves=True, noise=2, negzero=True)
CASES = [  # id, cost, (W, H), search, kernel, make_pair keywords
    ("a1-abs", 0, (60, 40), (12, 9), (9, 9), A1),
    ("a1-sq", 1, (60, 40), (12, 9), (9, 9), A1),
    ("a1-ncc", 2, (60, 40), (12, 9), (9, 9), A1),
    ("a1-low-abs", 0, (60, 40), (12, 9), (9, 9), A1_LOW),
    ("a1-low-sq", 1, (60, 40), (12, 9), (9, 9), A1_LOW),
    ("a1-low-ncc", 2, (60, 40), (12, 9), (9, 9), A1_LOW),
    ("a2-abs", 0, (60, 40), (12, 9), (9, 9), dict(lo=-8192, hi=-1, negzero=True)),
    ("b1-abs-8191-k31x41", 0, (50, 30), (12, 9), (31, 41), dict(lo=0, hi=8191, texture="binary")),
    ("b1-abs-8192-k21", 0, (60, 40), (12, 9), (21, 21), dict(lo=-4096, hi=4096, texture="binary")),
    ("b2-sq-4095-k15x17", 1, (60, 40), (12, 9), (15, 17), dict(lo=0, hi=4095, texture="binary")),
    ("b3-ncc-4095", 2, (60, 40), (12, 9), (9, 9), dict(lo=0, hi=4095)),
    ("b3-ncc-minus1", 2, (60, 40), (12, 9), (9, 9), dict(lo=-1, hi=4095)),
    ("b4-abs-999999", 0, (60, 40), (12, 9), (9, 9), dict(lo=995904, hi=999999)),
    ("b4-sq-minus999999", 1, (60, 40), (12, 9), (9, 9), dict(lo=-999999, hi=-995904)),
    ("b5-abs-k17-58052", 0, (60, 40), (11, 9), (17, 17), dict(lo=0, hi=58052, texture="binary")),
    ("b5-sq-k15-4095", 1, (60, 40), (11, 9), (15, 15), dict(lo=0, hi=4095, texture="binary")),
    ("b5-abs-offset-3e7", 0, (60, 40), (11, 9), (15, 15), dict(lo=30000000, hi=30004094)),
    ("b5-sq-offset-3e7", 1, (60, 40), (11, 9), (15, 15), dict(lo=30000000, hi=30004094)),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_calc_disparity_matches_brute_force(oracle, case):
    what, cost, (W, H), search, kernel, kw = case
    left, right = make_pair(W, H, search, kernel, seed=len(what), **kw)
    ref = brute_calc_disparity(cost, left, right, search, kernel)
    got = oracle.calc_disparity(cost, left, right, search, kernel)
    assert np.array_equal(got, ref), f"{what}: {int((got != ref).any(-1).sum())} of {W * H} pixels differ"
    assert ref[..., 2].any()
