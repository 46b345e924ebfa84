"""The SGM oracle across its penalty range, checked against an independent restatement of the reference
(tests/sgm_reference.py).  Explicit P1 / P2 up to 30000 drive the accumulated costs past 65535, where the reference's uint16
accumulation wraps; these cases assert that the wrap happens and that it decides winners, so the GPU tests that reuse the
same inputs (test_gpu_sgm_penalties.py) compare the kernels' wrapping arithmetic, not just their easy regime."""
import numpy as np
import pytest

import sgm_reference as R

# census 5 defaults: P1 = 15, P2 = 750.  (0, 0) is the control; (700, 0) keeps the default P2 with an explicit P1.
GRID = [(0, 0), (1, 1), (1, 30000), (30000, 30000), (29999, 30000), (200, 8000), (0, 30000), (700, 0)]
# P2 = 30000 with moving boxes: the 8-path sums reach ~240000.  (200, 8000) cannot wrap: a path costs at most
# P2 + 24 with census 5, and 8 x 8024 < 65536.
WRAPS = {(1, 30000), (30000, 30000), (29999, 30000), (0, 30000)}
SEARCH = (15, 11)
OH, OW = 32, 40


def _case(kernel, seed=1):
    left, right = R.flat_pair(seed, OH, OW, SEARCH, kernel)
    return left, right, R.moving_boxes(seed + 1, OH, OW, SEARCH, 7, 5)


def test_census_signatures_match_the_oracle(oracle):
    """binary census 3/5/7/9 (CensusTransform.h:64-160): every signature of a random 8-bit image, bit for bit"""
    img = np.random.default_rng(3).integers(0, 256, (14, 15)).astype(np.uint8)
    img[5:9, 5:9] = 77                                   # ties with the centre count as "not greater"
    for k in (3, 5, 7, 9):
        hk = k // 2
        for row in range(hk, img.shape[0] - hk):
            for col in range(hk, img.shape[1] - hk):
                assert R.census_value(img, col, row, k) == oracle.census_value(img, col, row, k), (k, col, row)


def test_census_reference_kat():
    """Image/tests/TestCensusTransform.cxx:25-46 through the restatement's bit order"""
    src = np.array([[1, 2, 7, 2, 2, 8, 5, 2], [1, 4, 2, 9, 8, 8, 2, 6], [5, 2, 7, 2, 2, 2, 4, 6], [1, 2, 2, 2, 1, 4, 5, 2],
                    [6, 6, 3, 7, 2, 2, 5, 5], [1, 2, 9, 2, 2, 2, 2, 2], [7, 9, 2, 8, 5, 2, 3, 2], [1, 2, 2, 2, 2, 2, 2, 1]], np.uint8)
    assert R.census_value(src, 2, 2, 3) == 0x20 and R.census_value(src, 4, 5, 3) == 0x86 and R.census_value(src, 6, 1, 3) == 0xDB
    assert R.census_value(src, 4, 4, 5) == 0x0088F60D and R.census_value(src, 2, 3, 5) == 0x005D03C4
    assert R.census_value(src, 3, 4, 7) == 0x00001C0000041400


def test_u8_stretch_is_the_identity_on_the_test_imagery():
    left, right, _ = _case(5)
    for im in (left, right):
        assert np.array_equal(R.as_u8(im), im)
    with pytest.raises(AssertionError):
        R.as_u8(left[1:-1, 1:-1])                        # no 0 / 255 left: the stretch would rescale


def test_select_best_disparity_tie_smoothing():
    """SGM.cc:1159-1284 on hand-made boxes: a unique minimum is taken as is; a tie is broken by the horizontal 3-tap mean
    (edges average two values); a tie the horizontal passes cannot break goes to the vertical pass after five of them."""
    assert R.select_best_disparity(np.array([[5, 3, 4]])) == (1, False, 3)
    # pass 1: (7+3)/2 = 5, (7+3+9)/3 = 6.33 -> 6, (3+9+3)/3 = 5, (9+3)/2 = 6 still ties; pass 2: 5.5 -> 6, 5.33 -> 5, ...
    assert R.select_best_disparity(np.array([[7, 3, 9, 3]])) == (1, True, 3)
    # columns never differ: five horizontal passes change nothing, the vertical one still ties rows 1 and 2 after the
    # sixth pass, and the first of the tied entries wins
    v = np.array([[40000, 40000], [39000, 39000], [39000, 39000], [40000, 40000]])
    assert R.select_best_disparity(v) == (2, True, 39000)


@pytest.mark.parametrize("p1,p2", GRID)
def test_restatement_matches_oracle_over_the_penalty_grid(oracle, p1, p2):
    """census 5, 32 x 40 outputs: the constant search box and moving boxes of <= 7 x 5, bit for bit"""
    left, right, b = _case(5)
    res = R.sgm(left, right, SEARCH, 5, b, p1, p2)
    ri, _ = oracle.sgm_calc_disparity_bounds(left, right, SEARCH, 5, b, p1=p1, p2=p2)
    assert np.array_equal(res.disparity, ri), f"{int((res.disparity != ri).any(-1).sum())} pixels differ"
    const = R.sgm(left, right, SEARCH, 5, None, p1, p2)
    rc = oracle.sgm_calc_disparity(left, right, SEARCH, 5, p1, p2)
    assert np.array_equal(const.disparity, rc), f"{int((const.disparity != rc).any(-1).sum())} pixels differ"
    if (p1, p2) in WRAPS:
        R.assert_wrap_decides(res)
        assert (res.smoothed & (res.lowest > 30000)).any(), "no tie smoothing on wrapped costs above 30000"
    else:
        assert res.max_sum <= R.U16 and np.array_equal(res.disparity, res.unwrapped)
    if (p1, p2) == (0, 0):
        assert const.max_sum <= R.U16


@pytest.mark.parametrize("kernel", [3, 7, 9])
@pytest.mark.parametrize("p1,p2", [(0, 30000), (30000, 30000)])
def test_restatement_matches_oracle_other_kernels(oracle, kernel, p1, p2):
    left, right, b = _case(kernel, seed=10 + kernel)
    res = R.sgm(left, right, SEARCH, kernel, b, p1, p2)
    ri, _ = oracle.sgm_calc_disparity_bounds(left, right, SEARCH, kernel, b, p1=p1, p2=p2)
    assert np.array_equal(res.disparity, ri), f"{int((res.disparity != ri).any(-1).sum())} pixels differ"
    R.assert_wrap_decides(res)
    rc = oracle.sgm_calc_disparity(left, right, SEARCH, kernel, p1, p2)
    assert np.array_equal(R.sgm(left, right, SEARCH, kernel, None, p1, p2).disparity, rc)


def test_defaults_never_wrap(oracle):
    """At the reference's default penalties a path costs at most 255 + P2 <= 2255, so even moving boxes stay below 65536."""
    for kernel in (3, 5, 7, 9):
        left, right, b = _case(kernel, seed=20 + kernel)
        res = R.sgm(left, right, SEARCH, kernel, b)
        assert res.max_sum <= R.U16 and np.array_equal(res.disparity, res.unwrapped)
        assert np.array_equal(res.disparity, oracle.sgm_calc_disparity_bounds(left, right, SEARCH, kernel, b)[0])
