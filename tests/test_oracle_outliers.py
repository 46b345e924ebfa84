"""The oracle's neighbourhood outlier filters (oracle/vw_outlier_oracle.c: rm_outliers_using_{thresh,mean,stddev} and
disparity_cleanup_using_*, on int32 and float32 disparities) against the restatement that walks the reference's
accessors literally (tests/outlier_reference.py), bit for bit; its integer thresh filters against the main oracle's; and
hand cases, each built so that a wrong reading of the reference flips at least one output.  The GPU tests
(test_gpu_zz_outlier_filters.py) hold the engine to the oracle on the same inputs."""
import numpy as np
import pytest

import outlier_reference as R

METHODS = (R.THRESH, R.MEAN, R.STDDEV)
TYPES = (np.int32, np.float32)
INVALID = [0.0, 0.25, 0.6, 0.9, 1.0]
HALVES = [(1, 1), (2, 1), (1, 3), (3, 3), (5, 5), (7, 4)]
SHAPE = (9, 12)
# thresholds per case: (pixel_threshold, rejection_threshold, max_mean_diff)
THRESHOLDS = [(3.0, 0.5, 3.0), (1.0, 0.2, 1.0), (2.0, 1.0, 6.0), (0.5, 0.75, 0.5)]
SMALL = [((1, 1), (1, 1)), ((1, 9), (2, 1)), ((9, 1), (1, 2)), ((3, 2), (5, 5)), ((2, 5), (3, 4)), ((1, 4), (7, 4))]


@pytest.fixture(scope="session")
def ou():
    """the outlier-filter oracle (oracle/outliers.py)"""
    import oracle.outliers as o
    o.build()
    return o


def same(got, want):
    """bit for bit: the same dtype, shape and bytes (float outputs compared as raw bits)"""
    return got.dtype == want.dtype and got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32))


def params(method, i):
    pt, rt, mmd = THRESHOLDS[i % len(THRESHOLDS)]
    if method == R.STDDEV:
        rt = (0.5, 2.0, 0.1, 1.0)[i % 4]            # the standard deviation's floor, in disparity units
    return dict(pt=pt, rt=rt, mmd=mmd)


def matrix_case(invalid, half, dtype, shape=SHAPE):
    seed = 2000 + int(invalid * 100) * 13 + half[0] * 7 + half[1] * 3 + (dtype == np.float32)
    return R.random_disparity(seed, shape, invalid, dtype)


def oracle_run(ou, method, cleanup, d, hx, hy, pt, rt, mmd):
    return ou.outlier_filter(method, cleanup, d, hx, hy, pt, rt, mmd)


def check_all(ou, d, hx, hy, i):
    """every method, both composites, against the restatement; returns how many pixels the filters changed"""
    changed = 0
    for method in METHODS:
        p = params(method, i)
        for cleanup in (False, True):
            want = R.outlier_filter(method, cleanup, d, hx, hy, **p)
            got = oracle_run(ou, method, cleanup, d, hx, hy, **p)
            assert same(got, want), (method, cleanup, np.argwhere((got != want).any(-1))[:5])
            changed += int((got != d).any(-1).sum())
    return changed


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
@pytest.mark.parametrize("half", HALVES, ids=lambda h: f"{h[0]}x{h[1]}")
@pytest.mark.parametrize("invalid", INVALID)
def test_oracle_matches_restatement(ou, invalid, half, dtype):
    d = matrix_case(invalid, half, dtype)
    changed = check_all(ou, d, half[0], half[1], HALVES.index(half) + INVALID.index(invalid))
    if 0 < invalid < 0.9:
        assert changed > 0, "the case exercises no rejection"


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
@pytest.mark.parametrize("shape,half", SMALL)
def test_small_and_thin_images(ou, shape, half, dtype):
    """1x1, 1xN and Nx1 images and images smaller than the window: the edge extension supplies the window"""
    d = R.random_disparity(31 + shape[0] * 10 + shape[1], shape, 0.2, dtype)
    check_all(ou, d, half[0], half[1], shape[0] + shape[1])


@pytest.mark.parametrize("cleanup", [False, True])
@pytest.mark.parametrize("half", [(1, 1), (2, 3), (5, 5)])
def test_integer_thresh_matches_main_oracle(ou, oracle, half, cleanup):
    """the restated integer thresh filters are the main oracle's (vw_oracle.c), which the level loop is held to"""
    for invalid in (0.0, 0.3, 0.8):
        d = R.random_disparity(77 + half[0] + int(invalid * 10), (37, 45), invalid, np.int32)
        for pt, rt in ((3.0, 0.5), (1.0, 0.3), (0.0, 0.9)):
            f = oracle.disparity_cleanup_using_thresh if cleanup else oracle.rm_outliers_using_thresh
            assert same(ou.outlier_filter(R.THRESH, cleanup, d, half[0], half[1], pt, rt), f(d, half[0], half[1], pt, rt))


# ---- hand cases ---------------------------------------------------------------------------------------------------------
def disp(dx, dy=None, valid=None, dtype=np.int32):
    dx = np.asarray(dx, np.float64)
    dy = np.zeros_like(dx) if dy is None else np.asarray(dy, np.float64)
    v = np.ones_like(dx) if valid is None else np.asarray(valid, np.float64)
    return np.stack([dx, dy, v], -1).astype(dtype)


def hand_truncated_row(dtype):
    """5 x 3, one window (2, 1) over the whole image at the centre (2, 1).  Lengths: twelve 2s, two 3s, one 100, so the
    cutoff is 2 * 2 = 4.  Row 1 is [2, 100, c = 2, 3, 3]: the 100 ends the row, so the mean is 2 and the centre is kept
    (max_mean_diff 0.1).  Skipping only the 100 would take in 2, 3, 3: mean 30 / 14, and the centre would be rejected."""
    dx = [[2, 2, 2, 2, 2], [2, 100, 2, 3, 3], [2, 2, 2, 2, 2]]
    return disp(dx, dtype=dtype), (2, 1), 0.1


def hand_quantile_index(dtype):
    """3 x 3, window (1, 1) at the centre: lengths 1 x 6, 2, 10, 10 with the 2 and the 10s in the last row.  n = 9, so
    the index is floor(0.75 * 9) = 6: cutoff 2 * 2 = 4, the 10s are dropped, the mean is 8 / 7 and the centre (1) is kept
    (max_mean_diff 1).  Index 7 (rounding) would keep the 10s: mean 28 / 9, and the centre would be rejected."""
    dx = [[1, 1, 1], [1, 1, 1], [2, 10, 10]]
    return disp(dx, dtype=dtype), (1, 1), 1.0


def hand_float_tie():
    """3 x 3 float, window (1, 1) at the centre: eight pixels (1, 0) and q = (1, 1 + 2^-23) first in the last row.  The
    cutoff is 2 * 1 = 2.  q's length is 2 + 2^-23 in float64 but rounds to 2.0 in float32, so the reference (float32)
    keeps q and its row: mean dy = (1 + 2^-23) / 9, error^2 = 0.0123 > 0.01, the centre is rejected.  A float64 length
    would drop q and the rest of its row: mean (1, 0), the centre kept."""
    dx = np.ones((3, 3))
    dy = np.zeros((3, 3))
    dy[2, 0] = 1.0 + 2.0 ** -23
    d = disp(dx, dy, dtype=np.float32)
    assert np.float32(1.0) + np.float32(d[2, 0, 1]) == np.float32(2.0) and 1.0 + float(d[2, 0, 1]) > 2.0
    return d, (1, 1), 0.1


def hand_stddev_floor(dtype):
    """3 x 3, window (1, 1) at the centre: dx 0 around a centre of 9, dy 0.  Mean dx 1, error 8, std sqrt(8) < the floor 4,
    so pt * std = 2 * 4 = 8 = error: kept, because the comparison is strict.  Without the floor (8 > 2 sqrt 8) or with a
    non-strict comparison the centre would be rejected."""
    dx = np.zeros((3, 3))
    dx[1, 1] = 9
    return disp(dx, dtype=dtype)


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
def test_hand_truncated_row(ou, dtype):
    d, (hx, hy), mmd = hand_truncated_row(dtype)
    got = ou.rm_outliers_using_mean(d, hx, hy, mmd)
    assert same(got, R.outlier_filter(R.MEAN, False, d, hx, hy, mmd=mmd))
    assert got[1, 2, 2] == 1, "the centre is kept: the row ends at the long pixel"
    skip_one = R.outlier_filter(R.MEAN, False, d, hx, hy, mmd=mmd, literal=False)
    assert skip_one[1, 2, 2] == 0, "skipping only the long pixel rejects the centre"


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
def test_hand_quantile_index(ou, dtype):
    d, (hx, hy), mmd = hand_quantile_index(dtype)
    got = ou.rm_outliers_using_mean(d, hx, hy, mmd)
    assert same(got, R.outlier_filter(R.MEAN, False, d, hx, hy, mmd=mmd))
    assert got[1, 1, 2] == 1
    # the contrast, by hand: with the 10s in, the mean is 28 / 9 and the centre's error 19 / 9 > 1
    assert (28 / 9 - 1) ** 2 > mmd * mmd


def test_hand_float_tie(ou, monkeypatch):
    d, (hx, hy), mmd = hand_float_tie()
    got = ou.rm_outliers_using_mean(d, hx, hy, mmd)
    assert same(got, R.outlier_filter(R.MEAN, False, d, hx, hy, mmd=mmd))
    assert got[1, 1, 2] == 0, "the float32 length keeps q, and q moves the mean"
    # the contrast: lengths summed in float64 drop q and the rest of its row, and the centre stays
    monkeypatch.setattr(R, "length", lambda p: abs(float(p[0])) + abs(float(p[1])))
    assert R.outlier_filter(R.MEAN, False, d, hx, hy, mmd=mmd)[1, 1, 2] == 1


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
def test_hand_invalid_centre_keeps_children(ou, dtype):
    """an invalid centre is returned as it is: children included, for every filter; a float valid of 0.5 is valid and,
    when kept, copied as 0.5"""
    d = R.random_disparity(5, (6, 7), 0.0, dtype)
    d[2, 3] = (7, -3, 0)
    if dtype == np.float32:
        d[3, 3, 2] = 0.5
    for method in METHODS:
        for cleanup in (False, True):
            p = dict(pt=1e9, rt=0.0, mmd=1e9)
            got = ou.outlier_filter(method, cleanup, d, 1, 1, p["pt"], p["rt"], p["mmd"])
            assert same(got, R.outlier_filter(method, cleanup, d, 1, 1, **p))
            assert tuple(got[2, 3]) == (7, -3, 0)
            assert same(got, d), "nothing is rejected with these thresholds"


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
def test_hand_stddev_floor(ou, dtype):
    d = hand_stddev_floor(dtype)
    for pt, rt, kept in ((2.0, 4.0, 1), (1.99, 4.0, 0), (2.0, 0.0, 0)):
        got = ou.rm_outliers_using_stddev(d, 1, 1, pt, rt)
        assert same(got, R.outlier_filter(R.STDDEV, False, d, 1, 1, pt, rt))
        assert got[1, 1, 2] == kept, (pt, rt)


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
@pytest.mark.parametrize("method", METHODS)
def test_hand_cleanup_border(ou, method, dtype):
    """pass 2 of each composite reads pass 1 at out-of-image centres: on this raster an edge-extended pass 1 gives a
    different border"""
    for seed in range(40):
        d = R.random_disparity(900 + seed, (8, 10), 0.3, dtype, outliers=0.25)
        p = params(method, seed)
        want = R.outlier_filter(method, True, d, 2, 2, **p)
        other = R.outlier_filter(method, True, d, 2, 2, pass2_edge_extended=True, **p)
        if (want != other).any():
            break
    else:
        pytest.fail("no raster tells the two border readings apart")
    got = ou.outlier_filter(method, True, d, 2, 2, p["pt"], p["rt"], p["mmd"])
    assert same(got, want)
    diff = np.argwhere((want != other).any(-1))
    assert all(y in (0, d.shape[0] - 1) or x in (0, d.shape[1] - 1) for y, x in diff), diff


def stddev_wide_cases():
    """(disparity, half) pairs for stddev with half_h > half_v: one where every window holds at most (2 half_v + 1)^2 valid
    pixels (the reference is defined there), and one where some windows hold more"""
    inside = R.random_disparity(61, (10, 14), 0.75, np.float32)
    beyond = R.random_disparity(62, (10, 14), 0.05, np.float32)
    return [(inside, (3, 1), True), (beyond, (3, 1), False), (beyond.astype(np.int32), (4, 2), False)]


@pytest.mark.parametrize("case", range(3))
def test_stddev_wide_window(ou, case):
    d, (hx, hy), defined = stddev_wide_cases()[case]
    h, w = d.shape[:2]
    counts = [R.valid_count(d, x, y, hx, hy) for y in range(-1, h + 1) for x in range(-1, w + 1)]
    assert (max(counts) <= (2 * hy + 1) ** 2) == defined
    for cleanup in (False, True):
        for pt, rt in ((1.0, 0.5), (2.0, 0.1)):
            assert same(ou.outlier_filter(R.STDDEV, cleanup, d, hx, hy, pt, rt), R.outlier_filter(R.STDDEV, cleanup, d, hx, hy, pt, rt))


def test_oracle_refuses_zero_half_kernels(ou):
    d = R.random_disparity(1, (4, 4), 0.0, np.int32)
    for hx, hy in ((0, 1), (1, 0), (-1, 2)):
        with pytest.raises(ValueError):
            ou.outlier_filter(R.MEAN, 0, d, hx, hy, 1.0, 1.0, 1.0)
