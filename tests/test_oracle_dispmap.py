"""The disparity-map oracle (oracle/vw_dispmap_oracle.c): the reference's known-answer tests of
Stereo/tests/TestDisparity.cxx:34-219 (Transform1, Transform2, DisparitySubsample, DisparityUpsample, GetDisparityRange),
and the oracle against tests/dispmap_reference.py, an independent restatement, bit for bit (floats as raw bits, NaN equal to
NaN) across invalid densities, thin and tiny sizes, negative disparities, signed zeros, NaNs, the range mask's y-coordinate
quirk, invalid pixels under the lazy transform and do_round on and off.  The GPU module test_gpu_zz_disparity_map.py
reuses these cases."""
import numpy as np
import pytest

import dispmap_reference as R

TYPES = (np.int32, np.float32)
INVALID = (0.0, 0.3, 0.7, 1.0)
SHAPES = ((1, 1), (1, 9), (9, 1), (2, 2), (5, 7), (8, 6), (13, 16))
# an affine homography (Transform2 of the KAT), a projective one, and a translation
MATRICES = (np.array([[1.00679, -0.0125401, 116.812], [0.00788373, 0.996033, -1.93039], [0, 0, 1]]),
            np.array([[0.98, 0.03, 12.5], [-0.02, 1.01, -7.25], [1.5e-5, -2e-5, 1.0]]),
            np.array([[1, 0, 45], [0, 1, -30], [0, 0, 1.0]]))


@pytest.fixture(scope="module")
def dm():
    import oracle.dispmap as dm
    dm.build()
    return dm


def same(a, b):
    """bit for bit, NaN equal to NaN"""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype == np.float32:
        nan = np.isnan(a) & np.isnan(b)
        return bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | nan))
    return bool(np.array_equal(a, b))


def pix(dx, dy, dtype=np.float32):
    return np.array([dx, dy, 1], dtype)


# ---- the reference's known-answer tests ----------------------------------------------------------------------------------------
def kat_map():
    """map(i, j) = PixelDisp(i*5 + j, j*7 + i) of Transform1 / Transform2, as (rows, cols, 3)"""
    m = np.zeros((5, 5, 3), np.float32)
    for i in range(5):
        for j in range(5):
            m[j, i] = (i * 5 + j, j * 7 + i, 1)
    return m


@pytest.mark.parametrize("matrix", [MATRICES[2], MATRICES[0]], ids=["Transform1", "Transform2"])
def test_kat_transform(dm, matrix):
    m = kat_map()
    res = dm.transform_disparities(dm.LAZY, np.linalg.inv(matrix), m)
    for i in range(5):
        for j in range(5):
            t = np.array([res[j, i, 0], res[j, i, 1], 1.0])
            loc = np.array([i, j, 0.0])
            check = matrix @ (t + loc) - loc
            assert np.allclose(m[j, i, :2], check[:2], atol=1e-1)


def test_kat_subsample(dm):
    m = np.zeros((4, 4, 3), np.float32)
    m[0, 0], m[0, 2], m[1, 2] = pix(3, 1), pix(4, 2), pix(2, 2)
    s = dm.disparity_subsample(m)
    assert s.shape == (2, 2, 3)
    assert s[0, 0, 2] and s[0, 1, 2] and not s[1, 0, 2] and s[1, 1, 2]
    assert np.allclose(s[0, 0, :2], (1.5, 0.5), atol=1e-3)
    assert np.allclose(s[0, 1, :2], (1.75, 1.0), atol=1e-3)
    assert np.allclose(s[1, 1, :2], (1, 1), atol=1e-3)
    im = np.zeros((1, 3, 3), np.int32)
    im[0, 0], im[0, 1] = (4, 2, 1), (10, -8, 1)
    si = dm.disparity_subsample(im)
    assert si.shape == (1, 2, 3) and si[0, 0, 2] and si[0, 1, 2]
    assert tuple(si[0, 0, :2]) == (2, 0) and tuple(si[0, 1, :2]) == (5, -4)     # truncation toward zero


def test_kat_upsample(dm):
    m = np.zeros((2, 2, 3), np.float32)
    m[0, 0], m[1, 1] = pix(3, 1), pix(5, 5)
    u = dm.disparity_upsample(m)
    assert u.shape == (4, 4, 3)
    assert all(u[i, i, 2] for i in range(4)) and not any(u[i, 3 - i, 2] for i in range(4))
    assert tuple(u[0, 0, :2]) == (6, 2) and tuple(u[1, 1, :2]) == (6, 2)
    assert tuple(u[2, 2, :2]) == (10, 10) and tuple(u[2, 3, :2]) == (10, 10)


def test_kat_range(dm):
    d = np.zeros((1, 4, 3), np.float32)
    d[0, 0], d[0, 1], d[0, 2] = pix(2, 2), pix(3, 5), (-4, -1, 0)
    assert tuple(dm.get_disparity_range(d)) == (2, 2, 3, 5)
    d[0, 0, 2] = d[0, 1, 2] = 0
    assert tuple(dm.get_disparity_range(d)) == (0, 0, 0, 0)


# ---- the oracle against the restatement ----------------------------------------------------------------------------------------
def check_all(dm, d, i):
    """every operation on d against the restatement; i picks the matrices and bounds"""
    assert same(dm.disparity_subsample(d), R.disparity_subsample(d))
    assert same(dm.disparity_upsample(d), R.disparity_upsample(d))
    assert same(dm.get_disparity_range(d), R.get_disparity_range(d))
    h, w = d.shape[:2]
    for mn, mx in (((-5, -3), (w + 4, h + 2)), ((0, 0), (w, h)), ((-30, 10), (w - 3, h + 40))):
        assert same(dm.disparity_range_mask(d, mn, mx), R.disparity_range_mask(d, mn, mx)), (mn, mx)
    m = MATRICES[i % len(MATRICES)]
    inv = np.linalg.inv(m)
    assert same(dm.transform_disparities(dm.LAZY, inv, d), R.transform_lazy(inv, d))
    for do_round in (False, True):
        for origin in ((0, 0), (17, -9)):
            got = dm.transform_disparities(dm.EXPLICIT, m, d, do_round, origin)
            assert same(got, R.transform_explicit(do_round, origin, m, d)), (do_round, origin)


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("invalid", INVALID)
def test_matrix(dm, invalid, shape, dtype):
    i = SHAPES.index(shape) + INVALID.index(invalid)
    check_all(dm, R.random_disparity(1000 + 7 * i, shape, invalid, dtype), i)


def signed_zero_case():
    """-0.0 and +0.0 in both channels: the first in raster order wins the range, and zeros meet the subsample's sums"""
    d = np.zeros((3, 4, 3), np.float32)
    d[..., 2] = 1
    d[0, 0, :2] = (-0.0, 0.0)
    d[0, 1, :2] = (0.0, -0.0)
    d[1, 1, :2] = (-0.0, -0.0)
    d[2, 3, :2] = (1.5, -2.5)
    return d


def nan_cases():
    """a NaN in the first valid pixel (it sticks) and a NaN later (skipped)"""
    a = R.random_disparity(5, (4, 6), 0.0, np.float32)
    a[0, 0, 2] = 0
    a[0, 1, 0] = np.nan                     # first valid pixel, dx only
    b = R.random_disparity(6, (4, 6), 0.0, np.float32)
    b[2, 3, 1] = np.nan
    return a, b


def test_signed_zeros_and_nans(dm):
    d = signed_zero_case()
    r = dm.get_disparity_range(d)
    assert same(r, R.get_disparity_range(d))
    assert np.signbit(r[0]) and r[0] == 0 and r[1] == -2.5  # min dx: -0.0, the first of the zeros
    assert r[2] == 1.5 and r[3] == 0 and not np.signbit(r[3])  # max dy: +0.0, the first of the zeros
    check_all(dm, d, 0)
    a, b = nan_cases()
    ra, rb = dm.get_disparity_range(a), dm.get_disparity_range(b)
    assert np.isnan(ra[0]) and np.isnan(ra[2]) and not np.isnan(ra[1])
    assert not np.isnan(rb).any()
    assert same(ra, R.get_disparity_range(a)) and same(rb, R.get_disparity_range(b))
    check_all(dm, a, 1)
    check_all(dm, b, 2)


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
def test_negative_disparities_truncate(dm, dtype):
    """negative sums divide toward zero (int) and round to nearest float (float)"""
    d = R.random_disparity(77, (9, 11), 0.25, dtype, scale=1e3)
    d[..., :2] = -np.abs(d[..., :2])
    check_all(dm, d, 0)
    s = dm.disparity_subsample(d)
    if dtype == np.int32:
        assert (s[..., :2] <= 0).all()


def test_range_mask_y_compares_against_min_x(dm):
    """a pixel whose y + dy lies below min[1] but not below min[0] is kept (:279 compares y against m_min[0])"""
    d = np.zeros((3, 3, 3), np.int32)
    d[...] = (0, 0, 1)
    d[1, 1] = (0, -5, 1)                    # y + dy = -4
    got = dm.disparity_range_mask(d, (-10, 0), (10, 10))
    assert got[1, 1, 2] == 1 and same(got, R.disparity_range_mask(d, (-10, 0), (10, 10)))
    got = dm.disparity_range_mask(d, (-3, -10), (10, 10))
    assert got[1, 1, 2] == 0 and tuple(got[1, 1]) == (0, 0, 0)
    assert got[0, 0, 2] == 1                # max - 1 bound: x + dx = 0 < 9
    got = dm.disparity_range_mask(d, (0, 0), (3, 3))
    assert got[2, 2, 2] == 0 and got[1, 1, 2] == 0 and got[0, 0, 2] == 1


def test_lazy_transform_keeps_invalid_values(dm):
    d = R.random_disparity(9, (4, 5), 0.5, np.float32)
    m = np.linalg.inv(MATRICES[1])
    got = dm.transform_disparities(dm.LAZY, m, d)
    inv = d[..., 2] == 0
    assert inv.any() and (got[inv][:, 2] == 0).all() and (got[inv][:, :2] != 0).all()
    got_e = dm.transform_disparities(dm.EXPLICIT, MATRICES[1], d)
    assert (got_e[inv] == 0).all()


def test_do_round_halves(dm):
    """do_round rounds halves away from zero"""
    d = np.zeros((1, 4, 3), np.float32)
    d[0] = [(0.5, -0.5, 1), (1.5, -1.5, 1), (2.5, -2.5, 1), (0.49999997, -0.49999997, 1)]
    ident = np.eye(3)
    got = dm.transform_disparities(dm.EXPLICIT, ident, d, True)
    assert got[0, :, :2].tolist() == [[1, -1], [2, -2], [3, -3], [0, -0.0]]
    assert same(got, R.transform_explicit(True, (0, 0), ident, d))


def test_int32_results_outside_the_range(dm):
    """a projective matrix whose w crosses zero: NaN and out-of-range int32 results become INT32_MIN, as x86-64's conversion
    gives them"""
    d = R.random_disparity(12, (30, 4), 0.1, np.int32)
    m = MATRICES[1]
    with np.errstate(all="ignore"):
        got = dm.transform_disparities(dm.EXPLICIT, m, d, True, (0, 49985))
        assert same(got, R.transform_explicit(True, (0, 49985), m, d))
    assert (got[..., :2] == -2 ** 31).any() and (np.abs(got[..., :2]) < 2 ** 20).any()
