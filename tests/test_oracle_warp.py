"""The image-warp oracle (oracle/vw_warp_oracle.c): the reference's known-answer tests of Image/tests/TestInterpolation.cxx:32-90
(Bilinear, Bicubic, Nearest), Image/tests/TestTransform.cxx:36-107 (Translate and Resample by 2, as the homographies they are
exactly) and Stereo/tests/TestDisparity.cxx:188-202 (DisparityTransform), and the oracle against tests/warp_reference.py, an
independent restatement, bit for bit (floats as raw bits, NaN equal to NaN) inside the contract's domain, with 0.0f outside
it.  The matrix covers both transforms x three interpolations x two edge extensions on 1 x 1, 1 x N, N x 1 and 50 x 147
images; identity, integer and fractional shifts, rotation with scale, a projective matrix and one whose w crosses 0 inside
the window; NaN / inf / -0.0 pixels; reversed points on integers, on .5 ties of both signs and within 2^-24 of the next
integer; windows with negative origins and beyond the image; disparities with 0-100 % invalid pixels and windows beyond the
disparity.  The GPU module test_gpu_zz_warp.py reuses these cases."""
import math

import numpy as np
import pytest

import warp_reference as R

KINDS = (R.HOMOGRAPHY, R.DISPARITY)
INTERPS = (R.BILINEAR, R.BICUBIC, R.NEAREST)
EDGES = (R.ZERO, R.CONSTANT)
SHAPES = ((1, 1), (1, 23), (23, 1), (50, 147))                      # (rows, cols)
INVALID = (0.0, 0.3, 1.0)


def shift(tx, ty):
    return np.array([[1, 0, tx], [0, 1, ty], [0, 0, 1.0]])


def _rot_scale():
    c, s = 1.1 * math.cos(0.3), 1.1 * math.sin(0.3)
    return np.array([[c, -s, 5.5], [s, c, -3.25], [0, 0, 1.0]])


# the matrices reverse() applies (inverse(H))
MATRICES = {
    "identity": np.eye(3),
    "int_shift": shift(3, -2),
    "frac_shift": shift(0.3125, -1.75),
    "halves": shift(0.5, -0.5),                                      # .5 ties of both signs for nearest-pixel rounding
    "near_int": shift(-2.0 ** -26, 1 - 2.0 ** -25),                  # within 2^-24 of the next integer: normx rounds to 1
    "rot_scale": _rot_scale(),
    "projective": np.array([[0.98, 0.03, 2.5], [-0.02, 1.01, -1.25], [1.5e-3, -2e-3, 1.0]]),
    "w_crosses_0": np.array([[1, 0, 0], [0, 1, 0], [0.05, 0, -1.0]]),  # w = 0.05 x - 1 is 0 at x = 20: inf / NaN there
}


@pytest.fixture(scope="module")
def wo():
    import oracle.warp as wo
    wo.build()
    return wo


def same(a, b):
    """bit for bit, NaN equal to NaN"""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    nan = np.isnan(a) & np.isnan(b)
    return bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | nan))


def image(seed, shape, special=0.0):
    """float32 values in [-100, 100), a quarter of them integral; `special` of the pixels NaN, +-inf or -0.0"""
    rng = np.random.default_rng(seed)
    im = (rng.random(shape) * 200 - 100).astype(np.float32)
    ints = rng.random(shape) < 0.25
    im[ints] = np.rint(im[ints])
    if special:
        pick = rng.random(shape) < special
        im[pick] = rng.choice(np.array([np.nan, np.inf, -np.inf, -0.0, -0.0], np.float32), int(pick.sum()))
    return im


def disparity(seed, shape, invalid):
    """a float32 {dx, dy, valid} raster: offsets in [-6, 6], a third of them integral and a third on halves; `invalid` of
    the pixels invalid, with nonzero offsets"""
    rng = np.random.default_rng(seed)
    d = (rng.random(shape + (2,)) * 12 - 6).astype(np.float32)
    k = rng.integers(0, 3, shape)
    d[k == 0] = np.rint(d[k == 0])
    d[k == 1] = np.rint(2 * d[k == 1]) / 2
    v = (rng.random(shape) >= invalid).astype(np.float32)
    return np.concatenate([d, v[..., None]], -1)


def windows(shape):
    """the plain window, and one with a negative origin reaching beyond the image on every side"""
    h, w = shape
    return ((0, 0, w, h), (-3, -2, w + 7, h + 5))


def cases(kind, shape):
    """(label, image, window, matrix, disparity) of the matrix for one transform kind and image shape"""
    seed = 100 * SHAPES.index(shape) + 10 * kind
    im = image(seed, shape)
    out = []
    if kind == R.HOMOGRAPHY:
        for name, m in MATRICES.items():
            for k, win in enumerate(windows(shape)):
                out.append((f"{name}/w{k}", im, win, m, None))
    else:
        for inv in INVALID:
            d = disparity(seed + 1, shape, inv)
            for k, win in enumerate(windows(shape)):                     # the second window runs beyond the disparity too
                out.append((f"invalid{inv}/w{k}", im, win, None, d))
    return out


def run_both(wo, im, kind, interp, edge, win, m, d):
    got = wo.transform(im, kind, interp, edge, win, matrix=m, disparity=d)
    want, inside = R.transform(im, kind, interp, edge, win, matrix=m, disparity=d)
    return got, want, inside


def check(wo, im, kind, interp, edge, win, m, d, label):
    got, want, inside = run_both(wo, im, kind, interp, edge, win, m, d)
    assert same(got[inside], want[inside]), (label, np.argwhere(~((got == want) | (np.isnan(got) & np.isnan(want))) & inside)[:5])
    assert (got[~inside].view(np.uint32) == 0).all(), (label, "outside the domain: +0.0f")
    return got, inside


# ---- the reference's known-answer tests ----------------------------------------------------------------------------------------
KAT = np.array([[1, 2], [3, 4], [5, 6]], np.float32)                # im(0,0)=1 im(1,0)=2 im(0,1)=3 im(1,1)=4 im(0,2)=5 im(1,2)=6


def at(wo, interp, edge, i, j):
    """InterpolationView(i, j) of the KAT image: the identity warp of a shifted 1 x 1 window"""
    x, y = math.floor(i), math.floor(j)
    return float(wo.transform(KAT, R.HOMOGRAPHY, interp, edge, (x, y, 1, 1), matrix=shift(i - x, j - y))[0, 0])


def test_kat_interpolation(wo):
    b = lambda i, j: at(wo, R.BILINEAR, R.CONSTANT, i, j)            # noqa: E731  (interpolate(im, Bilinear()): constant edges)
    assert (b(1, 1), b(1, 1.5), b(0.5, 1), b(0.5, 0.5)) == (4, 5, 3.5, 2.5)
    c = lambda i, j: at(wo, R.BICUBIC, R.ZERO, i, j)                 # noqa: E731
    assert (c(1, 1), c(1, 1.5), c(0.5, 1)) == (4, 5.5, 3.9375)
    assert abs(c(0.5, 0.5) - 2.7773) <= 0.001
    n = lambda i, j: at(wo, R.NEAREST, R.CONSTANT, i, j)             # noqa: E731
    assert (n(1, 1), n(1, 1.5), n(1, 1.2), n(0.7, 1), n(0.4, 1.8)) == (4, 6, 4, 4, 5)


def test_kat_transform(wo):
    # transform(im, TranslateTransform(1, 1)): reverse(p) = p - (1, 1), bilinear, zero edges
    t = wo.transform(KAT, R.HOMOGRAPHY, R.BILINEAR, R.ZERO, (-100, -100, 102, 103), matrix=shift(-1, -1))
    px = lambda i, j: float(t[j + 100, i + 100])                     # noqa: E731
    assert (px(1, 1), px(0, 0), px(1, 2), px(-1, -1), px(-100, -100)) == (1, 0, 3, 0, 0)
    # resample(im, 2, 2): reverse(p) = p / 2, bilinear, constant edges; 4 x 6
    r = wo.transform(KAT, R.HOMOGRAPHY, R.BILINEAR, R.CONSTANT, (-100, -100, 201, 201), matrix=np.diag([0.5, 0.5, 1.0]))
    px = lambda i, j: float(r[j + 100, i + 100])                     # noqa: E731
    assert (px(0, 0), px(2, 2), px(1, 1), px(-1, -1), px(-100, -100), px(100, 100)) == (1, 4, 2.5, 1, 1, 6)


def test_kat_disparity_transform(wo):
    """DisparityTransform(disparity).reverse(i, 0)[0] == delta + i (TestDisparity.cxx:188-202, EXPECT_NEAR 1e-5), read through
    a ramp image whose pixel x holds x: bilinear interpolation of the ramp adds at most a few float32 ulps of ~100.  The ramp
    can only show reversed points on the image, so i = 0, 1, 2 (reversed to -3, -1.9, -0.8) are left out."""
    d = np.zeros((1, 100, 3), np.float32)
    for i in range(100):
        d[0, i] = (np.float32(2 + (i - 50) * 0.1), 0, 1)
    ramp = np.arange(256, dtype=np.float32)[None, :]
    got = wo.transform(ramp, R.DISPARITY, R.BILINEAR, R.ZERO, (0, 0, 100, 1), disparity=d)[0]
    for i in range(3, 100):
        assert abs(float(np.float32(2 + (i - 50) * 0.1)) + i - got[i]) <= 3e-5, i


# ---- the oracle against the restatement ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("edge", EDGES, ids=["zero", "constant"])
@pytest.mark.parametrize("interp", INTERPS, ids=["bilinear", "bicubic", "nearest"])
@pytest.mark.parametrize("kind", KINDS, ids=["homography", "disparity"])
def test_matrix(wo, kind, interp, edge, shape):
    outside = 0
    for label, im, win, m, d in cases(kind, shape):
        _, inside = check(wo, im, kind, interp, edge, win, m, d, label)
        outside += int((~inside).sum())
    if kind == R.HOMOGRAPHY and shape[1] > 20:
        assert outside > 0, "the w_crosses_0 matrix leaves the domain inside the window"


@pytest.mark.parametrize("edge", EDGES, ids=["zero", "constant"])
@pytest.mark.parametrize("interp", INTERPS, ids=["bilinear", "bicubic", "nearest"])
def test_special_pixels(wo, interp, edge):
    """NaN, +-inf and -0.0 pixels: the integer shortcut returns them unchanged, interpolation spreads them as IEEE does"""
    im = image(5, (21, 34), special=0.08)
    for name in ("identity", "frac_shift", "rot_scale", "near_int"):
        check(wo, im, R.HOMOGRAPHY, interp, edge, (-2, -2, 38, 25), MATRICES[name], None, name)
    check(wo, im, R.DISPARITY, interp, edge, (-2, -2, 38, 25), None, disparity(6, (21, 34), 0.3), "disparity")


def test_integral_points_keep_their_pixel(wo):
    """identity and integer shifts hit pixels exactly: every interpolation returns the (edge-extended) pixel bit for bit"""
    im = image(8, (9, 13), special=0.1)
    for interp in INTERPS:
        got = wo.transform(im, R.HOMOGRAPHY, interp, R.ZERO, (0, 0, 13, 9), matrix=np.eye(3))
        assert same(got, im), interp
        got = wo.transform(im, R.HOMOGRAPHY, interp, R.CONSTANT, (0, 0, 13, 9), matrix=shift(-20, 30))
        assert same(got, np.broadcast_to(im[8, 0], (9, 13)).astype(np.float32)), interp


def test_near_integer_gives_normx_one(wo):
    """a reversed x of 5 - 2^-26 floors to 4 and rounds to 5.0f: normx == 1, so bilinear returns pixel 5 in float arithmetic"""
    im = np.array([[0, 1, 2, 3, 4, 5, 6, 7]], np.float32) * np.float32(1.1)
    got = wo.transform(im, R.HOMOGRAPHY, R.BILINEAR, R.ZERO, (5, 0, 1, 1), matrix=shift(-2.0 ** -26, 0))
    assert same(got, im[:, 5:6] * np.float32(1.0) + im[:, 4:5] * np.float32(0.0))


def test_out_of_domain_is_zero(wo):
    """w == 0 (inf / NaN) and |c| >= 2^30 give +0.0f, whatever the edge extension"""
    im = image(9, (4, 4)) + 1000
    for edge in EDGES:
        for interp in INTERPS:
            z = wo.transform(im, R.HOMOGRAPHY, interp, edge, (0, 0, 4, 4), matrix=np.array([[1, 0, 0], [0, 1, 0], [0, 0, 0.0]]))
            assert (z.view(np.uint32) == 0).all()
        big = wo.transform(im, R.HOMOGRAPHY, interp, R.CONSTANT, (0, 0, 2, 1), matrix=shift(2.0 ** 30 - 1, 0))
        assert big[0, 0] == im[0, 3] and big[0, 1].view(np.uint32) == 0      # 2^30 - 1 is inside (clamped), 2^30 is not
