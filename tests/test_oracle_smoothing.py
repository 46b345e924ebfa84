"""The oracle's disparity smoothing (disparity_median_filter, texture_measure, texture_preserving_disparity_filter) against
the restatement written from the reference's loops (tests/smoothing_reference.py), bit for bit with -0.0 == +0.0; the
reference's own known answers; a hand-sized case that pins the in-place, raster-order semantics; and the C ABI's argument
checks and its loud failure without a device.  The GPU tests (test_gpu_wavefront_smoothing.py) hold the engine to the oracle on
the same inputs."""
import ctypes as C

import numpy as np
import pytest

import smoothing_reference as S

F = np.float32
INVALID = [0.0, 0.1, 0.5, 1.0]
KERNELS = [1, 2, 3, 4, 5, 7, 11]
SHAPE = (19, 23)


@pytest.fixture(scope="session")
def so():
    """the disparity smoothing oracle (oracle/smoothing.py)"""
    import oracle.smoothing as s
    s.build()
    return s


def same(got, want):
    """equal as numbers (so -0.0 == +0.0), shape and all; NaN-free inputs"""
    return got.shape == want.shape and np.array_equal(got, want)


def median_case(invalid, k, integer):
    return S.random_disparity(1000 + int(invalid * 100) * 7 + k + 50 * integer, SHAPE, invalid, integer=integer)


@pytest.mark.parametrize("integer", [False, True])
@pytest.mark.parametrize("k", KERNELS)
@pytest.mark.parametrize("invalid", INVALID)
def test_median_matches_restatement(so, invalid, k, integer):
    """integer disparities give ties and even counts; random floats give distinct values"""
    d = median_case(invalid, k, integer)
    want = S.disparity_median_filter(d, k)
    assert same(so.disparity_median_filter(d, k), want)
    if k >= 3 and 0 < invalid < 1:
        assert not np.array_equal(want, d)


@pytest.mark.parametrize("shape,k", [((5, 6), 7), ((6, 5), 7), ((1, 30), 3), ((30, 1), 3), ((1, 1), 3), ((7, 7), 7), ((8, 9), 8)])
def test_median_small_images(so, shape, k):
    """images smaller than the window, one row, one column: nothing or only the interior changes"""
    d = S.random_disparity(7 + shape[0] * 31 + shape[1], shape, 0.2, integer=True)
    want = S.disparity_median_filter(d, k)
    assert same(so.disparity_median_filter(d, k), want)
    half = (k - 1) // 2
    if shape[0] <= 2 * half or shape[1] <= 2 * half:
        assert np.array_equal(want.view(np.int32), d.view(np.int32))


def test_median_keeps_invalid_and_border_pixels_bit_for_bit(so):
    d = S.random_disparity(3, SHAPE, 0.3)
    d[..., 2][d[..., 2] != 0] = 2.0                    # any nonzero is valid; processed pixels come out with valid = 1
    got = so.disparity_median_filter(d, 5)
    keep = np.ones(SHAPE, bool)
    keep[2:-2, 2:-2] = d[2:-2, 2:-2, 2] == 0
    assert np.array_equal(got[keep].view(np.int32), d[keep].view(np.int32))
    assert (got[~keep][:, 2] == 1).all()


def test_destructive_median_kat(so):
    """Math/tests/TestFunctors.cxx:111-121"""
    assert so.destructive_median([8, 9, 3, 5]) == 6.5
    assert S.destructive_median([8, 9, 3, 5]) == 6.5
    assert so.destructive_median([8, 9, 3]) == S.destructive_median([8, 9, 3]) == 8


def test_derivative_kat(oracle):
    """Image/tests/TestFilter.cxx:114-121: derivative_filter(src, 1, 0) of {1, 2; 3, 4} is 0.5 everywhere"""
    src = np.array([[1, 2], [3, 4]], F)
    k = np.array([0.5, 0, -0.5], F)
    assert (oracle.separable_convolve(src, k, []) == 0.5).all()
    assert (S.derivative(src, 1) == 0.5).all()
    assert (S.derivative(src, 0) == 1.0).all()
    rng = np.random.default_rng(4)
    img = (rng.random((9, 12)) * 100).astype(F)
    assert np.array_equal(oracle.separable_convolve(img, k, []), S.derivative(img, 1))
    assert np.array_equal(oracle.separable_convolve(img, [], k), S.derivative(img, 0))


# ---- the aliasing, by hand --------------------------------------------------------------------------------------------
def hand_disparity():
    """5 x 5, all valid but (1, 2); dy = dx / 2"""
    x = np.array([[0, 0, 0, 0, 0], [0, 4, 6, 1, 0], [0, 5, 2, 7, 0], [0, 3, 8, 9, 0], [0, 0, 0, 0, 0]], F)
    d = np.zeros((5, 5, 3), F)
    d[..., 0], d[..., 1], d[..., 2] = x, x / 2, 1
    d[2, 1, 2] = 0
    return d


# 3 x 3 median, in place: (1, 1) sees {0,0,0, 0,4,6, 0,2} (the invalid 5 left out): 8 values, (0 + 0) / 2 = 0; (2, 1) then
# sees the 0 just written, ...  A Jacobi filter (every window from the input) gives the second raster.
HAND_MEDIAN = np.array([[0, 0, 0, 0, 0], [0, 0, 0.5, 0, 0], [0, 5, 2.5, 0.5, 0], [0, 0, 0.25, 0, 0], [0, 0, 0, 0, 0]], F)
HAND_MEDIAN_JACOBI = np.array([[0, 0, 0, 0, 0], [0, 0, 1.5, 0, 0], [0, 5, 5, 2, 0], [0, 0, 2.5, 0, 0], [0, 0, 0, 0, 0]], F)
# texture filter with zero texture, texture_max 1, max_kernel_size 3: every valid pixel becomes its clamped 3 x 3 mean
HAND_TEXTURE = np.array([[0.44444445, 1.2098765, 1.4910836, 1.1091297, 0.35758436],
                         [0.7623457, 1.9884688, 2.72482, 1.7425131, 1.1740901],
                         [0.814145, 5.0, 4.4319754, 3.7859333, 1.8751807],
                         [0.5785363, 2.1030822, 3.415124, 2.5009127, 1.1152452],
                         [0.36223942, 0.7579135, 1.0594385, 1.0166843, 0.7516413]], F)


def test_hand_case_pins_in_place_raster_order(so):
    d = hand_disparity()
    got = so.disparity_median_filter(d, 3)
    assert np.array_equal(got[..., 0], HAND_MEDIAN) and np.array_equal(got[..., 1], HAND_MEDIAN / 2)
    assert np.array_equal(S.disparity_median_filter(d, 3)[..., 0], HAND_MEDIAN)
    assert np.array_equal(S.disparity_median_filter(d, 3, jacobi=True)[..., 0], HAND_MEDIAN_JACOBI)
    assert np.array_equal(got[..., 2], d[..., 2])
    t = np.zeros((5, 5), F)
    got = so.texture_preserving_disparity_filter(d, t, 1.0, 3)
    assert np.array_equal(got[..., 0], HAND_TEXTURE)
    assert np.array_equal(S.texture_preserving_disparity_filter(d, t, 1.0, 3)[..., 0], HAND_TEXTURE)
    assert not np.array_equal(S.texture_preserving_disparity_filter(d, t, 1.0, 3, jacobi=True)[..., 0], HAND_TEXTURE)


# ---- texture_measure ----------------------------------------------------------------------------------------------------
def texture_image(seed, shape):
    rng = np.random.default_rng(seed)
    img = (rng.random(shape) * 255).astype(F)
    img[: shape[0] // 2] = np.round(img[: shape[0] // 2])            # integer half: exact sums; float half: rounding
    return img


@pytest.mark.parametrize("k", [1, 2, 3, 4, 5, 9, 15])
@pytest.mark.parametrize("shape", [(17, 21), (1, 12), (12, 1), (3, 2)])
def test_texture_measure_matches_restatement(so, shape, k):
    img = texture_image(k * 13 + shape[0], shape)
    for gw, sw in ((0.5, 0.5), (1.0, 0.0), (0.3, 2.5)):
        assert same(so.texture_measure(img, k, gw, sw), S.texture_measure(img, k, gw, sw)), (gw, sw)


# ---- texture_preserving_disparity_filter ----------------------------------------------------------------------------------
def texture_case(seed, shape, invalid):
    """a disparity and a texture that covers every branch: negative texture, texture >= texture_max, texture giving
    kernels from 1 to max_k"""
    d = S.random_disparity(seed, shape, invalid)
    rng = np.random.default_rng(seed + 1)
    t = (rng.random(shape) * 0.2).astype(F)
    t[rng.random(shape) < 0.1] = -0.05
    t[rng.random(shape) < 0.1] = 0.15
    t[rng.random(shape) < 0.1] = 0.0
    return d, t


@pytest.mark.parametrize("tmax,maxk", [(0.15, 11), (0.15, 13), (0.15, 12), (0.2, 3), (0.05, 7), (0.0, 11), (-1.0, 11), (0.15, 2)])
@pytest.mark.parametrize("invalid", INVALID)
def test_texture_filter_matches_restatement(so, invalid, tmax, maxk):
    d, t = texture_case(200 + int(invalid * 10) + maxk, SHAPE, invalid)
    want = S.texture_preserving_disparity_filter(d, t, tmax, maxk)
    assert same(so.texture_preserving_disparity_filter(d, t, tmax, maxk), want)
    if tmax <= 0 or maxk < 3:
        assert np.array_equal(want.view(np.int32), d.view(np.int32))


def test_texture_filter_branches():
    """the kernel rule of Algorithms.h:243-257: negative texture skips, texture >= texture_max gives kernel 1 (skipped),
    floor(adj * scale) is made odd, kernels above max_kernel_size are skipped"""
    k = S.texture_kernel_size
    assert k(-0.01, 0.15, 11) is None and k(0.15, 0.15, 11) is None and k(0.5, 0.15, 11) is None
    assert k(0.0, 0.15, 11) == 11 and k(0.0, 0.15, 12) is None               # even max_k: floor gives 12, made 13 > 12
    assert k(0.0, 0.15, 13) == 13 and k(0.1, 0.15, 13) == 5
    assert k(float("nan"), 0.15, 11) is None


@pytest.mark.parametrize("shape", [(1, 25), (25, 1), (2, 2)])
def test_texture_filter_thin_images(so, shape):
    d, t = texture_case(77 + shape[0], shape, 0.1)
    assert same(so.texture_preserving_disparity_filter(d, t, 0.15, 11), S.texture_preserving_disparity_filter(d, t, 0.15, 11))


# ---- the C ABI without a device ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def vwb():
    from visionworkbench_b200 import build
    build.build()
    import visionworkbench_b200 as v
    return v


def test_abi_argument_validation(vwb):
    L = vwb.lib()
    d = np.zeros((8, 8, 3), F)
    img = np.zeros((8, 8), F)
    p, t = d.ctypes.data, img.ctypes.data
    assert L.vwb200_disparity_median_filter(None, 8, 8, 8, 3, 0, None) == -1
    assert L.vwb200_disparity_median_filter(p, 8, 8, 7, 3, 0, None) == -1              # pitch < cols
    assert L.vwb200_disparity_median_filter(p, -1, 8, 8, 3, 0, None) == -1
    assert L.vwb200_disparity_median_filter(p, 8, 8, 8, 32, 0, None) == -4             # above the supported 31
    assert L.vwb200_disparity_median_filter(p, 8, 8, 1 << 30, 3, 0, None) == -4         # pitch beyond the kernels' offsets
    assert L.vwb200_texture_measure(t, 8, 8, 8, 0, 0.5, 0.5, t, 8, 0, None) == -1       # kernel_size < 1
    assert L.vwb200_texture_measure(t, 8, 8, 8, -3, 0.5, 0.5, t, 8, 0, None) == -1
    assert L.vwb200_texture_measure(None, 8, 8, 8, 9, 0.5, 0.5, t, 8, 0, None) == -1
    assert L.vwb200_texture_measure(t, 8, 8, 8, 9, 0.5, 0.5, t, 7, 0, None) == -1       # opitch < cols
    assert L.vwb200_texture_measure(t, 8, 8, 8, 33, 0.5, 0.5, t, 8, 0, None) == -4
    assert L.vwb200_texture_preserving_disparity_filter(p, 8, 8, 8, None, 8, C.c_float(0.15), 11, 0, None) == -1
    assert L.vwb200_texture_preserving_disparity_filter(p, 8, 8, 8, t, 7, C.c_float(0.15), 11, 0, None) == -1
    assert L.vwb200_texture_preserving_disparity_filter(p, 8, 8, 8, t, 8, C.c_float(0.15), 33, 0, None) == -4
    with pytest.raises(vwb.ArgumentErr):
        vwb.disparity_median_filter(np.zeros((8, 8, 3), np.float64), 3)                # cannot be filtered in place
    with pytest.raises(vwb.ArgumentErr):
        vwb.texture_preserving_disparity_filter(d, np.zeros((8, 9), F))
    with pytest.raises(vwb.ArgumentErr):
        vwb.texture_measure(img, 0)
    with pytest.raises(vwb.NoImplErr):
        vwb.texture_measure(img, 32)


def test_abi_no_device(vwb):
    if vwb.device_count() > 0:
        pytest.skip("a CUDA device is present")
    d = np.zeros((8, 8, 3), F)
    img = np.zeros((8, 8), F)
    for call in (lambda: vwb.disparity_median_filter(d, 3), lambda: vwb.disparity_median_filter(d, 1),
                 lambda: vwb.texture_measure(img), lambda: vwb.texture_preserving_disparity_filter(d, img),
                 lambda: vwb.texture_preserving_disparity_filter(d, img, 0.0)):
        with pytest.raises(vwb.NoDeviceErr):
            call()
