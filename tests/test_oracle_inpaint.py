"""The hole-filling oracle (oracle/vw_inpaint_oracle.c) against the reference's known-answer tests, hand cases that pin each
step of fill_holes_grass, and the independent numpy restatement in inpaint_reference.py, bit for bit (raw bits, NaN == NaN)."""
import numpy as np
import pytest
from scipy import ndimage

from oracle import inpaint as oi
import inpaint_reference as ref


def bits(a):
    a = np.ascontiguousarray(a)
    if a.dtype == np.float32:
        b = a.view(np.uint32).copy()
        b[np.isnan(a)] = 0x7fc00000
        return b
    return a


def same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(bits(a), bits(b))


def field(w, h, density, dtype, seed, lo=-50, hi=50):
    """a disparity with random children (invalid pixels keep theirs) and the given fraction of invalid pixels"""
    rng = np.random.default_rng(seed)
    d = np.zeros((h, w, 3), dtype)
    if dtype == np.int32:
        d[..., :2] = rng.integers(lo, hi, (h, w, 2))
    else:
        d[..., :2] = rng.uniform(lo, hi, (h, w, 2)).astype(np.float32)
    d[..., 2] = (rng.random((h, w)) >= density).astype(dtype)
    return d


def valid_field(w, h, dtype, seed=0):
    d = field(w, h, 0.0, dtype, seed)
    return d


def punch(d, pts, child=None):
    for x, y in pts:
        d[y, x, 2] = 0
        if child is not None:
            d[y, x, :2] = child
    return d


def both(d, length, window=None):
    got, st = oi.fill_holes_grass(d, length, window, stats=True)
    want = ref.fill_holes_grass(d, length, window)
    assert same(got, want), f"oracle != numpy restatement (len {length}, window {window})"
    return got, st


# ---- the reference's known-answer tests ---------------------------------------------------------------------------------
def test_kat_grassfire_alpha():
    """TestAlgorithms.cxx:143-157"""
    im = np.zeros((5, 5), np.uint8)
    im[1:4, 1:4] = 255
    g = ref.grassfire(im)
    assert (g[0, 0], g[1, 1], g[2, 2], g[3, 3], g[4, 4], g[2, 1]) == (0, 1, 2, 1, 0, 1)


def test_kat_grassfire_no_border_distance():
    """TestAlgorithms.cxx:160-173 gives the city-block distance to the one zero pixel.  The bordered grassfire inpainting uses
    equals that distance wherever the mask's border is zero, as it is around every hole."""
    im = np.full((7, 7), 255, np.uint8)
    im[3, 3] = 0
    im[0, :] = im[-1, :] = im[:, 0] = im[:, -1] = 0
    g = ref.grassfire(im)
    want = ndimage.distance_transform_cdt(im != 0, metric="taxicab")
    assert np.array_equal(g, want)
    inner = ndimage.distance_transform_cdt(np.pad(np.full((5, 5), 1), 0) - (np.arange(25).reshape(5, 5) == 12), metric="taxicab")
    assert all(inner[r, c] == abs(2 - r) + abs(2 - c) for r in range(5) for c in range(5))


def test_kat_inpaint_view_three_blobs():
    """TestInpaintView.cxx:36-44: four marked pixels, three 8-connected blobs.  fill_holes_grass labels the invalid ones."""
    d = valid_field(5, 5, np.float32)
    punch(d, [(1, 2), (3, 1), (3, 3), (3, 4)])
    _, st = both(d, 100)
    assert st[0] == 3


# ---- hand cases -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.int32, np.float32])
def test_diagonal_holes_are_one_blob(dtype):
    d = valid_field(12, 12, dtype, 1)
    punch(d, [(5, 5), (6, 6)])
    got, st = both(d, 1)
    assert st[:2] == (1, 0)  # one blob, 2 x 2: wider than len 1
    got, st = both(d, 2)
    assert st[:2] == (1, 1) and got[5, 5, 2] == 1 and got[6, 6, 2] == 1


@pytest.mark.parametrize("dtype", [np.int32, np.float32])
def test_culls_at_their_limits(dtype):
    """A len x len square stays; one more pixel (over len*len, and a box over len) goes.  A box of width / height len stays
    and len + 1 goes.  With w, h <= len the pixel count is <= len*len, so the size cull never removes a hole the box cull keeps."""
    n = 4
    d = valid_field(16, 16, dtype, 2)
    punch(d, [(x, y) for x in range(5, 5 + n) for y in range(5, 5 + n)])
    _, st = both(d, n)
    assert st[:2] == (1, 1)
    punch(d, [(5 + n, 5)])
    _, st = both(d, n)
    assert st[:2] == (1, 0)
    for pts in ([(x, 7) for x in range(3, 3 + n)], [(7, y) for y in range(3, 3 + n)]):
        d = valid_field(16, 16, dtype, 3)
        punch(d, pts)
        assert both(d, n)[1][:2] == (1, 1)
        punch(d, [(pts[-1][0] + (pts[-1][1] == 7), pts[-1][1] + (pts[-1][0] == 7))])
        assert both(d, n)[1][:2] == (1, 0)


@pytest.mark.parametrize("dtype", [np.int32, np.float32])
def test_asymmetric_edge_skip(dtype):
    """A hole is skipped when it touches column / row 0, or reaches column cols-2 / row rows-2 (or beyond)."""
    w, h = 10, 9
    for pt, filled in [((0, 4), False), ((1, 4), True), ((w - 3, 4), True), ((w - 2, 4), False), ((w - 1, 4), False),
                       ((4, 0), False), ((4, 1), True), ((4, h - 3), True), ((4, h - 2), False), ((4, h - 1), False)]:
        d = valid_field(w, h, dtype, 4)
        punch(d, [pt])
        got, st = both(d, 3)
        assert st[:2] == (1, int(filled)), pt
        assert got[pt[1], pt[0], 2] == int(filled), pt


def test_first_sweep_reads_invalid_children():
    d = valid_field(12, 12, np.float32, 5)
    punch(d, [(5, 5), (6, 5)], child=(0.0, 0.0))
    zero, _ = both(d, 3)
    # the first pixel reads the second one's invalid child; the coupling decays by about .073^2 a sweep, so a huge child
    # still shows after the 10 sweeps
    d[5, 6, :2] = (1e30, -1e30)
    big, _ = both(d, 3)
    assert not np.array_equal(zero, big)
    d[5, 6, :2] = (np.nan, 3.0)
    nan, _ = both(d, 3)
    assert np.isnan(nan[5, 5, 0]) and np.isnan(nan[5, 6, 0]) and not np.isnan(nan[5, 5, 1])
    for child in [(1 << 29, -(1 << 29)), (7, -7)]:
        di = valid_field(12, 12, np.int32, 5)
        punch(di, [(5, 5), (6, 5)], child=child)
        both(di, 3)


def _stencil(nb, product):
    s = np.float32(0)
    for (dx, dy, wt), v in zip(ref.STENCIL, nb):
        p = np.float64(np.float32(wt) * np.float32(v)) if product == "float" else wt * np.float64(v)
        s = np.float32(np.float64(s) + p)
    return s


def test_product_precision():
    """Each product is in double (ProductType<double, float>), the sum is narrowed to float at each +=.  Find neighbours for
    which a float product would give other bits, and check the oracle follows the double reading."""
    rng = np.random.default_rng(6)
    for _ in range(1000):
        nb = rng.uniform(-100, 100, 8).astype(np.float32)
        if _stencil(nb, "double") != _stencil(nb, "float"):
            break
    else:
        pytest.fail("no discriminating neighbourhood found")
    d = valid_field(5, 5, np.float32, 6)
    for (dx, dy, _), v in zip(ref.STENCIL, nb):
        d[2 + dy, 2 + dx, 0] = v
    punch(d, [(2, 2)])
    got, _ = both(d, 1)
    assert got[2, 2, 0] == _stencil(nb, "double") and got[2, 2, 0] != _stencil(nb, "float")


def test_int32_truncation():
    for v, want in [(3, 3), (-3, -3)]:
        d = np.zeros((5, 5, 3), np.int32)
        d[..., 2] = 1
        d[1:4, 1:4, 0] = v
        d[1, 1, 0] = d[1, 3, 0] = 0  # two corners at 0: sum = v * (1 - 2 * .176765)
        punch(d, [(2, 2)])
        got, _ = both(d, 1)
        exact = v * (1 - 2 * .176765)
        assert got[2, 2, 0] == int(np.trunc(exact)) and abs(got[2, 2, 0]) < abs(exact), (v, got[2, 2, 0])


@pytest.mark.parametrize("dtype", [np.int32, np.float32])
def test_window_decides(dtype):
    """The tile is the window grown by len, so a hole is filled in one window and skipped in its neighbour."""
    d = valid_field(30, 10, dtype, 7)
    punch(d, [(20, 5)])
    a, _ = both(d, 1, (20, 0, 2, 10))
    b, _ = both(d, 1, (19, 0, 2, 10))
    assert a[5, 0, 2] == 1 and b[5, 1, 2] == 0
    whole, _ = both(d, 1)
    assert same(whole[:, 20:22], a)


@pytest.mark.parametrize("dtype", [np.int32, np.float32])
def test_len_0_and_1(dtype):
    d = field(20, 17, 0.3, dtype, 8)
    got, st = both(d, 0)
    assert same(got, d) and st[1] == 0  # wipe_big_blobs(0) removes every hole
    got, st = both(d, 1)
    assert st[2] in (0, 10)  # only single pixels are filled, one distance level


# ---- the numpy restatement on random fields -------------------------------------------------------------------------------
CASES = [(w, h, dens, length, seed) for seed, (w, h) in enumerate([(1, 1), (1, 9), (9, 1), (7, 5), (23, 17), (50, 31)])
         for dens, length in [(0.0, 3), (0.15, 2), (0.3, 4), (0.5, 6), (1.0, 3)]]


@pytest.mark.parametrize("dtype", [np.int32, np.float32])
@pytest.mark.parametrize("w,h,dens,length,seed", CASES)
def test_random_fields(w, h, dens, length, seed, dtype):
    d = field(w, h, dens, dtype, 100 + seed)
    both(d, length)
    if w > 4 and h > 4:
        both(d, length, (2, 1, w - 4, h - 3))
        both(d, length, (w // 2, h // 2, 1, 1))


@pytest.mark.parametrize("dtype", [np.int32, np.float32])
def test_round_holes(dtype):
    """Holes of diameter 2..8 (several distance levels) in a valid field"""
    d = field(40, 36, 0.0, dtype, 9)
    yy, xx = np.mgrid[:36, :40]
    for cx, cy, r in [(8, 8, 1.0), (25, 8, 2.2), (10, 25, 3.1), (28, 26, 4.0)]:
        d[(xx - cx) ** 2 + (yy - cy) ** 2 <= r * r, 2] = 0
    got, st = both(d, 9)
    assert st[1] == 4 and st[2] > 10
