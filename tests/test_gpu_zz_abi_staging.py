"""How every C ABI entry point that takes `on_device` moves a caller's rasters.  Each call runs with host arrays and with
CUDA tensors, with a NULL stream and with a side stream, and every raster the ABI takes a pitch for has rows wider than
the image.  Host and device results must be bit for bit the same (and the oracle's where there is one), and a sentinel in
the pitch padding of every buffer (inputs, outputs and in-out buffers) must be untouched.

The module sorts after the ones that trace kernels with torch.profiler (see test_gpu_wavefront_smoothing.py)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
PAD = 5                      # pixels of padding per row wherever the ABI takes a pitch
PLACES = [(False, False), (False, True), (True, False), (True, True)]      # (device tensors, side stream)
SENTINEL = {np.dtype(np.float32): -7.25, np.dtype(np.int32): -123456789, np.dtype(np.uint8): 0xA5}


@pytest.fixture(scope="module")
def vwb():
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "GPU tests need a CUDA device: the engine has no CPU path"
    return v


@pytest.fixture(scope="module")
def L(vwb):
    return vwb.lib()


class Place:
    """the buffers of one call: numpy arrays or CUDA tensors, each row followed by `pad` sentinel pixels"""

    def __init__(self, dev, side):
        import torch
        self.dev = dev
        self.flag = int(dev)
        self.bufs = []
        self.side = torch.cuda.Stream() if side else None
        self.stream = C.c_void_p(self.side.cuda_stream) if side else None

    def buf(self, a, pad=PAD):
        """(pointer, pitch in pixels) of a padded copy of `a` (rows, cols[, channels])"""
        import torch
        a = np.asarray(a)
        rows, cols = a.shape[:2]
        full = np.full((rows, cols + pad) + a.shape[2:], SENTINEL[a.dtype], a.dtype)
        full[:, :cols] = a
        if self.dev:
            full = torch.from_numpy(full).cuda()
            torch.cuda.synchronize()
        self.bufs.append((full, cols))
        return (full.data_ptr() if self.dev else full.ctypes.data), cols + pad

    def ptr(self, a):
        """pointer of a dense copy of `a`, for the arguments the ABI takes without a pitch"""
        return self.buf(a, 0)[0]

    def read(self, i):
        """buffer i without its padding, after checking that the padding still holds the sentinel"""
        full, cols = self.bufs[i]
        if not isinstance(full, np.ndarray):
            full = full.cpu().numpy()
        pad = full[:, cols:]
        want = np.full(pad.shape, SENTINEL[full.dtype], full.dtype)
        assert pad.tobytes() == want.tobytes(), f"buffer {i}: padding written"
        return full[:, :cols].copy()


def each_place(call):
    """run call(place) -> (rc, indices of the buffers it writes) at every placement; the results must be bit-identical"""
    got = []
    for dev, side in PLACES:
        p = Place(dev, side)
        rc, outs = call(p)
        assert rc == 0, (dev, side, rc)
        for i in range(len(p.bufs)):
            p.read(i)
        got.append([p.read(i) for i in outs])
    for place, res in zip(PLACES[1:], got[1:]):
        for a, b in zip(got[0], res):
            assert a.shape == b.shape and a.tobytes() == b.tobytes(), place
    return got[0]


def image(seed, shape, integer=True):
    a = np.random.default_rng(seed).random(shape, dtype=np.float32) * 255
    return np.floor(a) if integer else a


def zeros(shape, dtype=np.float32):
    return np.zeros(shape, dtype)


# ---- calc_disparity, pyramid, prefilter, mask subsampling -----------------------------------------------------------
@pytest.mark.parametrize("cost", [0, 1, 2])
@pytest.mark.parametrize("integer", [True, False])
def test_calc_disparity(L, cost, integer):
    import oracle
    from visionworkbench_b200.synth import make_rasters
    sx, sy, kx, ky = 9, 6, 5, 7
    left, right = make_rasters(61, 47, (sx, sy), (kx, ky), seed=3 + cost)
    if not integer:
        left, right = left + np.float32(0.25), right + np.float32(0.25)
    lh, lw = left.shape
    rw, rh = lw + sx - 1, lh + sy - 1
    right = right[:rh, :rw]
    H, W = lh - ky + 1, lw - kx + 1

    def call(p):
        lp, lpi = p.buf(left)
        rp, rpi = p.buf(right)
        op, opi = p.buf(zeros((H, W, 3), np.int32))
        return L.vwb200_calc_disparity(cost, lp, lw, lh, lpi, rp, rw, rh, rpi, sx, sy, kx, ky, op, opi, p.flag, p.stream), [2]
    (out,) = each_place(call)
    assert np.array_equal(out, oracle.calc_disparity(cost, left, right, (sx, sy), (kx, ky)))


def test_pyramid_down_and_mask_subsampling(L):
    import oracle
    img = image(1, (33, 47), integer=False)
    mask = ((image(2, (33, 47)) > 60) * 255).astype(np.uint8)

    def down(p):
        ip, ipi = p.buf(img)
        op, opi = p.buf(zeros((17, 24)))
        return L.vwb200_pyramid_down(ip, 47, 33, ipi, op, opi, p.flag, p.stream), [1]

    def sub(p):
        ip, ipi = p.buf(mask)
        op, opi = p.buf(zeros((17, 24), np.uint8))
        return L.vwb200_subsample_mask_by_two(ip, 47, 33, ipi, op, opi, p.flag, p.stream), [1]
    assert np.array_equal(each_place(down)[0], oracle.pyramid_down(img))
    assert np.array_equal(each_place(sub)[0], oracle.subsample_mask_by_two(mask))


@pytest.mark.parametrize("mode,width", [(0, 0.0), (1, 1.4), (2, 3.0)])
def test_prefilter(L, mode, width):
    import oracle
    img = image(4, (40, 53))

    def call(p):
        ip, ipi = p.buf(img)
        op, opi = p.buf(zeros(img.shape))
        return L.vwb200_prefilter(ip, 53, 40, ipi, mode, C.c_float(width), op, opi, p.flag, p.stream), [1]
    (out,) = each_place(call)
    assert np.array_equal(out, oracle.prefilter(img, mode, width))


# ---- SGM -----------------------------------------------------------------------------------------------------------------
def sgm_case():
    from visionworkbench_b200.synth import make_sgm_case
    left, right, prev, _ = make_sgm_case(48, 20, 5, seed=11)
    return left, right, prev


def sgm_size(L, left, right, search):
    ow, oh = C.c_int(0), C.c_int(0)
    assert L.vwb200_sgm_calc_disparity(left.ctypes.data, left.shape[1], left.shape[0], left.shape[1], right.ctypes.data, right.shape[1], right.shape[0],
                                       right.shape[1], search, search, 5, 0, 0, None, 0, C.byref(ow), C.byref(oh), 0, None) == 0
    return oh.value, ow.value


def test_sgm_calc_disparity(L):
    import oracle
    left, right, _ = sgm_case()
    h, w = sgm_size(L, left, right, 20)
    ow, oh = C.c_int(0), C.c_int(0)

    def call(p):
        lp, lpi = p.buf(left)
        rp, rpi = p.buf(right)
        op, opi = p.buf(zeros((h, w, 3), np.int32))
        return L.vwb200_sgm_calc_disparity(lp, left.shape[1], left.shape[0], lpi, rp, right.shape[1], right.shape[0], rpi, 20, 20, 5, 0, 0,
                                           op, opi, C.byref(ow), C.byref(oh), p.flag, p.stream), [2]
    (out,) = each_place(call)
    assert np.array_equal(out, oracle.sgm_calc_disparity(left, right, (20, 20), 5))


@pytest.mark.parametrize("mode", [2, 3])
def test_sgm_calc_disparity_subpixel(L, mode):
    import oracle
    left, right, _ = sgm_case()
    h, w = sgm_size(L, left, right, 20)
    ow, oh = C.c_int(0), C.c_int(0)

    def call(p):
        lp, lpi = p.buf(left)
        rp, rpi = p.buf(right)
        op, opi = p.buf(zeros((h, w, 3), np.int32))
        sp, spi = p.buf(zeros((h, w, 3)), PAD + 2)
        return L.vwb200_sgm_calc_disparity_subpixel(lp, left.shape[1], left.shape[0], lpi, rp, right.shape[1], right.shape[0], rpi, 20, 20, 5,
                                                    0, 0, mode, op, opi, sp, spi, C.byref(ow), C.byref(oh), p.flag, p.stream), [2, 3]
    out, sub = each_place(call)
    want, want_sub = oracle.sgm_calc_disparity_subpixel(left, right, (20, 20), 5, mode)
    assert np.array_equal(out, want) and np.array_equal(sub, want_sub)


def test_sgm_ex_and_disp_bounds(vwb, L):
    """masks, prior and boxes in; disparity, sub-pixel disparity and boxes out; then the boxes fed back with only the
    sub-pixel output requested (the integer output is then a device scratch buffer)"""
    left, right, prev = sgm_case()
    h, w = sgm_size(L, left, right, 20)
    lm = ((image(5, (h, w)) > 30) * 255).astype(np.uint8)
    rm = ((image(6, right.shape) > 30) * 255).astype(np.uint8)
    sp = vwb.api._sgm_params((20, 20), 5, subpixel_mode=5, conserve_level=1)
    ow, oh = C.c_int(0), C.c_int(0)

    def bounds(p):
        pp, ppi = p.buf(prev)
        lp, lpi = p.buf(lm)
        rp, rpi = p.buf(rm)
        bp = p.ptr(zeros((h, w, 4), np.int32))
        return L.vwb200_sgm_disp_bounds(C.byref(sp), pp, prev.shape[1], prev.shape[0], ppi, lp, lpi, rp, rm.shape[1], rm.shape[0], rpi,
                                        w, h, bp, p.flag, p.stream), [3]
    (b,) = each_place(bounds)

    def full(p):
        lp, lpi = p.buf(left)
        rp, rpi = p.buf(right)
        lmp, lmpi = p.buf(lm)
        rmp, rmpi = p.buf(rm)
        pp, ppi = p.buf(prev)
        op, opi = p.buf(zeros((h, w, 3), np.int32))
        sbp, sbpi = p.buf(zeros((h, w, 3)))
        bo = p.ptr(zeros((h, w, 4), np.int32))
        return L.vwb200_sgm_calc_disparity_ex(C.byref(sp), lp, left.shape[1], left.shape[0], lpi, rp, right.shape[1], right.shape[0], rpi,
                                              lmp, lmpi, rmp, rm.shape[1], rm.shape[0], rmpi, pp, prev.shape[1], prev.shape[0], ppi, None,
                                              op, opi, sbp, sbpi, bo, C.byref(ow), C.byref(oh), p.flag, p.stream), [5, 6, 7]
    out, sub, bo = each_place(full)
    assert np.array_equal(bo, b)
    want_out, want_sub = vwb.calc_disparity_sgm_ex(vwb.CENSUS_TRANSFORM, left, right, (20, 20), 5, subpixel_mode=5, left_mask=lm,
                                                   right_mask=rm, prev_disparity=prev, conserve_level=1)
    assert np.array_equal(out, want_out) and np.array_equal(sub, want_sub)

    def given_bounds(p):
        lp, lpi = p.buf(left)
        rp, rpi = p.buf(right)
        bp = p.ptr(b)
        sbp, sbpi = p.buf(zeros((h, w, 3)))
        return L.vwb200_sgm_calc_disparity_ex(C.byref(sp), lp, left.shape[1], left.shape[0], lpi, rp, right.shape[1], right.shape[0], rpi,
                                              None, 0, None, 0, 0, 0, None, 0, 0, 0, bp, None, 0, sbp, sbpi, None,
                                              C.byref(ow), C.byref(oh), p.flag, p.stream), [3]
    (sub2,) = each_place(given_bounds)
    assert np.array_equal(sub2, vwb.calc_disparity_sgm_ex(vwb.CENSUS_TRANSFORM, left, right, (20, 20), 5, subpixel_mode=5, bounds=b)[1])


# ---- ParabolaSubpixelView ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dest_pad", [0, PAD])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_parabola_subpixel(L, dest_pad, mode):
    import oracle
    from visionworkbench_b200.synth import make_pair
    left, right, _, _, _ = make_pair(64, 48, (-4, -3, 4, 3), seed=8)
    d = oracle.pyramid_correlate(oracle.make_params((-4, -3, 4, 3), (5, 5)), left, right)
    rows, cols = left.shape
    x0, y0, x1, y1 = 3, 2, 57, 41

    def call(p):
        dp = p.ptr(d)
        lp, lpi = p.buf(left)
        rp, rpi = p.buf(right)
        op, opi = p.buf(zeros((y1 - y0, x1 - x0, 3)), dest_pad)
        return L.vwb200_parabola_subpixel(dp, cols, rows, lp, lpi, rp, right.shape[1], right.shape[0], rpi, 5, 5, mode, C.c_float(1.5),
                                          x0, y0, x1, y1, op, opi, p.flag, p.stream), [3]
    (out,) = each_place(call)
    want = oracle.parabola_subpixel(d, left, right, (5, 5), mode, 1.5, (x0, y0, x1, y1))
    assert np.array_equal(out[..., 2], want[..., 2])
    np.testing.assert_allclose(out[..., :2], want[..., :2], rtol=0, atol=1e-5)


# ---- smoothing, consistency check, outlier filters -------------------------------------------------------------------------
def test_smoothing(L):
    import oracle.smoothing as so
    from test_oracle_smoothing import texture_case, texture_image
    so.build()
    d, t = texture_case(41, (57, 66), 0.1)
    img = texture_image(42, (57, 66))

    def median(p):
        dp, dpi = p.buf(d)
        return L.vwb200_disparity_median_filter(dp, 66, 57, dpi, 5, p.flag, p.stream), [0]

    def texture_filter(p):
        dp, dpi = p.buf(d)
        tp, tpi = p.buf(t, PAD + 3)
        return L.vwb200_texture_preserving_disparity_filter(dp, 66, 57, dpi, tp, tpi, C.c_float(0.15), 11, p.flag, p.stream), [0]

    def measure(p):
        ip, ipi = p.buf(img)
        op, opi = p.buf(zeros(img.shape), PAD + 1)
        return L.vwb200_texture_measure(ip, 66, 57, ipi, 9, C.c_double(0.5), C.c_double(0.5), op, opi, p.flag, p.stream), [1]
    assert np.array_equal(each_place(median)[0], so.disparity_median_filter(d, 5))
    assert np.array_equal(each_place(texture_filter)[0], so.texture_preserving_disparity_filter(d, t, 0.15, 11))
    assert np.array_equal(each_place(measure)[0], so.texture_measure(img, 9))


def random_disparity(seed, shape, invalid=0.2, r=4):
    rng = np.random.default_rng(seed)
    d = rng.integers(-r, r + 1, shape + (3,)).astype(np.int32)
    d[..., 2] = rng.random(shape) >= invalid
    return d


def test_consistency_check(L):
    import oracle
    l2r = random_disparity(50, (40, 50), r=2)
    r2l = random_disparity(51, (44, 55), r=2)

    def call(p):
        lp, lpi = p.buf(l2r)
        rp, rpi = p.buf(r2l, PAD + 2)
        return L.vwb200_cross_corr_consistency_check(lp, 50, 40, lpi, rp, 55, 44, rpi, C.c_float(1.0), p.flag, p.stream), [0]
    (out,) = each_place(call)
    assert np.array_equal(out, oracle.cross_corr_consistency_check(l2r, r2l, 1.0))


def test_outlier_filters_and_mask(L):
    import oracle
    d = random_disparity(60, (37, 45), invalid=0.1, r=3)
    lm = ((image(61, (37, 45)) > 40) * 255).astype(np.uint8)
    rm = ((image(62, (40, 50)) > 40) * 255).astype(np.uint8)

    def rm_outliers(p):
        ip, op = p.ptr(d), p.ptr(zeros(d.shape, np.int32))
        return L.vwb200_rm_outliers_using_thresh(ip, 45, 37, 2, 3, C.c_double(3.0), C.c_double(0.5), op, p.flag, p.stream), [1]

    def cleanup(p):
        ip, op = p.ptr(d), p.ptr(zeros(d.shape, np.int32))
        return L.vwb200_disparity_cleanup_using_thresh(ip, 45, 37, 2, 2, C.c_double(3.0), C.c_double(0.5), op, p.flag, p.stream), [1]

    def mask(p):
        ip, lp, rp, op = p.ptr(d), p.ptr(lm), p.ptr(rm), p.ptr(zeros(d.shape, np.int32))
        return L.vwb200_disparity_mask(ip, 45, 37, lp, rp, 50, 40, op, p.flag, p.stream), [3]
    assert np.array_equal(each_place(rm_outliers)[0], oracle.rm_outliers_using_thresh(d, 2, 3, 3.0, 0.5))
    assert np.array_equal(each_place(cleanup)[0], oracle.disparity_cleanup_using_thresh(d, 2, 2, 3.0, 0.5))
    assert np.array_equal(each_place(mask)[0], oracle.disparity_mask(d, lm, rm))


# ---- the view: inputs, dest and lr_disp_diff each on the host or the device -------------------------------------------------
VIEW_SEARCH, VIEW_KERNEL, REGION_UL = (-6, -4, 6, 4), (5, 5), (7, 3)


def view_case(dead_left=False):
    from visionworkbench_b200.synth import make_pair
    left, right, lm, rm, _ = make_pair(112, 96, VIEW_SEARCH, seed=21)
    if dead_left:
        lm = np.zeros_like(lm)
    diff = np.random.default_rng(22).random((100, 110, 2), dtype=np.float32)
    return left, right, lm, rm, diff


def run_view(L, vwb, p, inputs, diff_on_device, algorithm, bbox, case):
    """one rasterize of bbox; inputs: 0 host, 1 device, 2 streamed host rasters.  Buffers: 0-3 inputs, 4 diff, 5 dest"""
    import torch
    left, right, lm, rm, diff = case
    params = vwb.api.CorrParams(*VIEW_SEARCH, *VIEW_KERNEL, 3 if algorithm else 0, 0, 0.0, 1.0, 0, 2, 2, 0, 0, 0.0, algorithm, 0, 5, 2, 2,
                                *REGION_UL, 0, 4, 6000.0)
    h = C.c_void_p()
    assert L.vwb200_corr_create(C.byref(params), C.byref(h)) == 0
    try:
        dev_in, p.dev = p.dev, inputs == 1
        lp, lpi = p.buf(left)
        rp, rpi = p.buf(right)
        lmp, lmpi = p.buf(lm)
        rmp, rmpi = p.buf(rm)
        p.dev = diff_on_device
        dp, dpi = p.buf(diff, PAD + 1)
        p.dev = dev_in
        op, opi = p.buf(zeros((bbox[3] - bbox[1], bbox[2] - bbox[0], 3)))
        assert L.vwb200_corr_set_inputs(h, lp, 112, 96, lpi, rp, 112, 96, rpi, lmp, lmpi, rmp, rmpi, inputs) == 0
        assert L.vwb200_corr_set_lr_disp_diff(h, dp, 110, 100, dpi, int(diff_on_device)) == 0
        torch.cuda.synchronize()
        return L.vwb200_corr_rasterize(h, *bbox, op, opi, p.flag, p.stream)
    finally:
        L.vwb200_corr_destroy(h)


def read_view(p):
    """(dest, lr_disp_diff) of run_view, after checking the padding of every buffer"""
    for i in range(len(p.bufs)):
        p.read(i)
    return p.read(5), p.read(4)


@pytest.mark.parametrize("algorithm", [0, 1])
def test_view_placements(vwb, L, algorithm):
    import oracle
    case = view_case()
    left, right, lm, rm, diff = case
    bbox = (9, 5, 101, 83)
    got = {}
    for inputs in (0, 1, 2):
        for dest_dev in (False, True):
            for diff_dev in (False, True):
                side = (inputs + dest_dev + diff_dev) % 2 == 1
                p = Place(dest_dev, side)
                assert run_view(L, vwb, p, inputs, diff_dev, algorithm, bbox, case) == 0, (inputs, dest_dev, diff_dev)
                got[inputs, dest_dev, diff_dev] = read_view(p)
    first = got[0, False, False]
    for key, res in got.items():
        assert all(a.tobytes() == b.tobytes() for a, b in zip(first, res)), key
    if algorithm == 0:
        p = oracle.make_params(VIEW_SEARCH, VIEW_KERNEL, consistency_threshold=1.0, filter_half_kernel=2, max_pyramid_levels=2)
        want_diff = diff.copy()
        want = oracle.pyramid_correlate(p, left, right, lm, rm, bbox, want_diff, REGION_UL)
        assert np.array_equal(first[0], want) and np.array_equal(first[1], want_diff)
    assert not np.array_equal(first[1], diff)          # the check wrote into the tile's window


def test_view_all_invalid_tile_keeps_lr_disp_diff(vwb, L):
    """a tile whose left mask is all zero is all invalid: the lr_disp_diff window is left as it was, on the host and the device"""
    case = view_case(dead_left=True)
    for inputs, dest_dev, diff_dev in ((0, False, False), (1, True, True), (0, True, False), (1, False, True)):
        p = Place(dest_dev, inputs == 1)
        assert run_view(L, vwb, p, inputs, diff_dev, 0, (9, 5, 101, 83), case) == 0
        dest, diff = read_view(p)
        assert not dest.any() and diff.tobytes() == case[4].tobytes()
