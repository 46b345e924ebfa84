"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on the same inputs.
Bit-exact for integer disparities / validity / pyramid floats (float ops are issued in the
reference's order with no FMA contraction)."""
import numpy as np
import pytest

from kernel_trace import trace  # noqa: F401  (the profiler fixture: the kernels a call ran)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def vwb():
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "GPU tests need a CUDA device"
    return v


def _assert_disp_equal(got, ref, what=""):
    got = np.asarray(got)
    ref = np.asarray(ref)
    assert got.shape == ref.shape, what
    gv, rv = got[..., 2] != 0, ref[..., 2] != 0
    nbad_valid = int((gv != rv).sum())
    both = gv & rv
    nbad_d = int(((got[..., 0] != ref[..., 0]) | (got[..., 1] != ref[..., 1]))[both].sum())
    assert nbad_valid == 0 and nbad_d == 0, f"{what}: {nbad_valid} validity mismatches, {nbad_d} disparity mismatches of {gv.size}"
    # children of invalid pixels are observable through PixelMask::child(): keep them equal too
    assert np.array_equal(got[..., :2], ref[..., :2]), f"{what}: children of invalid pixels differ"


def _known_shift(rng, scale):
    left = np.floor(rng.random((25, 25)) * scale).astype(np.float32) if scale > 1 else rng.random((25, 25)).astype(np.float32)
    ys = np.clip(np.arange(46) - 8, 0, 24)
    xs = np.clip(np.arange(31) - 3, 0, 24)
    return left, left[np.ix_(ys, xs)]


@pytest.mark.parametrize("cost", [0, 1, 2])
@pytest.mark.parametrize("scale", [255.0, 32767.0, 1.0])
def test_calc_disparity_reference_kat(vwb, oracle, cost, scale):
    """Stereo/tests/TestCorrelation.cxx:45-65: shift (3,8), kernel 7x5, search 7x12."""
    left, right = _known_shift(np.random.default_rng(10), scale)
    d = vwb.calc_disparity(cost, left, right, (7, 12), (7, 5))
    assert d.shape == (21, 19, 3)
    assert (d[..., 2] == 1).all() and (d[..., 0] == 3).all() and (d[..., 1] == 8).all()
    _assert_disp_equal(d, oracle.calc_disparity(cost, left, right, (7, 12), (7, 5)))


@pytest.mark.parametrize("cost", [0, 1, 2])
@pytest.mark.parametrize("shape", [((96, 70), (9, 7), (7, 7)), ((200, 130), (33, 33), (15, 15)), ((64, 64), (1, 1), (5, 5)),
                                   ((37, 41), (5, 1), (3, 9)), ((130, 90), (16, 20), (21, 21))])
def test_calc_disparity_matches_oracle(vwb, oracle, cost, shape):
    from visionworkbench_b200.synth import make_rasters
    (W, H), search, kernel = shape
    left, right = make_rasters(W, H, search, kernel, seed=101 + cost)
    got = vwb.calc_disparity(cost, left, right, search, kernel)
    ref = oracle.calc_disparity(cost, left, right, search, kernel)
    _assert_disp_equal(got, ref, f"cost {cost} {shape}")


@pytest.mark.parametrize("cost", [0, 1, 2])
def test_calc_disparity_general_float_inputs(vwb, oracle, cost):
    """Non-integer imagery (what pyramid levels look like): fp64 path; values are multiples of 2^-8."""
    rng = np.random.default_rng(5)
    W, H, search, kernel = 80, 60, (9, 9), (9, 9)
    right = (np.floor(rng.random((H + 16, W + 16)) * 4096 * 256) / 256).astype(np.float32)
    left = np.ascontiguousarray(right[3:3 + H + 8, 5:5 + W + 8]) + (np.floor(rng.random((H + 8, W + 8)) * 512) / 256).astype(np.float32)
    got = vwb.calc_disparity(cost, left, right, search, kernel)
    ref = oracle.calc_disparity(cost, left, right, search, kernel)
    _assert_disp_equal(got, ref)


def test_calc_disparity_constant_image_is_invalid(vwb, oracle):
    """Correlation.cc:121-133: every disparity gives the same cost -> invalid."""
    left = np.full((30, 30), 7.0, np.float32)
    right = np.full((34, 34), 7.0, np.float32)
    for cost in (0, 1, 2):
        got = vwb.calc_disparity(cost, left, right, (5, 5), (5, 5))
        ref = oracle.calc_disparity(cost, left, right, (5, 5), (5, 5))
        _assert_disp_equal(got, ref)
    assert not vwb.calc_disparity(0, left, right, (5, 5), (5, 5))[..., 2].any()


def test_calc_disparity_ncc_zero_windows(vwb, oracle):
    """NCC with zero-energy windows: 1/0 = inf, inf*0 = NaN; the reference's best/worst state machine is
    order dependent (Correlation.cc:97-117).  The GPU replays it for flagged pixels."""
    rng = np.random.default_rng(3)
    right = np.floor(rng.random((50, 50)) * 255).astype(np.float32)
    right[:, :18] = 0
    right[20:40, 25:45] = 0
    left = np.ascontiguousarray(right[2:2 + 40, 3:3 + 40])
    left[5:25, 5:30] = 0
    got = vwb.calc_disparity(2, left, right, (8, 8), (7, 7))
    ref = oracle.calc_disparity(2, left, right, (8, 8), (7, 7))
    _assert_disp_equal(got, ref)


def test_pyramid_down_bit_exact(vwb, oracle):
    rng = np.random.default_rng(11)
    for shape in [(64, 64), (65, 97), (3, 5), (1, 1), (2, 7), (300, 211)]:
        img = (rng.random(shape) * 4096).astype(np.float32)     # arbitrary floats: rounding on every op
        a = vwb.pyramid_down(img)
        b = oracle.pyramid_down(img)
        assert a.shape == b.shape
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), shape
    # three levels deep
    img = np.floor(rng.random((257, 301)) * 4096).astype(np.float32)
    a, b = img, img
    for _ in range(3):
        a, b = vwb.pyramid_down(a), oracle.pyramid_down(b)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_subsample_mask(vwb, oracle):
    rng = np.random.default_rng(12)
    for shape in [(64, 64), (65, 97), (1, 1), (2, 7)]:
        m = (rng.random(shape) > 0.5).astype(np.uint8) * 255
        assert np.array_equal(vwb.subsample_mask_by_two(m), oracle.subsample_mask_by_two(m))


def _random_disp(rng, h, w, invalid_frac=0.2, spread=6):
    d = np.zeros((h, w, 3), np.int32)
    d[..., 0] = rng.integers(-spread, spread + 1, (h, w))
    d[..., 1] = rng.integers(-spread, spread + 1, (h, w))
    d[..., 2] = rng.random((h, w)) > invalid_frac
    return d


def test_consistency_check(vwb, oracle):
    rng = np.random.default_rng(13)
    l2r = _random_disp(rng, 40, 50)
    r2l = _random_disp(rng, 46, 58)
    for thr in (0, 1, 2):
        _assert_disp_equal(vwb.cross_corr_consistency_check(l2r, r2l, thr), oracle.cross_corr_consistency_check(l2r, r2l, thr))


@pytest.mark.parametrize("r", [1, 2, 5])
def test_outlier_filters(vwb, oracle, r):
    rng = np.random.default_rng(14 + r)
    for shape in [(40, 50), (7, 9), (100, 33)]:
        d = _random_disp(rng, *shape, spread=4)
        _assert_disp_equal(vwb.rm_outliers_using_thresh(d, r, r, 3.0, 0.5), oracle.rm_outliers_using_thresh(d, r, r, 3.0, 0.5), "rm_outliers")
        _assert_disp_equal(vwb.disparity_cleanup_using_thresh(d, r, r, 3.0, 0.5), oracle.disparity_cleanup_using_thresh(d, r, r, 3.0, 0.5), "cleanup")


def test_disparity_mask(vwb, oracle):
    rng = np.random.default_rng(15)
    d = _random_disp(rng, 40, 50, spread=8)
    lm = (rng.random((40, 50)) > 0.1).astype(np.uint8) * 255
    rm = (rng.random((45, 56)) > 0.1).astype(np.uint8) * 255
    _assert_disp_equal(vwb.disparity_mask(d, lm, rm), oracle.disparity_mask(d, lm, rm))


def _view_case(vwb, oracle, W, H, search, kernel, cost, levels, consistency, fhk, seed, bbox=None, collar=0, masks=True):
    from visionworkbench_b200.synth import make_pair
    left, right, lm, rm, _ = make_pair(W, H, search, seed, dropout=0.03 if masks else 0.0)
    view = vwb.pyramid_correlate(left, right, lm, rm, vwb.PREFILTER_NONE, 0.0, search, kernel, cost, 0, 0.0,
                                 consistency, 0, fhk, levels, collar_size=collar)
    got = view.rasterize(None, bbox)
    p = oracle.make_params(search, kernel, cost=cost, consistency_threshold=consistency, filter_half_kernel=fhk,
                           max_pyramid_levels=levels, collar_size=collar)
    ref = oracle.pyramid_correlate(p, left, right, lm, rm, bbox=bbox)
    _assert_disp_equal(got, ref, f"view cost={cost} levels={levels} bbox={bbox}")
    return got


@pytest.mark.parametrize("cost", [0, 1, 2])
def test_view_single_level(vwb, oracle, cost):
    """BASELINE config 1 shape at reduced size: pyramid_correlate(max_pyramid_levels=0)."""
    _view_case(vwb, oracle, 160, 128, (-8, -8, 8, 8), (7, 7), cost, 0, -1.0, 0, seed=101)


@pytest.mark.parametrize("cost", [0, 1, 2])
def test_view_pyramid_full_pipeline(vwb, oracle, cost):
    """5 levels requested, L/R check, outlier filters, masks: the whole prerasterize()."""
    got = _view_case(vwb, oracle, 300, 260, (-20, -12, 24, 16), (7, 7), cost, 5, 2.0, 5, seed=103)
    assert got[..., 2].mean() > 0.5


def test_view_tile_bboxes_and_collar(vwb, oracle):
    """Parity is defined per bbox (pyramid phase depends on the tile origin, CorrelationView.cc:89-93)."""
    for bbox in [(0, 0, 128, 128), (128, 64, 300, 200), (37, 41, 165, 169), (-16, -16, 64, 64), (250, 200, 330, 290)]:
        _view_case(vwb, oracle, 320, 280, (-10, -6, 14, 10), (9, 9), 0, 3, 2.0, 3, seed=104, bbox=bbox)
    _view_case(vwb, oracle, 320, 280, (-10, -6, 14, 10), (9, 9), 1, 3, 2.0, 3, seed=105, bbox=(64, 64, 192, 192), collar=16)


def test_view_fully_masked_tile_is_all_invalid(vwb, oracle):
    from visionworkbench_b200.synth import make_pair
    left, right, lm, rm, _ = make_pair(200, 200, (-4, -4, 4, 4), 7, dropout=0)
    lm[:] = 0
    view = vwb.pyramid_correlate(left, right, lm, rm, 0, 0.0, (-4, -4, 4, 4), (7, 7), 0, 0, 0.0, 2.0, 0, 3, 2)
    got = view.rasterize(None, (0, 0, 100, 100))
    assert (got == 0).all()                                     # CorrelationView.cc:321-331
    with pytest.raises(vwb.NoImplErr):
        view(0, 0)


def test_view_is_reentrant(vwb, oracle):
    """prerasterize is called concurrently from the tile thread pool (Image/ImageIO.h:228-235)."""
    import threading
    from visionworkbench_b200.synth import make_pair
    search, kernel = (-6, -6, 6, 6), (7, 7)
    left, right, lm, rm, _ = make_pair(256, 256, search, 9)
    view = vwb.pyramid_correlate(left, right, lm, rm, 0, 0.0, search, kernel, 0, 0, 0.0, 2.0, 0, 3, 3)
    boxes = [(x, y, x + 128, y + 128) for y in (0, 128) for x in (0, 128)]
    res = {}

    def work(b):
        res[b] = view.rasterize(None, b)
    ts = [threading.Thread(target=work, args=(b,)) for b in boxes]
    [t.start() for t in ts]
    [t.join() for t in ts]
    p = oracle.make_params(search, kernel, consistency_threshold=2.0, filter_half_kernel=3, max_pyramid_levels=3)
    for b in boxes:
        _assert_disp_equal(res[b], oracle.pyramid_correlate(p, left, right, lm, rm, bbox=b), f"threaded {b}")


def test_device_tensor_path(vwb, oracle):
    import torch
    from visionworkbench_b200.synth import make_rasters
    left, right = make_rasters(100, 80, (12, 10), (9, 9), seed=21)
    dl, dr = torch.from_numpy(left).cuda(), torch.from_numpy(right).cuda()
    got = vwb.calc_disparity(0, dl, dr, (12, 10), (9, 9))
    assert got.is_cuda
    _assert_disp_equal(got.cpu().numpy(), oracle.calc_disparity(0, left, right, (12, 10), (9, 9)))


@pytest.mark.parametrize("side_stream", [False, True])
def test_device_inputs_are_ordered_after_their_producer(vwb, oracle, side_stream):
    """ADVICE r1 (medium): device-resident inputs are produced on the caller's stream -- torch's default stream is the NULL
    (legacy) stream -- and the engine must run after the producer.  A long matmul is queued in front of the copy that gives
    the rasters their content; an engine that ran on a private stream would read the zeros underneath."""
    import torch
    from visionworkbench_b200.synth import make_rasters
    left, right = make_rasters(160, 120, (16, 12), (9, 9), seed=23)
    ref = oracle.calc_disparity(0, left, right, (16, 12), (9, 9))
    hl, hr = torch.from_numpy(left).pin_memory(), torch.from_numpy(right).pin_memory()
    big = torch.randn(8192, 8192, device="cuda")
    stream = torch.cuda.Stream() if side_stream else torch.cuda.current_stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        dl, dr = torch.zeros(left.shape, device="cuda"), torch.zeros(right.shape, device="cuda")
        for _ in range(4):
            big = big @ big * 1e-4                      # tens of milliseconds of queued work
        dl.copy_(hl, non_blocking=True)
        dr.copy_(hr, non_blocking=True)
        got = vwb.calc_disparity(0, dl, dr, (16, 12), (9, 9))
    _assert_disp_equal(got.cpu().numpy(), ref)


@pytest.mark.parametrize("shape", [((300, 70), (16, 8), (21, 21)), ((500, 40), (32, 4), (7, 7)), ((237, 33), (64, 3), (15, 15)),
                                   ((64, 64), (8, 8), (3, 5)), ((260, 100), (128, 2), (21, 21)), ((473, 65), (24, 11), (31, 9))])
def test_calc_disparity_exact_int_fast_path(vwb, oracle, shape):
    """The exact-integer TMA/shuffle kernel (k1_fast) must be bit-identical to the oracle: strips (W > 236),
    bands (H > 32), ragged edges, ties (first disparity in raster order wins)."""
    from visionworkbench_b200.synth import make_rasters
    (W, H), search, kernel = shape
    left, right = make_rasters(W, H, search, kernel, seed=7 + W)
    got = vwb.calc_disparity(0, left, right, search, kernel)
    assert vwb.last_k1_stats()["path"] == "exact-int"
    ref = oracle.calc_disparity(0, left, right, search, kernel)
    _assert_disp_equal(got, ref, f"fast {shape}")


def test_fast_path_ties_and_constant_regions(vwb, oracle):
    """8-bit imagery with flat regions: many exact ties and all-equal (invalid) pixels."""
    rng = np.random.default_rng(77)
    W, H, search, kernel = 280, 70, (16, 8), (7, 7)
    right = np.floor(rng.random((H + 6 + 7, W + 6 + 15)) * 4).astype(np.float32)    # 2-bit noise: ties everywhere
    right[20:60, 40:200] = 3.0                                                        # flat block: all-equal costs
    left = np.ascontiguousarray(right[2:2 + H + 6, 5:5 + W + 6])
    got = vwb.calc_disparity(0, left, right, search, kernel)
    assert vwb.last_k1_stats()["path"] == "exact-int"
    ref = oracle.calc_disparity(0, left, right, search, kernel)
    assert (ref[..., 2] == 0).any() and (ref[..., 2] == 1).any()
    _assert_disp_equal(got, ref, "ties")


@pytest.mark.parametrize("mode,width", [(1, 1.4), (2, 1.4), (1, 0.7), (2, 3.0)])
def test_prefilter_bit_exact(vwb, oracle, mode, width):
    """Stereo/PreFilter.h:45-95: LoG and subtracted-mean prefilters, identical float op order."""
    rng = np.random.default_rng(31)
    for shape in [(64, 80), (5, 3), (131, 77)]:
        img = (rng.random(shape) * 4096).astype(np.float32)
        a = vwb.prefilter_image(img, mode, width)
        b = oracle.prefilter(img, mode, width)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (mode, width, shape)


@pytest.mark.parametrize("mode", [1, 2])
def test_view_with_prefilter(vwb, oracle, mode):
    """correlate's default is PREFILTER_LOG 1.4 (tools/correlate.cc:210): full pipeline on prefiltered pyramids."""
    from visionworkbench_b200.synth import make_pair
    search, kernel = (-10, -6, 14, 10), (9, 9)
    left, right, lm, rm, _ = make_pair(260, 230, search, 41)
    view = vwb.pyramid_correlate(left, right, lm, rm, mode, 1.4, search, kernel, 0, 0, 0.0, 2.0, 0, 3, 3)
    got = view.rasterize(None, (0, 0, 260, 230))
    p = oracle.make_params(search, kernel, cost=0, prefilter_mode=mode, prefilter_width=1.4, consistency_threshold=2.0,
                           filter_half_kernel=3, max_pyramid_levels=3)
    ref = oracle.pyramid_correlate(p, left, right, lm, rm)
    _assert_disp_equal(got, ref, f"prefilter {mode}")


def _subpixel_case(rng, W=120, H=90, stretch=0.95):
    base = np.floor(rng.random((H, W + 20)) * 1024).astype(np.float32)
    base = np.floor((base + np.roll(base, 1, 0) + np.roll(base, 1, 1) + np.roll(base, -1, 0) + np.roll(base, -1, 1)) / 5)
    left = np.ascontiguousarray(base[:, :W])
    xs = np.arange(W) * stretch
    x0 = np.floor(xs).astype(int)
    f = (xs - x0).astype(np.float32)
    right = np.floor(base[:, np.clip(x0, 0, W + 18)] * (1 - f) + base[:, np.clip(x0 + 1, 0, W + 18)] * f).astype(np.float32)
    true = np.arange(W) / stretch - np.arange(W)
    disp = np.zeros((H, W, 3), np.float32)
    disp[..., 0] = np.rint(true)[None, :]
    disp[..., 1] = rng.integers(-1, 2, (H, W))
    disp[..., 2] = rng.random((H, W)) > 0.1
    return disp, left, right


@pytest.mark.parametrize("mode,width", [(0, 0.0), (1, 1.4), (2, 1.4)])
def test_parabola_subpixel(vwb, oracle, mode, width):
    """Stereo/ParabolaSubpixelView.cc:31-330 (a11).  north_star: sub-pixel floats agree within 1e-5; validity and
    the untouched integer parts are exact.  bboxes touch the image border (edge-extended prefilter semantics)."""
    rng = np.random.default_rng(51)
    disp, left, right = _subpixel_case(rng)
    view = vwb.parabola_subpixel(disp, left, right, mode, width, (7, 7))
    for bbox in [(0, 0, 120, 90), (10, 5, 70, 60), (64, 32, 120, 90)]:
        got = view.rasterize(None, bbox)
        ref = oracle.parabola_subpixel(disp, left, right, (7, 7), mode, width, bbox)
        assert np.array_equal(got[..., 2], ref[..., 2])
        np.testing.assert_allclose(got[..., :2], ref[..., :2], rtol=0, atol=1e-5)
    with pytest.raises(vwb.NoImplErr):
        view(0, 0)


def test_parabola_subpixel_reference_kat(vwb):
    """Stereo/tests/TestSubPixel.cxx:95-139: constant images leave (1,1) untouched; a 95 % stretch is recovered with
    mean error well below the integer rounding error (< 0.6 px in the reference test)."""
    const = np.full((50, 50), 7.0, np.float32)
    d = np.zeros((50, 50, 3), np.float32)
    d[..., 0] = 1; d[..., 1] = 1; d[..., 2] = 1
    o = vwb.parabola_subpixel(d, const, const, 0, 0.0, (7, 7)).rasterize()
    assert np.abs(o[..., :2] - 1).max() <= 0.1 and (o[..., 2] == 1).all()
    rng = np.random.default_rng(52)
    disp, left, right = _subpixel_case(rng)
    disp[..., 1] = 0; disp[..., 2] = 1
    o = vwb.parabola_subpixel(disp, left, right, 0, 0.0, (7, 7)).rasterize()
    true = np.arange(120) / 0.95 - np.arange(120)
    err = np.abs(o[10:80, 10:100, 0] - true[None, 10:100]).mean()
    assert err < 0.6 and err < np.abs(np.rint(true) - true)[10:100].mean()


def test_generic_kernel_unsplit_large_search(vwb, oracle, trace):
    """1200 disparities on float imagery: the generic kernel splits the zone into five chunks of 256 disparities
    (40 * 24 * 5 partial results are far below the 2^29 scratch limit) and k1_generic_merge_kernel must find the matches
    that lie beyond the first chunk (regression: a CTA covered only the first 256 disparities).  An unsplit zone of this
    many disparities needs a scratch of 2^29 elements, beyond what a test raster here reaches."""
    from visionworkbench_b200.synth import make_rasters
    W, H, search, kernel = 40, 24, (40, 30), (5, 5)
    left, right = make_rasters(W, H, search, kernel, seed=77)
    left, right = left + 0.5, right + 0.5                   # not integer valued: the generic kernel, same SquaredCost costs
    got = trace.run(lambda: vwb.calc_disparity(1, left, right, search, kernel))
    exp = trace.assert_hot(1, left, right, search, kernel)
    assert exp.family == "k1_generic_kernel" and exp.geom["nchunks"] == 5
    assert [k[0] for k in trace.merges()] == ["k1_generic_merge_kernel"]
    ref = oracle.calc_disparity(1, left, right, search, kernel)
    _assert_disp_equal(got, ref)
    assert (ref[..., 0] + ref[..., 1] * 40).max() > 256     # the true matches lie beyond the first chunk


@pytest.mark.parametrize("consistency", [-1.0, 2.0])
def test_view_single_level_uses_fast_kernel(vwb, oracle, consistency):
    """pyramid_correlate(max_pyramid_levels=0) on integer imagery: one big zone with a (search+1)^2 window
    (CorrelationView.cc:338-342) -> exact-integer fast kernel incl. the partial last dx octet, the R->L pass with
    edge-extended reads and the output offsets; masked pixels keep the tile on the general kernel."""
    from visionworkbench_b200.synth import make_pair
    search, kernel = (-20, -7, 12, 9), (9, 9)        # 33 x 17 window after the +1: not a multiple of 8
    left, right, lm, rm, _ = make_pair(420, 300, search, 61, dropout=0.0)
    view = vwb.pyramid_correlate(left, right, lm, rm, 0, 0.0, search, kernel, 0, 0, 0.0, consistency, 0, 3, 0)
    p = oracle.make_params(search, kernel, cost=0, consistency_threshold=consistency, filter_half_kernel=3, max_pyramid_levels=0)
    for bbox in [(0, 0, 420, 300), (100, 60, 400, 290)]:
        n0 = vwb.kernel_launches()
        got = view.rasterize(None, bbox)
        ref = oracle.pyramid_correlate(p, left, right, lm, rm, bbox=bbox)
        _assert_disp_equal(got, ref, f"single level fast {bbox}")


@pytest.mark.parametrize("shape", [((300, 70), (16, 8), (21, 21)), ((260, 100), (33, 5), (7, 7)), ((473, 65), (24, 11), (15, 9))])
def test_calc_disparity_exact_int_fast_path_squared(vwb, oracle, trace, shape):
    """SquaredCost on K1 fast: uint32 window sums, compare/select arg-min.  The imagery is capped at 3000 so that every
    shape stays on K1 fast (441 * 3000^2 < 2^32 at 21 x 21; a range of 3121 or more would take K1 screen)."""
    from visionworkbench_b200.synth import make_rasters
    (W, H), search, kernel = shape
    left, right = make_rasters(W, H, search, kernel, seed=17 + W)
    left, right = np.minimum(left, 3000.0), np.minimum(right, 3000.0)
    got = trace.run(lambda: vwb.calc_disparity(1, left, right, search, kernel))
    assert vwb.last_k1_stats()["path"] == "exact-int"
    assert trace.assert_hot(1, left, right, search, kernel).family == "k1_fast_abs_kernel"
    _assert_disp_equal(got, oracle.calc_disparity(1, left, right, search, kernel), f"fast sq {shape}")
    # range too large for uint32 sums -> general kernel, same answer
    big = left * 16.0
    bigr = right * 16.0
    got = vwb.calc_disparity(1, big, bigr, search, kernel)
    assert vwb.last_k1_stats()["path"] == "general-fp64"
    _assert_disp_equal(got, oracle.calc_disparity(1, big, bigr, search, kernel), f"generic sq {shape}")


@pytest.mark.parametrize("shape", [((300, 70), (16, 8), (21, 21)), ((260, 100), (33, 5), (7, 7)), ((473, 65), (24, 11), (15, 9)),
                                   ((64, 64), (8, 8), (3, 5)), ((250, 40), (128, 2), (21, 21))])
def test_calc_disparity_exact_int_fast_path_ncc(vwb, oracle, shape):
    """NCC on the exact-integer kernel (k1_screen): integer numerators, fp32 upper-bound screening, exact double
    evaluation (reference arithmetic) of the surviving candidates."""
    from visionworkbench_b200.synth import make_rasters
    (W, H), search, kernel = shape
    left, right = make_rasters(W, H, search, kernel, seed=11 + W)
    got = vwb.calc_disparity(2, left, right, search, kernel)
    assert vwb.last_k1_stats()["path"] == "exact-int"
    ref = oracle.calc_disparity(2, left, right, search, kernel)
    _assert_disp_equal(got, ref, f"fast ncc {shape}")


def test_fast_ncc_ties_zero_windows_and_constant_regions(vwb, oracle):
    """2-bit imagery: exact cost ties (first disparity in raster order wins), zero-energy windows (NaN state machine),
    flat regions (all-equal -> invalid)."""
    rng = np.random.default_rng(78)
    W, H, search, kernel = 280, 70, (16, 8), (7, 7)
    right = np.floor(rng.random((H + 6 + 7, W + 6 + 15)) * 4).astype(np.float32)
    right[20:60, 40:120] = 3.0
    right[10:50, 150:230] = 0.0
    left = np.ascontiguousarray(right[2:2 + H + 6, 5:5 + W + 6])
    left[40:70, 10:60] = 0.0
    got = vwb.calc_disparity(2, left, right, search, kernel)
    assert vwb.last_k1_stats()["path"] == "exact-int"
    ref = oracle.calc_disparity(2, left, right, search, kernel)
    assert (ref[..., 2] == 0).any() and (ref[..., 2] == 1).any()
    _assert_disp_equal(got, ref, "ncc ties")


@pytest.mark.parametrize("shape", [((300, 70), (16, 8), (21, 21)), ((260, 100), (33, 5), (7, 7)), ((250, 40), (128, 2), (21, 21)),
                                   ((64, 64), (8, 8), (3, 5))])
def test_calc_disparity_screened_squared_12bit(vwb, oracle, trace, shape):
    """SquaredCost on 12-bit imagery with the full range 4095.  At 21 x 21 the window sums exceed uint32 and the screened
    exact-integer kernel (k1_screen) runs: centred int32 numerators, fp32 screening, exact int64 evaluation of the
    surviving candidates.  The 7 x 7 and 3 x 5 shapes fit uint32 (Sq on K1 screen needs kx * ky >= 257) and test K1 fast."""
    from visionworkbench_b200.synth import make_rasters
    (W, H), search, kernel = shape
    left, right = make_rasters(W, H, search, kernel, seed=5 + W, bits=12)
    left[0, 0], left[0, 1] = 0.0, 4095.0                # the full 12-bit range, whatever the smoothing left
    left = left - 700.0; right = right - 700.0          # SquaredCost only needs a bounded range, not non-negative values
    got = trace.run(lambda: vwb.calc_disparity(1, left, right, search, kernel))
    assert vwb.last_k1_stats()["path"] == "exact-int"
    family = trace.assert_hot(1, left, right, search, kernel).family
    assert family == ("k1_screen_kernel" if kernel[0] * kernel[1] >= 257 else "k1_fast_abs_kernel")
    ref = oracle.calc_disparity(1, left, right, search, kernel)
    _assert_disp_equal(got, ref, f"screened sq {shape}")


@pytest.mark.parametrize("cost", [1, 2])
def test_screened_kernel_flat_regions_overflow_to_replay(vwb, oracle, cost):
    """A flat region makes every disparity tie: the candidate lists overflow and the pixels are replayed exactly."""
    rng = np.random.default_rng(79)
    W, H, search, kernel = 300, 40, (32, 16), (21, 21)
    right = np.floor(rng.random((H + 20 + 15, W + 20 + 31)) * 4096).astype(np.float32)
    right[:, 100:260] = 1000.0
    left = np.ascontiguousarray(right[3:3 + H + 20, 7:7 + W + 20])
    got = vwb.calc_disparity(cost, left, right, search, kernel)
    assert vwb.last_k1_stats()["path"] == "exact-int"
    ref = oracle.calc_disparity(cost, left, right, search, kernel)
    assert (ref[..., 2] == 0).any() and (ref[..., 2] == 1).any()
    _assert_disp_equal(got, ref, "flat")


@pytest.mark.parametrize("cost,kernel", [(2, (9, 9)), (1, (21, 21)), (2, (21, 21))])
def test_view_single_level_uses_screened_kernel(vwb, oracle, cost, kernel):
    """pyramid_correlate(max_pyramid_levels=0) with NCC / wide SquaredCost: the level-0 zone goes to k1_screen with the
    zone's origins (edge-extended reads), the R->L pass' negative offsets and the half-resolution seeding stage."""
    from visionworkbench_b200.synth import make_pair
    search = (-20, -7, 12, 9)
    left, right, lm, rm, _ = make_pair(420, 300, search, 63, dropout=0.0)
    view = vwb.pyramid_correlate(left, right, lm, rm, 0, 0.0, search, kernel, cost, 0, 0.0, 2.0, 0, 3, 0)
    p = oracle.make_params(search, kernel, cost=cost, consistency_threshold=2.0, filter_half_kernel=3, max_pyramid_levels=0)
    for bbox in [(0, 0, 420, 300), (100, 60, 400, 290)]:
        got = view.rasterize(None, bbox)
        ref = oracle.pyramid_correlate(p, left, right, lm, rm, bbox=bbox)
        _assert_disp_equal(got, ref, f"single level screened cost {cost} {bbox}")


@pytest.mark.parametrize("seed", range(8))
def test_screened_kernel_randomised_imagery(vwb, oracle, seed):
    """Adversarial inputs for the fp32 screening of k1_screen: narrow-band (low contrast) imagery with masses of near ties,
    dark / zero areas, full 12-bit range, shifted origins, odd sizes -- NCC and SquaredCost must stay bit-identical."""
    rng = np.random.default_rng(1000 + seed)
    W, H = int(rng.integers(64, 330)), int(rng.integers(64, 120))
    kx = int(rng.choice([3, 7, 15, 21])); ky = int(rng.choice([3, 7, 15, 21]))
    sx = int(rng.choice([8, 11, 16, 37])); sy = int(rng.integers(8, 13))
    style = seed % 4
    rw, rh = W + kx - 1 + sx - 1, H + ky - 1 + sy - 1
    if style == 0:      # narrow band near the top of the range
        right = 3900.0 + np.floor(rng.random((rh, rw)) * 40)
    elif style == 1:    # full range noise with a dark quarter and a zero block
        right = np.floor(rng.random((rh, rw)) * 4096)
        right[: rh // 2, : rw // 2] = np.floor(right[: rh // 2, : rw // 2] / 512)
        right[rh // 3: rh // 3 + 12, rw // 3: rw // 3 + 40] = 0
    elif style == 2:    # smooth ramp + 1 bit of noise: long plateaus of equal costs
        yy, xx = np.mgrid[0:rh, 0:rw]
        right = np.floor((xx * 7 + yy * 3) % 1024 + rng.integers(0, 2, (rh, rw)))
    else:               # 10-bit texture
        right = np.floor(rng.random((rh, rw)) * 1024)
    right = right.astype(np.float32)
    dx0, dy0 = int(rng.integers(0, sx)), int(rng.integers(0, sy))
    left = np.ascontiguousarray(right[dy0:dy0 + H + ky - 1, dx0:dx0 + W + kx - 1]).copy()
    left += np.floor(rng.random(left.shape) * 3).astype(np.float32) * (style != 2)
    left = np.clip(left, 0, 4095)
    for cost in (2, 1):
        got = vwb.calc_disparity(cost, left, right, (sx, sy), (kx, ky))
        assert vwb.last_k1_stats()["path"] == "exact-int"
        ref = oracle.calc_disparity(cost, left, right, (sx, sy), (kx, ky))
        _assert_disp_equal(got, ref, f"random screened seed {seed} cost {cost} {W}x{H} k{kx}x{ky} s{sx}x{sy} style {style}")


def _sgm_pair(seed, W, H, search, off, bits=8):
    rng = np.random.default_rng(seed)
    sx, sy = search
    base = np.floor(rng.random((H + sy + 40, W + sx + 40)) * (1 << bits))
    base = np.floor((base + np.roll(base, 1, 0) + np.roll(base, 1, 1) + np.roll(base, (1, 1), (0, 1))) / 4).astype(np.float32)
    left = base[20:20 + H, 20:20 + W]
    right = base[20 - off[1]:20 - off[1] + H + sy, 20 - off[0]:20 - off[0] + W + sx]
    return np.ascontiguousarray(left), np.ascontiguousarray(right)


@pytest.mark.parametrize("kernel,search,shape", [(3, (8, 8), (150, 120)), (5, (8, 8), (133, 77)), (7, (12, 4), (160, 90)), (9, (6, 10), (97, 141)),
                                                 (3, (0, 0), (40, 30)), (5, (31, 31), (70, 60))])
def test_sgm_core_matches_oracle(vwb, oracle, kernel, search, shape):
    """calc_disparity_sgm (census costs, 8-direction SGM, integer winner) is pure integer arithmetic: bit-identical to
    oracle/vw_sgm_oracle.c, which the reference's own KAT pins (tests/test_oracle_sgm.py)."""
    W, H = shape
    left, right = _sgm_pair(31 + kernel + W, W, H, search, (min(3, search[0]), min(2, search[1])))
    got = vwb.calc_disparity_sgm(left, right, search, kernel)
    ref = oracle.sgm_calc_disparity(left, right, search, kernel)
    assert got.shape == ref.shape
    assert np.array_equal(got, ref), f"{int((got != ref).any(-1).sum())} of {ref.shape[0] * ref.shape[1]} pixels differ"


def test_sgm_core_ties_and_float_ranges(vwb, oracle):
    """Textureless and few-level imagery (masses of tied accumulated costs -> select_best_disparity's smoothing iterations),
    and a float input range that u8_convert stretches (Image/ImageThresh.h:274-286)."""
    rng = np.random.default_rng(99)
    for left, right in [
        (np.full((40, 50), 100.0, np.float32), np.full((48, 58), 100.0, np.float32)),
        (np.floor(rng.random((60, 70)) * 3).astype(np.float32), np.floor(rng.random((68, 78)) * 3).astype(np.float32)),
        ((rng.random((64, 64)) * 1000.0 - 300.0).astype(np.float32), (rng.random((72, 72)) * 900.0 - 250.0).astype(np.float32)),
    ]:
        got = vwb.calc_disparity_sgm(left, right, (8, 8), 3)
        ref = oracle.sgm_calc_disparity(left, right, (8, 8), 3)
        assert np.array_equal(got, ref), f"{int((got != ref).any(-1).sum())} pixels differ"
    with pytest.raises(vwb.NoImplErr):
        vwb.calc_disparity_sgm(left, right, (8, 8), 11)


def test_sgm_core_device_tensors(vwb, oracle):
    import torch
    left, right = _sgm_pair(5, 120, 90, (8, 8), (2, 1))
    got = vwb.calc_disparity_sgm(torch.from_numpy(left).cuda(), torch.from_numpy(right).cuda(), (8, 8), 5)
    assert np.array_equal(got.cpu().numpy(), oracle.sgm_calc_disparity(left, right, (8, 8), 5))


@pytest.mark.parametrize("mode", [0, 2, 3, 4, 5])
def test_sgm_subpixel_modes(vwb, oracle, mode):
    """create_disparity_view_subpixel (SGM.cc:1497-1614): the integer part is bit-identical, the float offsets (double
    arithmetic with cos()) agree within 1e-5 -- the tolerance north_star states for floating point."""
    import scipy.ndimage as ndi
    rng = np.random.default_rng(17)
    base = ndi.gaussian_filter(np.floor(rng.random((130, 150)) * 256).astype(np.float32), 1.2)
    left = np.ascontiguousarray(base[10:100, 10:120])
    right = np.ascontiguousarray(ndi.shift(base, (1.4, 2.3), order=3)[10:108, 10:128]).astype(np.float32)
    gi, gf = vwb.calc_disparity_sgm_subpixel(left, right, (8, 8), 5, mode)
    ri, rf = oracle.sgm_calc_disparity_subpixel(left, right, (8, 8), 5, mode)
    assert np.array_equal(gi, ri)
    assert np.abs(gf - rf).max() <= 1e-5, float(np.abs(gf - rf).max())
    if mode:
        assert (gf[..., 0] != np.floor(gf[..., 0])).mean() > 0.5          # offsets were applied
    gi1, gf1 = vwb.calc_disparity_sgm_subpixel(left, right, (8, 8), 5, 1)          # SUBPIXEL_PARABOLA (2-D fit)
    ri1, rf1, _ = oracle.calc_disparity_sgm(left, right, (8, 8), 5, subpixel_mode=1, memory_limit_mb=1e9)
    assert np.array_equal(gi1, ri1) and np.abs(gf1 - rf1).max() <= 1e-5


@pytest.mark.parametrize("cost", [0, 1, 2])
def test_host_rasters_are_fed_in_bands(vwb, oracle, cost, monkeypatch):
    """the tile feeder of vwb200_calc_disparity (host buffers): H2D / correlate / D2H overlapped over output-row bands with
    three rotating band buffers; results identical to the one-shot path and to the oracle, whatever the band height"""
    from visionworkbench_b200.synth import make_rasters
    left, right = make_rasters(300, 333, (24, 17), (9, 7), seed=77 + cost)
    ref = oracle.calc_disparity(cost, left, right, (24, 17), (9, 7))
    for rows in ("32", "64", "100", "320"):          # 11, 6, 4 and 2 bands (the last one ragged)
        monkeypatch.setenv("VWB200_BAND_ROWS", rows)
        got = vwb.calc_disparity(cost, left, right, (24, 17), (9, 7))
        _assert_disp_equal(got, ref, f"bands of {rows} rows, cost {cost}")
    monkeypatch.delenv("VWB200_BAND_ROWS")
    monkeypatch.setenv("VWB200_NO_PIPELINE", "1")
    _assert_disp_equal(vwb.calc_disparity(cost, left, right, (24, 17), (9, 7)), ref, "one shot")
    # a strided (pitched) host view goes through the same feeder
    big_l = np.zeros((left.shape[0], left.shape[1] + 13), np.float32); big_l[:, :left.shape[1]] = left
    monkeypatch.delenv("VWB200_NO_PIPELINE")
    monkeypatch.setenv("VWB200_BAND_ROWS", "64")
    import ctypes as C
    out = np.empty((333, 300, 3), np.int32)
    rc = vwb.lib().vwb200_calc_disparity(cost, big_l.ctypes.data, left.shape[1], left.shape[0], big_l.shape[1], right.ctypes.data, right.shape[1],
                                         right.shape[0], right.shape[1], 24, 17, 9, 7, out.ctypes.data, 300, 0, None)
    assert rc == 0
    _assert_disp_equal(out, ref, "pitched input")


def test_view_streamed_inputs_tile_feeder(vwb, oracle):
    """VWB200_INPUTS_STREAMED: the rasters stay on the host and every rasterize() uploads its tile's region of interest
    (edge tiles clamp / zero-extend exactly like resident rasters)"""
    search, kernel = (-12, -8, 12, 8), (7, 7)
    left, right, lm, rm, _ = make_pair_for_tests(300, 260, search, seed=21)
    args = (vwb.PREFILTER_NONE, 0.0, search, kernel, vwb.SQUARED_DIFFERENCE, 0, 0.0, 2.0, 0, 3, 3)
    streamed = vwb.PyramidCorrelationView(left, right, lm, rm, *args, streamed=True)
    p = oracle.make_params(search, kernel, cost=1, consistency_threshold=2.0, filter_half_kernel=3, max_pyramid_levels=3)
    for bbox in [(0, 0, 128, 128), (172, 132, 300, 260), (100, 60, 220, 200), (0, 200, 90, 260), (0, 0, 300, 260)]:
        got = streamed.rasterize(None, bbox)
        ref = oracle.pyramid_correlate(p, left, right, lm, rm, bbox=bbox)
        assert np.array_equal(got, ref), (bbox, int((got != ref).any(-1).sum()))


def make_pair_for_tests(W, H, search, seed):
    from visionworkbench_b200.synth import make_pair
    return make_pair(W, H, search, seed=seed)
