"""The exact-integer kernels across the input value range.  Which kernel may take a raster is decided from the value range
image_stats_kernel (csrc/k1_fast.cu) reports -- vmin, vmax and whether every pixel is an integer -- against the limits of
k1_fast_supported, screen_params (k1_screen.cu) and k1_zone_int_mode (k1_zone_int.cu); the same vmin drives the u16 / int16
packing of every exact kernel and SGM's u8_convert stretch.  Every case here is compared bit for bit with the oracle:
  A  signed imagery holding -0.0 (a warp whose minimum is -0.0 must not hide the negative pixels of the others),
  B  both sides of every range limit of DESIGN §3/§4, with the path the predicates must choose,
  C  a non-finite pixel (not integer: the general kernel, no parity claim -- DESIGN §3)."""
import numpy as np
import pytest

from kernel_trace import trace  # noqa: F401  (the profiler fixture: the kernels a call ran)

pytestmark = pytest.mark.gpu

EXACT, FP64 = "exact-int", "general-fp64"
# image_stats_kernel runs 2 x 132 CTAs x 256 threads: below this many pixels each thread reads at most one pixel and a warp
# reads 32 consecutive ones, so a warp in the top rows of an A-family raster sees only -0.0 and non-negative values
STATS_THREADS = 2 * 132 * 256


@pytest.fixture(scope="module")
def vwb():
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "GPU tests need a CUDA device: the engine has no CPU path"
    return v


def make_raster(h, w, lo, hi, texture="uniform", seed=0, halves=False):
    """float32 (h, w) integer raster over [lo, hi] holding both ends.  texture "uniform": integers in [lo, hi]; "binary": only
    lo and hi, with a checkerboard in the top-left quarter so that some windows differ in every pixel (the largest window
    sum).  halves: the bottom half moves down by hi - lo + 1 (signed imagery)."""
    rng = np.random.default_rng(seed)
    if texture == "binary":
        v = np.where(rng.random((h, w)) < 0.5, lo, hi).astype(np.float64)
        yy, xx = np.mgrid[0:h // 2, 0:w // 2]
        v[:h // 2, :w // 2] = np.where((yy + xx) % 2 == 0, lo, hi)
    else:
        v = rng.integers(lo, hi, size=(h, w), endpoint=True).astype(np.float64)
    v[0, 0], v[0, 1] = lo, hi
    if halves:
        v[h // 2:] -= hi - lo + 1
        v[-1, 0], v[-1, 1] = lo - (hi - lo + 1), hi - (hi - lo + 1)
    return v.astype(np.float32)


def negative_zero(v):
    """in the top half of v, every zero and every 8th pixel becomes -0.0 (in place)"""
    top = v[:v.shape[0] // 2]
    top[top == 0] = -0.0
    top.reshape(-1)[::8] = -0.0
    return v


def add_noise(v, noise, seed, lo, hi):
    """v + integers in [-noise, noise], clipped to [lo, hi].  Row 0 is kept: noise may flip the sign of a pixel near zero,
    and the warps that read row 0 must still see no negative value"""
    n = np.clip(v + np.random.default_rng(seed).integers(-noise, noise, size=v.shape, endpoint=True), lo, hi)
    n[0] = v[0]
    return n.astype(np.float32)


def make_pair(W, H, search, kernel, lo, hi, texture="uniform", shift=(3, 2), seed=0, halves=False, noise=0, negzero=False):
    """calc_disparity inputs for a W x H output: `right` from make_raster, `left` its crop at the integer disparity `shift`
    plus add_noise(noise).  negzero: negative_zero() on both."""
    (sx, sy), (kx, ky), (dx, dy) = search, kernel, shift
    assert 0 <= dx < sx and 0 <= dy < sy
    right = make_raster(H + ky - 1 + sy - 1, W + kx - 1 + sx - 1, lo, hi, texture, seed, halves)
    assert right.size < STATS_THREADS
    left = right[dy:dy + H + ky - 1, dx:dx + W + kx - 1]
    if noise:
        left = add_noise(left, noise, seed + 1, right.min(), right.max())
    left = np.ascontiguousarray(left)
    if negzero:
        negative_zero(left), negative_zero(right)
    return left, right


def _assert_same(got, ref, what=""):
    assert got.shape == ref.shape, what
    bad = ~np.all(got == ref, axis=-1)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} pixels differ, first at {np.argwhere(bad)[0]}"


def _check(vwb, oracle, cost, left, right, search, kernel, path=None, what="", trace=None, zone_int=False):
    """parity with the oracle; with `trace`, also that the kernel the restated dispatch (tests/bm_reference.py) picks ran"""
    ref = oracle.calc_disparity(cost, left, right, search, kernel)
    run = lambda: vwb.calc_disparity(cost, left, right, search, kernel)
    got = trace.run(run) if trace else run()
    _assert_same(got, ref, what)
    if path is not None:
        assert vwb.last_k1_stats()["path"] == path, what
    if trace:
        return trace.assert_hot(cost, left, right, search, kernel, zone_int)


# ---- A: signed imagery with -0.0 ----------------------------------------------------------------------------------------
# top half of each raster >= 0 with -0.0 (the warps that reach -0.0 first), bottom half negative.  "wide": [0, 2047] over
# [-2048, -1], the left an exact crop of the right -- the true disparity costs 0, so a wrongly packed (larger) cost elsewhere
# rarely changes a winner; "low": [0, 3] over [-4, -1] with +-2 noise in the left, which flips the sign of pixels near
# zero, so that the pairs a wrong vmin packs wrongly decide winners.
A1 = {"wide": dict(lo=0, hi=2047, halves=True, negzero=True), "low": dict(lo=0, hi=3, halves=True, noise=2, negzero=True)}


@pytest.mark.parametrize("variant", list(A1))
@pytest.mark.parametrize("cost,path", [(0, EXACT), (1, EXACT), (2, FP64)])
def test_a1_signed_zero_calc_disparity(vwb, oracle, cost, path, variant):
    left, right = make_pair(100, 72, (16, 10), (15, 15), seed=11, **A1[variant])
    assert np.signbit(right[:8]).any() and (right < 0).any()
    _check(vwb, oracle, cost, left, right, (16, 10), (15, 15), path)


def test_a2_negative_imagery_with_negative_zero(vwb, oracle):
    """[-8192, -1] plus -0.0: the range is 8192, one past the Abs limit of K1 fast"""
    left, right = make_pair(100, 72, (16, 10), (15, 15), -8192, -1, seed=12, negzero=True)
    _check(vwb, oracle, 0, left, right, (16, 10), (15, 15), FP64)


@pytest.mark.parametrize("variant", list(A1))
@pytest.mark.parametrize("cost", [0, 1])
def test_a3_signed_zero_zone_int(vwb, oracle, monkeypatch, cost, variant):
    """A1 through the integer zone kernel (narrow for Abs, WIDE for Sq on "wide")"""
    left, right = make_pair(61, 45, (11, 9), (15, 15), seed=13, **A1[variant])
    monkeypatch.setenv("VWB200_K1_ZONE_INT", "1")
    _check(vwb, oracle, cost, left, right, (11, 9), (15, 15))


@pytest.mark.parametrize("variant", list(A1))
@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("levels", [0, 2])
@pytest.mark.parametrize("cost", [0, 1])
def test_a4_signed_zero_view(vwb, oracle, cost, levels, dropout, variant):
    """A1 imagery through PyramidCorrelationView: the level-0 tile statistics pick K1 fast (one level-0 zone of 320
    disparities) or the integer zone kernel (pyramid, or masked pixels that the mean fill makes non-integer)"""
    W, H, m, shift = 200, 160, 12, (5, -3)
    kw = A1[variant]
    base = make_raster(H + 2 * m, W + 2 * m, kw["lo"], kw["hi"], seed=14 + levels, halves=True)
    left = np.ascontiguousarray(base[m:m + H, m:m + W])
    right = base[m - shift[1]:m - shift[1] + H, m - shift[0]:m - shift[0] + W]
    if kw.get("noise"):
        right = add_noise(right, kw["noise"], levels, base.min(), base.max())
    right = np.ascontiguousarray(right)
    negative_zero(left), negative_zero(right)
    lm, rm = np.full((H, W), 255, np.uint8), np.full((H, W), 255, np.uint8)
    if dropout:
        lm[30:60, 40:90] = 0
        rm[100:130, 20:70] = 0
    search, kernel = (-10, -8, 10, 8), (7, 7)
    view = vwb.pyramid_correlate(left, right, lm, rm, vwb.PREFILTER_NONE, 0.0, search, kernel, cost, 0, 0.0, 2.0, 0, 3, levels)
    got = view.rasterize()
    p = oracle.make_params(search, kernel, cost=cost, consistency_threshold=2.0, filter_half_kernel=3, max_pyramid_levels=levels)
    ref = oracle.pyramid_correlate(p, left, right, lm, rm)
    _assert_same(got, ref, f"view cost={cost} levels={levels} dropout={dropout} {variant}")
    assert (ref[..., 2] == 1).mean() > 0.1


def test_a5_signed_zero_sgm(vwb, oracle):
    """u8_convert stretches [vmin, vmax] to [0, 255] before the census: a wrong vmin clamps every negative pixel to one
    value.  The two halves move by different disparities, so a flat (clamped) half cannot inherit the right answer from
    the SGM paths that enter it from the other half."""
    right = make_raster(98, 128, 0, 127, seed=15, halves=True)
    left = np.ascontiguousarray(right[3:93, 5:125])
    left[45:] = right[51:96, 1:121]
    negative_zero(left), negative_zero(right)
    got = vwb.calc_disparity_sgm(left, right, (8, 8), 5)
    ref = oracle.sgm_calc_disparity(left, right, (8, 8), 5)
    assert got.shape == ref.shape
    assert np.array_equal(got, ref), f"{int((got != ref).any(-1).sum())} of {ref.shape[0] * ref.shape[1]} pixels differ"


@pytest.mark.parametrize("variant", list(A1))
@pytest.mark.parametrize("feed", ["bands", "torch"])
@pytest.mark.parametrize("cost,path", [(0, EXACT), (1, EXACT), (2, FP64)])
def test_a6_signed_zero_feeders(vwb, oracle, monkeypatch, cost, path, feed, variant):
    """host band feeder (one set of statistics per 32-row band; one band straddles the sign change) and device tensors"""
    left, right = make_pair(100, 100, (12, 9), (15, 15), seed=16, **A1[variant])
    if feed == "bands":
        monkeypatch.setenv("VWB200_BAND_ROWS", "32")
        _check(vwb, oracle, cost, left, right, (12, 9), (15, 15), path)
    else:
        import torch
        ref = oracle.calc_disparity(cost, left, right, (12, 9), (15, 15))
        got = vwb.calc_disparity(cost, torch.from_numpy(left).cuda(), torch.from_numpy(right).cuda(), (12, 9), (15, 15))
        _assert_same(got.cpu().numpy(), ref)
        assert vwb.last_k1_stats()["path"] == path


# ---- B: both sides of every limit -----------------------------------------------------------------------------------------
LIMITS = [  # id, cost, (W, H), search, kernel, lo, hi, texture, path
    # Abs on K1 fast: range <= 8191 ((v - vmin) * 8 packs into u16)
    ("abs-8191-k31x41", 0, (64, 40), (16, 8), (31, 41), 0, 8191, "binary", EXACT),
    ("abs-8192-k31x41", 0, (64, 40), (16, 8), (31, 41), 0, 8192, "binary", FP64),
    ("abs-8191-k21", 0, (80, 60), (16, 8), (21, 21), -4096, 4095, "binary", EXACT),
    ("abs-8192-k21", 0, (80, 60), (16, 8), (21, 21), -4096, 4096, "binary", FP64),
    # Sq: 4095^2 * 15 * 17 < 2^32 - 1 keeps K1 fast (window sums above 2^31); 15 x 19 goes to K1 screen; range 4096 to fp64
    ("sq-4095-k15x17", 1, (80, 48), (16, 8), (15, 17), 0, 4095, "binary", EXACT),
    ("sq-4095-k15x19", 1, (80, 48), (16, 8), (15, 19), 0, 4095, "binary", EXACT),      # K1 screen (asserted below)
    ("sq-4096-k15x17", 1, (80, 48), (16, 8), (15, 17), 0, 4096, "binary", FP64),
    # NCC on K1 screen: pixels in [0, 4095]
    ("ncc-vmax-4095", 2, (80, 48), (16, 8), (9, 9), 0, 4095, "uniform", EXACT),
    ("ncc-vmax-4096", 2, (80, 48), (16, 8), (9, 9), 0, 4096, "uniform", FP64),
    ("ncc-vmin-minus1", 2, (80, 48), (16, 8), (9, 9), -1, 4095, "uniform", FP64),
    # magnitude: |v| < 1e6
    ("abs-max-999999", 0, (80, 48), (16, 8), (9, 9), 995904, 999999, "uniform", EXACT),
    ("abs-max-1e6", 0, (80, 48), (16, 8), (9, 9), 995905, 1000000, "uniform", FP64),
    ("abs-min-minus999999", 0, (80, 48), (16, 8), (9, 9), -999999, -995904, "uniform", EXACT),
    ("abs-min-minus1e6", 0, (80, 48), (16, 8), (9, 9), -1000000, -995905, "uniform", FP64),
    ("sq-max-999999", 1, (80, 48), (16, 8), (9, 9), 995904, 999999, "uniform", EXACT),
    ("sq-max-1e6", 1, (80, 48), (16, 8), (9, 9), 995905, 1000000, "uniform", FP64),
    ("sq-min-minus999999", 1, (80, 48), (16, 8), (9, 9), -999999, -995904, "uniform", EXACT),
    ("sq-min-minus1e6", 1, (80, 48), (16, 8), (9, 9), -1000000, -995905, "uniform", FP64),
]


@pytest.mark.parametrize("case", LIMITS, ids=[c[0] for c in LIMITS])
def test_b_range_limits(vwb, oracle, trace, case):
    what, cost, (W, H), search, kernel, lo, hi, texture, path = case
    left, right = make_pair(W, H, search, kernel, lo, hi, texture, seed=len(what) + W)
    exp = _check(vwb, oracle, cost, left, right, search, kernel, path, what, trace)
    if what == "sq-4095-k15x19":                         # the kernel the comment above names
        assert exp.family == "k1_screen_kernel"


ZONE_LIMITS = [  # id, cost, K, lo, hi, texture
    ("abs-k17-58052-narrow", 0, 17, 0, 58052, "binary"),          # 58052 * 289 < 2^24: keys cost << 8 just below 2^32
    ("abs-k17-58053-fp64", 0, 17, 0, 58053, "binary"),            # one past: the fp64 zone kernel
    ("sq-k15-4095-wide", 1, 15, 0, 4095, "binary"),               # window sums up to 4095^2 * 225 ~ 3.8e9
    ("abs-k15-offset-3e7", 0, 15, 30000000, 30004094, "uniform"),  # no magnitude guard; above 2^24 only even integers
    ("sq-k15-offset-3e7", 1, 15, 30000000, 30004094, "uniform"),
]


@pytest.mark.parametrize("case", ZONE_LIMITS, ids=[c[0] for c in ZONE_LIMITS])
def test_b5_zone_int_limits(vwb, oracle, monkeypatch, trace, case):
    what, cost, k, lo, hi, texture = case
    left, right = make_pair(61, 45, (11, 9), (k, k), lo, hi, texture, seed=k + cost)
    monkeypatch.setenv("VWB200_K1_ZONE_INT", "1")
    n0 = vwb.kernel_launches()
    exp = _check(vwb, oracle, cost, left, right, (11, 9), (k, k), None, what, trace, zone_int=True)
    assert vwb.kernel_launches() > n0
    variant = what.rsplit("-", 1)[1]                       # the variant the id names
    if variant in ("narrow", "wide"):
        assert exp.family == "k1_zone_int_kernel" and exp.args[2] == (variant == "wide"), what
    elif variant == "fp64":
        assert exp.family == "k1_generic_kernel", what


@pytest.mark.parametrize("cost", [0, 1, 2])
def test_b6_one_fractional_pixel(vwb, oracle, cost):
    left, right = make_pair(80, 48, (16, 8), (9, 9), 0, 4095, seed=17)
    left[20, 30] += 0.5
    _check(vwb, oracle, cost, left, right, (16, 8), (9, 9), FP64)


# ---- C: non-finite ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("zone_int", [False, True])
@pytest.mark.parametrize("cost", [0, 1, 2])
def test_c_infinite_pixel_takes_general_kernel(vwb, monkeypatch, cost, zone_int):
    """+inf is not an integer: the general kernel runs and the call succeeds.  No parity claim: the reference's sliding
    double sums make results around inf depend on the zone origin (DESIGN §3)."""
    left, right = make_pair(80, 48, (16, 8), (9, 9), 0, 4095, seed=18)
    right[30, 40] = np.inf
    if zone_int:
        monkeypatch.setenv("VWB200_K1_ZONE_INT", "1")
    got = vwb.calc_disparity(cost, left, right, (16, 8), (9, 9))
    assert got.shape == (48, 80, 3)
    assert vwb.last_k1_stats()["path"] == FP64
