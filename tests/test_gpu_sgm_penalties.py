"""SemiGlobalMatcher on the device across its penalty range: explicit P1 / P2 up to 30000, accumulated costs that wrap
in uint16, the p1 <= p2 <= 30000 limit on both sides, and config 4 at full size.  Compared with the oracle: integer
disparities bit for bit, sub-pixel disparities within 1e-5.

The wrap cases reuse the imagery of test_oracle_sgm_penalties.py (a flat texture, so p2_mod stays near P2, and search
boxes that jump between neighbours, so new entries start from 255 + P2).  Each asserts on its own inputs, through the
restatement in sgm_reference.py, that the 8-path sums pass 65535 and that the wrap changes winners."""
import functools
import re

import numpy as np
import pytest

import sgm_reference as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def vwb():
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "GPU tests need a CUDA device: the engine has no CPU path"
    return v


GRID = [(0, 0), (1, 1), (1, 30000), (30000, 30000), (29999, 30000), (200, 8000), (0, 30000), (700, 0)]
WRAPS = [(1, 30000), (30000, 30000), (29999, 30000), (0, 30000)]
OH, OW, MOVING = 64, 80, (15, 11)
LANES, SERIAL = "VWB200_SGM_LANES_PER_ENTRY", "VWB200_SGM_SERIAL"
# name: (search, boxes, environment).  boxes: None = the constant box; (w, h) = moving boxes of 1..w x 1..h;
# (w, h, "full") = the same plus full-search (192-entry) pixels, a block of them and 3 % scattered among the small boxes.
# sgm_paths_launch takes the rows-in-lanes kernel when every box is at most 6 wide and 8 high, else the lane-per-disparity
# kernel, whose pixels of more than 32 entries take the general step.  The 8 paths go into four partial volumes, two each
# (<= 2 x 30255: no wrap inside a path kernel); sgm_wta_kernel sums them, staged in shared memory when every box has <= 32
# entries, after sgm_sum4_kernel otherwise.  VWB200_SGM_SERIAL adds all 8 paths into one volume, as MGM always does, so
# that the wrap happens in the path kernels' own adds.
REGIMES = {
    "const-rows": ((5, 3), None, {}),                             # 6 x 4 everywhere
    "const-lines": ((10, 1), None, {}),                           # 11 x 2 = 22 entries, wider than 6
    "const-general": ((8, 5), None, {}),                          # 54 entries
    "moving-rows": (MOVING, (6, 5), {}),                          # <= 30 entries: staged sums (config 4's path)
    "moving-rows-tall": (MOVING, (6, 8), {}),                     # up to 48 entries: sgm_sum4_kernel
    "moving-lanes": (MOVING, (6, 5), {LANES: "1"}),
    "moving-general": (MOVING, (6, 8, "full"), {}),
    "moving-rows-serial": (MOVING, (6, 8), {SERIAL: "1"}),
    "moving-general-serial": (MOVING, (6, 8, "full"), {SERIAL: "1"}),
}


@functools.lru_cache(maxsize=None)
def _inputs(regime, levels=4):
    search, boxes, _ = REGIMES[regime]
    left, right = R.flat_pair(31, OH, OW, search, 5, levels=levels)
    if boxes is None:
        b = np.tile(np.array([0, 0, search[0], search[1]], np.int32), (OH, OW, 1))
    else:
        b = R.moving_boxes(32, OH, OW, search, boxes[0], boxes[1])
        if len(boxes) > 2:
            full = np.random.default_rng(33).random((OH, OW)) < 0.03
            full[20:30, 30:50] = True
            b[full] = (0, 0, search[0], search[1])
    return left, right, b, search


@functools.lru_cache(maxsize=None)
def _assert_wraps(regime, p1, p2):
    left, right, b, search = _inputs(regime)
    R.assert_wrap_decides(R.sgm(left, right, search, 5, b, p1, p2))


def _run_ex(vwb, monkeypatch, regime, cost_type, **kw):
    left, right, b, search = _inputs(regime, **({"levels": 12} if cost_type == vwb.TERNARY_CENSUS_TRANSFORM else {}))
    for k, v in REGIMES[regime][2].items():
        monkeypatch.setenv(k, v)
    bounds = None if REGIMES[regime][1] is None else b      # constant boxes: the entry point derives them
    return vwb.calc_disparity_sgm_ex(cost_type, left, right, search, 5, bounds=bounds, **kw)


def _same(gi, gf, ri, rf, what):
    assert np.array_equal(gi, ri), f"{what}: {int((gi != ri).any(-1).sum())} of {ri.shape[0] * ri.shape[1]} pixels differ"
    if rf is not None:
        assert np.abs(gf - rf).max() <= 1e-5, f"{what}: sub-pixel differs by {float(np.abs(gf - rf).max())}"


# ---- a. the penalty grid on every path kernel --------------------------------------------------------------------------------
@pytest.mark.parametrize("mgm", [False, True], ids=["sgm", "mgm"])
@pytest.mark.parametrize("p1,p2", GRID)
@pytest.mark.parametrize("regime", list(REGIMES))
def test_a_penalty_grid(vwb, oracle, monkeypatch, regime, p1, p2, mgm):
    left, right, b, search = _inputs(regime)
    if (p1, p2) in WRAPS and REGIMES[regime][1] is not None:
        _assert_wraps(regime, p1, p2)          # on the SGM restatement; MGM's four sweeps pass 65535 on the same inputs too
    ri, rf = oracle.sgm_calc_disparity_bounds(left, right, search, 5, b, subpixel_mode=5, p1=p1, p2=p2, use_mgm=mgm)
    gi, gf = _run_ex(vwb, monkeypatch, regime, vwb.CENSUS_TRANSFORM, use_mgm=mgm, subpixel_mode=5, p1=p1, p2=p2)
    _same(gi, gf, ri, rf, regime)
    if REGIMES[regime][1] is None and not mgm:
        _same(vwb.calc_disparity_sgm(left, right, search, 5, p1, p2), None, ri, None, "calc_disparity_sgm")


@pytest.mark.parametrize("mgm", [False, True], ids=["sgm", "mgm"])
@pytest.mark.parametrize("p1,p2", [(0, 30000), (30000, 30000)])
@pytest.mark.parametrize("regime", list(REGIMES))
def test_a_ternary_penalties(vwb, oracle, monkeypatch, regime, p1, p2, mgm):
    """TERNARY_CENSUS_TRANSFORM (threshold 5) on a 12-level texture, so that the signatures are not all "inside the band"."""
    left, right, b, search = _inputs(regime, levels=12)
    bounds = None if REGIMES[regime][1] is None else b
    ri, rf, _ = oracle.calc_disparity_sgm(left, right, search, 5, cost_type=4, use_mgm=mgm, subpixel_mode=5, bounds=bounds, p1=p1, p2=p2)
    assert ri[..., 2].mean() > 0.9
    gi, gf = _run_ex(vwb, monkeypatch, regime, vwb.TERNARY_CENSUS_TRANSFORM, use_mgm=mgm, subpixel_mode=5, p1=p1, p2=p2)
    _same(gi, gf, ri, rf, regime)


@pytest.mark.parametrize("mode", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("p1,p2", WRAPS)
def test_a_subpixel_modes_on_wrapped_costs(vwb, oracle, monkeypatch, p1, p2, mode):
    """every sub-pixel model reads the wrapped accumulated costs (and select_best_disparity's smoothed ones): moving boxes
    through calc_disparity_sgm_ex, the constant box through calc_disparity_sgm_subpixel"""
    _assert_wraps("moving-rows", p1, p2)
    left, right, b, search = _inputs("moving-rows")
    ri, rf, _ = oracle.calc_disparity_sgm(left, right, search, 5, subpixel_mode=mode, bounds=b, p1=p1, p2=p2)
    gi, gf = _run_ex(vwb, monkeypatch, "moving-rows", vwb.CENSUS_TRANSFORM, subpixel_mode=mode, p1=p1, p2=p2)
    _same(gi, gf, ri, rf, f"moving boxes, mode {mode}")
    left, right, _, search = _inputs("const-rows")
    ri, rf, _ = oracle.calc_disparity_sgm(left, right, search, 5, subpixel_mode=mode, p1=p1, p2=p2)
    gi, gf = vwb.calc_disparity_sgm_subpixel(left, right, search, 5, mode, p1, p2)
    _same(gi, gf, ri, rf, f"constant box, mode {mode}")


# ---- b. the penalty limit, on both sides -------------------------------------------------------------------------------------
ENTRIES = ["calc_disparity_sgm", "calc_disparity_sgm_subpixel", "calc_disparity_sgm_ex"]


def _entry(vwb, entry, left, right, search, kernel, p1, p2):
    if entry == "calc_disparity_sgm":
        return vwb.calc_disparity_sgm(left, right, search, kernel, p1, p2), None
    if entry == "calc_disparity_sgm_subpixel":
        return vwb.calc_disparity_sgm_subpixel(left, right, search, kernel, 5, p1, p2)
    return vwb.calc_disparity_sgm_ex(vwb.CENSUS_TRANSFORM, left, right, search, kernel, subpixel_mode=5, p1=p1, p2=p2)


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("kernel,p1,p2", [(5, 30000, 30000), (5, 0, 30000), (5, 750, 750), (7, 0, 30), (3, 0, 3)])
def test_b_limit_accepted(vwb, oracle, entry, kernel, p1, p2):
    """the largest P2, and P1 = P2 -- given, or reached through the default P1 (30 for census 7, 3 for census 3)"""
    left, right = R.flat_pair(40 + kernel, 40, 56, (9, 6), kernel)
    ri, rf = oracle.sgm_calc_disparity_subpixel(left, right, (9, 6), kernel, 5, p1, p2)
    gi, gf = _entry(vwb, entry, left, right, (9, 6), kernel, p1, p2)
    _same(gi, gf, ri, None if gf is None else rf, entry)


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("kernel,p1,p2,named", [(5, 0, 30001, "p1 = 15, p2 = 30001"), (5, 751, 750, "p1 = 751, p2 = 750"),
                                                (5, 30001, 30000, "p1 = 30001, p2 = 30000"),
                                                (7, 0, 29, "p1 = 30, p2 = 29"), (3, 0, 2, "p1 = 3, p2 = 2")])
def test_b_limit_rejected(vwb, entry, kernel, p1, p2, named):
    """outside p1 <= p2 <= 30000 (after the defaults) every entry point raises NoImplErr and names the penalties it got --
    including an explicit P2 below the default P1, which the reference would run"""
    left, right = R.flat_pair(50 + kernel, 40, 56, (9, 6), kernel)
    with pytest.raises(vwb.NoImplErr, match=re.escape(named)):
        _entry(vwb, entry, left, right, (9, 6), kernel, p1, p2)


# ---- c. config 4 at full size, and long lines --------------------------------------------------------------------------------
def test_c_config4_full_size(vwb, oracle):
    """config 4 of the benchmark on the whole raster: 4096^2, search 128, census 5, the half-resolution prior with search
    buffer (2, 2), LC_BLEND.  Only long lines reach the rows kernel's later meta epochs, the wrapped diagonals' restarts
    every out_w steps and offsets deep into the 0.42 G-entry ragged volume."""
    from visionworkbench_b200.synth import make_sgm_case
    left, right, prev, _ = make_sgm_case(4096, 128, 5, seed=104)
    gi, gf, gb = vwb.calc_disparity_sgm_ex(vwb.CENSUS_TRANSFORM, left, right, (128, 128), 5, subpixel_mode=vwb.SUBPIXEL_LC_BLEND,
                                           search_buffer=(2, 2), prev_disparity=prev, memory_limit_mb=1e9, return_bounds=True)
    assert gb.shape[:2] == (4092, 4092) and int(np.prod(gb[..., 2:] - gb[..., :2] + 1, -1).sum()) > 3.5e8
    ri, rf, rb = oracle.calc_disparity_sgm(left, right, (128, 128), 5, subpixel_mode=5, search_buffer=(2, 2), prev=prev, memory_limit_mb=1e9)
    assert np.array_equal(gb, rb), "boxes differ"
    _same(gi, gf, ri, rf, "config 4")


@pytest.mark.parametrize("oh,ow", [(48, 4096), (4096, 48)])
def test_c_long_lines_at_the_largest_penalties(vwb, oracle, oh, ow):
    """(30000, 30000) with moving boxes of <= 6 x 8 (the rows kernel) on lines of 4096 pixels"""
    search = (15, 11)
    left, right = R.flat_pair(60 + oh, oh, ow, search, 5)
    b = R.moving_boxes(61 + oh, oh, ow, search, 6, 8)
    ri, rf = oracle.sgm_calc_disparity_bounds(left, right, search, 5, b, subpixel_mode=5, p1=30000, p2=30000)
    gi, gf = vwb.calc_disparity_sgm_ex(vwb.CENSUS_TRANSFORM, left, right, search, 5, subpixel_mode=5, bounds=b, p1=30000, p2=30000)
    _same(gi, gf, ri, rf, f"{oh} x {ow}")
