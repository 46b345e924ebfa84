"""The device's sub-pixel floats against the restatements of the reference: SGM's five models through
calc_disparity_sgm_ex (tests/sgm_reference.py) and ParabolaSubpixelView with PREFILTER_NONE (tests/subpixel_reference.py),
on the inputs that test_oracle_subpixel.py checks the oracle with.

Integer disparities and validity are compared bit for bit.  So are the floats wherever no transcendental function is
involved: modes 2 (linear) and 3 (poly4), the two-value and both-bounds branches of every mode, the rejected 2-D fits and
every ParabolaSubpixelView result.  Where CUDA's cos (modes 4, 5) or erf (mode 1) are involved, the floats may differ by
1 float32 ulp from the restatement, which uses the host's libm: the test prints how many pixels are not bit-identical and
fails above 0.1 % of them."""
import re
import time

import numpy as np
import pytest

import sgm_reference as R
import subpixel_reference as S
from test_oracle_subpixel import PATCH_DISPARITIES, PENALTIES, SCENES, TARGETS, assert_bits, empty_bbox_case, restated, scene

pytestmark = pytest.mark.gpu
SERIAL = "VWB200_SGM_SERIAL"


@pytest.fixture(scope="module")
def vwb():
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "GPU tests need a CUDA device: the engine has no CPU path"
    return v


def ulps(a, b):
    """float32 ulp distance of same-shaped arrays (monotone integer keys of the bit patterns)"""
    ka, kb = (np.asarray(x, np.float32).view(np.int32).astype(np.int64) for x in (a, b))
    ka = np.where(ka < 0, -(ka & 0x7FFFFFFF), ka)
    kb = np.where(kb < 0, -(kb & 0x7FFFFFFF), kb)
    return np.abs(ka - kb)


def assert_float_contract(got, want, exact, what):
    """bit for bit where `exact`, within 1 ulp elsewhere, with at most 0.1 % of the pixels not bit-identical"""
    d = ulps(got[..., :2], want[..., :2]).max(-1)
    assert np.array_equal(got[..., 2], want[..., 2]), f"{what}: validity differs"
    assert not (d[exact] > 0).any(), f"{what}: {int((d[exact] > 0).sum())} exact pixels differ"
    off = int((d > 0).sum())
    print(f"{what}: {off} of {d.size} pixels not bit-identical, largest difference {int(d.max())} ulp")
    assert d.max() <= 1, f"{what}: {int(d.max())} ulps"
    assert off <= 0.001 * d.size, f"{what}: {off} pixels differ by 1 ulp"


def exact_pixels(res, want, mode):
    """pixels whose float no transcendental function touched in `mode`: all of them in modes 2 and 3; in modes 4 and 5
    those with the winner on a bound (or equal neighbours) along both axes; in mode 1 those whose fit was rejected"""
    if mode in (0, 2, 3):
        return np.ones(res.disparity.shape[:2], bool)
    if mode == 1:
        return (want[..., :2] == res.disparity[..., :2].astype(np.float32)).all(-1)
    dx, dy, b = res.disparity[..., 0], res.disparity[..., 1], res.bounds
    inner = ((dx > b[..., 0]) & (dx < b[..., 2])) | ((dy > b[..., 1]) & (dy < b[..., 3]))
    return ~inner | (res.disparity[..., 2] == 0)


_NAME = re.compile(r"\b((?:sgm|mgm)_\w+?)(?:<[^(]*>)?\(")


def sgm_kernels(fn):
    """(result, set of the sgm_ / mgm_ kernel names fn() launched), under torch.profiler.  A session loses the kernels
    launched right after it starts, so it opens with a warm-up step; one that still misses sgm_wta_kernel is repeated."""
    import torch
    from torch.profiler import ProfilerActivity, profile, schedule
    torch.cuda.init()
    for attempt in range(5):
        if attempt:
            time.sleep(0.5)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA], schedule=schedule(wait=0, warmup=1, active=1, repeat=1)) as prof:
            torch.ones(1, device="cuda").add_(1)
            torch.cuda.synchronize()
            prof.step()
            out = fn()
            torch.cuda.synchronize()
            prof.step()
        names = {m.group(1) for e in prof.events() if "vwb200" in e.name for m in [_NAME.search(e.name)] if m}
        if "sgm_wta_kernel" in names:
            return out, names
    pytest.fail(f"the profiler recorded no sgm_wta_kernel: {sorted(names)}")


def run_case(vwb, monkeypatch, case, mode, p1, p2, mgm=False):
    (left, right, b, search), _, _ = restated(case, 0, 0)
    if R.SUBPIXEL_CASES[case][4] == "serial":
        monkeypatch.setenv(SERIAL, "1")
    else:
        monkeypatch.delenv(SERIAL, raising=False)
    return vwb.calc_disparity_sgm_ex(vwb.CENSUS_TRANSFORM, left, right, search, 5, use_mgm=mgm, subpixel_mode=mode,
                                     bounds=b, p1=p1, p2=p2)


@pytest.mark.parametrize("mode", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("p1,p2", PENALTIES)
@pytest.mark.parametrize("case", list(R.SUBPIXEL_CASES))
def test_sgm_subpixel_matches_restatement(vwb, monkeypatch, case, p1, p2, mode):
    _, res, subs = restated(case, p1, p2)
    want, counts = subs[mode]
    gi, gf = run_case(vwb, monkeypatch, case, mode, p1, p2)
    assert np.array_equal(gi, res.disparity), f"{int((gi != res.disparity).any(-1).sum())} integer disparities differ"
    if mode in (2, 3):
        assert_bits(gf, want, f"{case}, mode {mode}")
    else:
        assert_float_contract(gf, want, exact_pixels(res, want, mode), f"{case} ({p1}, {p2}), mode {mode}")
    if mode == 1:
        assert counts["fit_rejected"] + counts["fit_kept"] + counts["fit_rescaled"] == int(res.disparity[..., 2].sum())
    if case == "wide-x" and mode == 2:
        big = res.disparity[..., 0] >= 128              # float32(dx + delta) rounds to 2^-16 there
        assert big.mean() > 0.5 and (gf[..., 0][big] != res.disparity[..., 0][big]).any()


@pytest.mark.parametrize("case", list(R.SUBPIXEL_CASES))
def test_sgm_branches_and_where_the_totals_live(vwb, monkeypatch, case):
    """the branches the case targets are reached (restatement counters over modes 1-5 and both penalty pairs), and the
    device kept the totals where the case says: summed in sgm_wta_kernel's shared memory, by sgm_sum4_kernel, or in
    one serial volume"""
    total = R.new_counts()
    for p1, p2 in PENALTIES:
        for _, counts in restated(case, p1, p2)[2].values():
            for k, v in counts.items():
                total[k] += v
    assert all(total[k] for k in TARGETS[case]), (case, total)
    _, names = sgm_kernels(lambda: run_case(vwb, monkeypatch, case, 5, 30000, 30000))
    where = R.SUBPIXEL_CASES[case][4]
    assert ("sgm_sum4_kernel" in names) == (where == "sum4"), (case, sorted(names))
    assert not any(n.startswith("mgm_") for n in names)


@pytest.mark.parametrize("mode", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("p1,p2", PENALTIES)
@pytest.mark.parametrize("case", ["moving-32", "full"])
def test_mgm_subpixel_matches_oracle(vwb, oracle, monkeypatch, case, p1, p2, mode):
    """MGM, which the restatement does not cover: the oracle's sub-pixel stage is checked against the restatement on
    the SGM cases, and here holds the device to the same float contract"""
    (left, right, b, search), _, _ = restated(case, 0, 0)
    ri, rf = oracle.sgm_calc_disparity_bounds(left, right, search, 5, b, subpixel_mode=mode, p1=p1, p2=p2, use_mgm=True)
    (gi, gf), names = sgm_kernels(lambda: run_case(vwb, monkeypatch, case, mode, p1, p2, mgm=True))
    assert any(n.startswith("mgm_") for n in names) and "sgm_sum4_kernel" not in names, sorted(names)
    assert np.array_equal(gi, ri)
    if mode in (2, 3):
        assert_bits(gf, rf, f"MGM {case}, mode {mode}")
    else:
        stub = R.SgmResult(ri, ri, None, None, 0, b, None, None, None)
        assert_float_contract(gf, rf, exact_pixels(stub, rf, mode), f"MGM {case} ({p1}, {p2}), mode {mode}")


# ---- ParabolaSubpixelView -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("disparity", PATCH_DISPARITIES)
def test_parabola_patches(vwb, disparity):
    """hand-made cost patches through a 1x1 kernel: all nine equal, eight equal, a 0 / 0 ridge, negative offsets, squared
    offset norms one ulp below 25, exactly 25 and one ulp above, disparities up to 200; bit for bit"""
    patches = np.concatenate(list(S.patch_set().values()))
    disp, left, right = S.patch_raster(patches, disparity)
    want = S.parabola_subpixel(disp, left, right, (1, 1))
    got = vwb.parabola_subpixel(disp, left, right, 0, 0.0, (1, 1)).rasterize()
    assert_bits(got, want, f"patches at {disparity}")
    edge = S.patch_raster(S.patch_set()["norm_edge"], disparity)
    got = vwb.parabola_subpixel(*edge, 0, 0.0, (1, 1)).rasterize()
    y, x = 3, 3
    assert got[y, x, 0] != disparity[0] and got[y, x + 4, 0] == disparity[0] and got[y, x + 8, 0] == disparity[0]


@pytest.mark.parametrize("kernel,base,spread,bboxes", SCENES)
def test_parabola_integer_imagery(vwb, kernel, base, spread, bboxes):
    """kernels 1x1 to 15x15, positive, negative and mixed ranges, bboxes on every border and of one pixel; bit for bit"""
    disp, left, right = scene(kernel, base, spread)
    view = vwb.parabola_subpixel(disp, left, right, 0, 0.0, kernel)
    for bbox in bboxes:
        want = S.parabola_subpixel(disp, left, right, kernel, bbox)
        assert_bits(view.rasterize(None, bbox), want, f"{kernel} {base} {bbox}")


def test_parabola_bbox_without_valid_pixels(vwb):
    disp, left, right, bbox = empty_bbox_case()
    got = vwb.parabola_subpixel(disp, left, right, 0, 0.0, (3, 3)).rasterize(None, bbox)
    assert_bits(got, S.parabola_subpixel(disp, left, right, (3, 3), bbox), "no valid pixel")
    assert not got.any()
