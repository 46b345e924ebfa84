"""The sub-pixel stages of the oracle against restatements written from the reference: SGM's five models
(create_disparity_view_subpixel, through tests/sgm_reference.py) and ParabolaSubpixelView with PREFILTER_NONE (through
tests/subpixel_reference.py).  Bit for bit, floats included, so that a disagreement is located here before any GPU runs;
the GPU tests (test_gpu_subpixel.py) hold the device to the same restatements on the same inputs."""
import functools

import numpy as np
import pytest

import sgm_reference as R
import subpixel_reference as S

PENALTIES = [(0, 0), (30000, 30000)]
# the branches each SGM case is there to reach (counted over modes 1-5 on the restatement)
TARGETS = {
    "const-flat": ("ld_lt_rd", "ld_gt_rd", "ld_eq_rd", "fit_kept"),
    "const-textured": ("ld_lt_rd", "ld_gt_rd", "ld_eq_rd", "fit_kept"),
    "w1": ("both_bounds", "fit_rejected", "smoothed_winner"),
    "h1": ("both_bounds", "fit_rejected", "smoothed_winner"),
    "1x1": ("both_bounds", "fit_rejected"),
    "w2": ("two_value_left", "two_value_right", "fit_rescaled"),
    "h2": ("two_value_left", "two_value_right", "smoothed_winner"),
    "moving-32": ("two_value_left", "two_value_right", "smoothed_winner", "fit_rescaled"),
    "moving-48": ("ld_lt_rd", "ld_gt_rd", "smoothed_winner", "fit_kept"),
    "full": ("ld_lt_rd", "ld_gt_rd", "ld_eq_rd", "smoothed_winner"),
    "serial": ("ld_lt_rd", "ld_gt_rd", "smoothed_winner"),
    "wide-x": ("two_value_right", "ld_lt_rd", "ld_gt_rd", "fit_kept"),
}


@functools.lru_cache(maxsize=None)
def restated(case, p1, p2):
    """(inputs, SgmResult, {mode: (float raster, counts)}) of one case on the restatement"""
    left, right, b, search = R.subpixel_case(case)
    res = R.sgm(left, right, search, 5, b, p1, p2)
    subs = {}
    for mode in range(1, 6):
        counts = R.new_counts()
        subs[mode] = (R.subpixel_stage(res, mode, counts), counts)
    return (left, right, b, search), res, subs


def assert_bits(got, want, what):
    """float32 rasters identical bit for bit (NaN-free; -0.0 and +0.0 differ)"""
    diff = (np.asarray(got, np.float32).view(np.int32) != np.asarray(want, np.float32).view(np.int32)).any(-1)
    assert not diff.any(), f"{what}: {int(diff.sum())} of {diff.size} pixels differ, first at {np.argwhere(diff)[0].tolist()}"


def test_case_table_is_covered():
    assert set(TARGETS) == set(R.SUBPIXEL_CASES)


@pytest.mark.parametrize("p1,p2", PENALTIES)
@pytest.mark.parametrize("case", list(R.SUBPIXEL_CASES))
def test_sgm_subpixel_matches_restatement(oracle, case, p1, p2):
    """modes 1-5 of the oracle on the restatement's winners and smoothed boxes, floats bit for bit; every branch the
    case targets is reached"""
    (left, right, b, search), res, subs = restated(case, p1, p2)
    total = R.new_counts()
    for mode, (want, counts) in subs.items():
        ri, rf = oracle.sgm_calc_disparity_bounds(left, right, search, 5, b, subpixel_mode=mode, p1=p1, p2=p2)
        assert np.array_equal(ri, res.disparity), f"mode {mode}: integer disparities differ"
        assert_bits(rf, want, f"{case}, mode {mode}")
        for k, v in counts.items():
            total[k] += v
    missing = [k for k in TARGETS[case] if not total[k]]
    assert not missing, f"{case}: branches not reached: {missing} ({total})"
    if case == "wide-x":
        assert (res.disparity[..., 0] >= 128).mean() > 0.5


def test_sgm_every_branch_is_reached():
    """over the case table, every branch of the sub-pixel stage, and the tie smoothing on wrapped costs above 30000"""
    total = R.new_counts()
    for case in R.SUBPIXEL_CASES:
        for p1, p2 in PENALTIES:
            for _, counts in restated(case, p1, p2)[2].values():
                for k, v in counts.items():
                    total[k] += v
    assert all(total.values()), total
    _, res, _ = restated("h2", 30000, 30000)
    assert (res.smoothed & (res.lowest > 30000)).any()


def test_find_peak_hand_cases():
    """ParabolaFit2d::find_peak (SGMAssist.h:99-135): a flat box is rejected; a paraboloid with its vertex inside the
    half-pixel circle is kept; one with its vertex far away is rescaled onto the circle of radius 0.5"""
    assert R.find_peak([5] * 9) is None
    near = [(x - 0.2) ** 2 + (y + 0.1) ** 2 for y in (-1, 0, 1) for x in (-1, 0, 1)]
    dx, dy = R.find_peak(near)
    assert 0 < dx < 0.5 and -0.5 < dy < 0
    far = [(x + 3) ** 2 + y ** 2 for y in (-1, 0, 1) for x in (-1, 0, 1)]
    counts = R.new_counts()
    dx, dy = R.find_peak(far, counts)
    assert counts["fit_rescaled"] == 1 and abs(np.hypot(dx, dy) - 0.5) < 1e-12 and dx < 0


def test_compute_subpixel_offset_hand_cases():
    """SGM.cc:1445-1479: equal neighbours give 0; at a bound the two-value rule; inside, the model of the smaller
    difference over the larger one, towards the lower neighbour"""
    assert R.compute_subpixel_offset(9, 9, 9, False, False, 2) == 0.0
    assert R.compute_subpixel_offset(4, 4, 8, True, False, 2) == 0.25
    assert R.compute_subpixel_offset(8, 4, 4, False, True, 2) == -0.25
    assert R.compute_subpixel_offset(6, 4, 12, False, False, 2) == (1 / 8 - 0.5)     # ld < rd: shift left
    assert R.compute_subpixel_offset(12, 4, 6, False, False, 2) == -(1 / 8 - 0.5)    # ld > rd: shift right
    assert R.compute_subpixel_offset(7, 4, 7, False, False, 3) == -((1 + 1) / 4 - 0.5) == 0.0


# ---- ParabolaSubpixelView ---------------------------------------------------------------------------------------------------
PATCH_DISPARITIES = [(0, 0), (-2, -1), (3, 2), (130, -1), (200, 3)]


def test_patch_set_reaches_every_branch():
    patches = S.patch_set()
    counts = dict.fromkeys(S.BRANCHES, 0)
    for name, p in patches.items():
        S.refine(np.zeros((len(p), 2), int), np.ones(len(p), bool), p, counts)
    assert all(v for k, v in counts.items() if k != "invalid"), counts
    ox, oy, nn, denom = S.fit(patches["ridge"])
    assert ((denom == 0) & np.isnan(ox)).any(), "no ridge with a 0 / 0 offset"
    ox, oy, nn, _ = S.fit(patches["norm_edge"])
    f25 = np.float32(25)
    assert nn.tolist() == [np.nextafter(f25, 0), f25, np.nextafter(f25, 100)]
    assert S.accepted(nn).tolist() == [True, False, False]
    ox, oy, nn, _ = S.fit(patches["negative"])
    assert ((ox < 0) & (oy < 0) & S.accepted(nn)).any()


@pytest.mark.parametrize("disparity", PATCH_DISPARITIES)
def test_parabola_patches_match_restatement(oracle, disparity):
    """hand-made cost patches through a 1x1 kernel, every branch of the output loop, bit for bit"""
    patches = np.concatenate(list(S.patch_set().values()))
    disp, left, right = S.patch_raster(patches, disparity)
    counts = dict.fromkeys(S.BRANCHES, 0)
    want = S.parabola_subpixel(disp, left, right, (1, 1), counts=counts)
    assert counts["kept"] and counts["too_far"] and counts["all_equal"] and counts["denom_zero"]
    assert_bits(oracle.parabola_subpixel(disp, left, right, (1, 1)), want, f"patches at {disparity}")


# (kernel, base disparity, spread, bboxes): positive ranges take the bboxes on the left and top borders, where every
# right window stays inside the right image; negative and mixed ranges the right and bottom ones
SCENE = (48, 64)
BBOXES_POS = [None, (0, 0, 20, 48), (0, 0, 64, 9), (0, 39, 64, 48), (44, 0, 64, 48), (17, 11, 18, 12), (5, 6, 30, 29)]
BBOXES_NEG = [(30, 20, 64, 48), (20, 40, 64, 48), (50, 12, 64, 48), (40, 30, 41, 31)]
SCENES = [((1, 1), (12, 10), 2, BBOXES_POS), ((3, 3), (13, 11), 2, BBOXES_POS), ((7, 7), (14, 12), 1, BBOXES_POS),
          ((5, 9), (-6, -3), 2, BBOXES_NEG), ((15, 15), (-1, 0), 2, BBOXES_NEG), ((7, 7), (140, 6), 2, BBOXES_POS[:1])]


def scene(kernel, base, spread):
    seed = 90 + kernel[0] * 7 + kernel[1] + (base[0] & 0xff)
    return S.integer_scene(seed, SCENE, base, spread, kernel)


def empty_bbox_case():
    """a bbox whose pixels are all invalid: the range falls back to (0, 0) and nothing is refined"""
    disp, left, right = scene((3, 3), (12, 10), 2)
    disp[20:30, 20:30, 2] = 0
    return disp, left, right, (20, 20, 30, 30)


@pytest.mark.parametrize("kernel,base,spread,bboxes", SCENES)
def test_parabola_integer_imagery_matches_restatement(oracle, kernel, base, spread, bboxes):
    disp, left, right = scene(kernel, base, spread)
    for bbox in bboxes:
        counts = dict.fromkeys(S.BRANCHES, 0)
        want = S.parabola_subpixel(disp, left, right, kernel, bbox, counts)
        assert_bits(oracle.parabola_subpixel(disp, left, right, kernel, bbox=bbox), want, f"{kernel} {base} {bbox}")
    if bboxes is BBOXES_POS or bboxes is BBOXES_NEG:
        assert counts["kept"] or bbox[2] - bbox[0] == 1


def test_parabola_bbox_without_valid_pixels(oracle):
    disp, left, right, bbox = empty_bbox_case()
    want = S.parabola_subpixel(disp, left, right, (3, 3), bbox)
    assert not want.any()
    assert_bits(oracle.parabola_subpixel(disp, left, right, (3, 3), bbox=bbox), want, "no valid pixel")
