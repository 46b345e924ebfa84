"""The ipfind oracle (oracle/vw_ipfind_oracle.c) against the reference's own unit tests (TestIntegral.IntegralSumming,
TestBoxFilter.ApplyBoxFilter / FilterView) and bit for bit against an independent numpy restatement that walks the
reference's loops (tests/ipfind_reference.py): normalize, the detector's list order unculled and culled (ties included),
remove_ip_near_nodata, and the descriptor's partition order, crop origins and 180 floats."""
import os

import numpy as np
import pytest

import ipfind_reference as ref
from oracle import ipfind as of

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_integral_summing_kat():
    """TestIntegral.cxx IntegralSumming on its sub.png"""
    from PIL import Image
    img = np.asarray(Image.open(os.path.join(GOLDEN, "ipfind_sub.png")).convert("L"), np.float32) / np.float32(255)
    I = of.integral(img)
    for size in range(10, 71, 10):
        block = np.float32(np.float32(np.float32(I[0, 0] + I[size, size]) - I[size, 0]) - I[0, size])
        actual = np.float32(0)
        for i in range(size):
            for j in range(size):
                actual = np.float32(actual + img[j, i])
        assert abs(float(actual) - float(block)) <= 1e-2


def test_box_filter_kats():
    """TestBoxFilter.cxx ApplyBoxFilter and FilterView: image(i, j) = count over i (column) then j (row)"""
    filt = [(0, 0, 1, 1, -9.0), (-1, -1, 3, 3, 1.0)]
    img3 = np.arange(9, dtype=np.float32).reshape(3, 3).T.copy()
    I3 = of.integral(img3)
    assert I3.shape == (4, 4)
    assert abs(of.box_filter(I3, filt)[1, 1]) < 1e-5
    img4 = np.arange(16, dtype=np.float32).reshape(4, 4).T.copy()
    img4[3, 3] = 20
    out = of.box_filter(of.integral(img4), filt)
    assert out.shape == (4, 4)
    assert abs(out[1, 1]) < 1e-5 and abs(out[2, 2] - 5) < 1e-5 and abs(out[2, 1]) < 1e-5 and abs(out[1, 2]) < 1e-5


def texture(h, w, seed, cell=3):
    rng = np.random.default_rng(seed)
    base = rng.random((h // cell + 2, w // cell + 2))
    return np.floor(np.kron(base, np.ones((cell, cell)))[:h, :w] * 255).astype(np.float32)


def same(oracle_pts, ref_pts):
    got = [tuple(p.item()) for p in oracle_pts]
    want = [tuple(np.float32(v).item() if isinstance(v, (np.floating, float)) else int(v) for v in p) for p in ref_pts]
    assert len(got) == len(want)
    for g, r in zip(got, want):
        assert np.array(g[:2], np.float32).tobytes() == np.array(r[:2], np.float32).tobytes()
        assert g[2:4] == r[2:4]
        assert np.array(g[4:], np.float32).tobytes() == np.array(r[4:], np.float32).tobytes()


def test_integral_and_interest_match_restatement():
    img = of.normalize(texture(40, 36, 1))
    I = of.integral(img)
    assert I.tobytes() == ref.integral(img).tobytes()
    assert np.array(of.gaussian_taps()).tobytes() == np.array(ref.gaussian_taps()).tobytes()


@pytest.mark.parametrize("nodata", [None, 0.0])
def test_normalize_matches_restatement(nodata):
    raw = texture(30, 40, 2)
    raw[3:6, 4:9] = 0
    assert of.normalize(raw, nodata).tobytes() == ref.normalize(raw, nodata).tobytes()


@pytest.mark.parametrize("case", ["texture", "ties"])
def test_detect_matches_restatement(case):
    if case == "texture":
        img = of.normalize(texture(72, 80, 3))
    else:
        tile = np.zeros((16, 16), np.float32)
        tile[6:9, 6:9] = 1
        img = of.normalize(np.tile(tile, (5, 5)))
    allp, _ = of.detect(img, 0)
    want_all = ref.detect(img, 0)
    same(allp, want_all)
    n = len(allp)
    assert n >= 4
    frac = img.shape[0] * img.shape[1] / 1024.0 ** 2
    # num_ip == count (the unsorted list), then well below it (the stable sort, ties kept in list order)
    for target in (n, n // 2):
        ipt = int(np.floor(target / frac))
        while int(np.ceil(frac * ipt)) > target:
            ipt -= 1
        got, st = of.detect(img, ipt)
        same(got, ref.detect(img, ipt))
        assert st[3] == (1 if int(np.ceil(frac * ipt)) < n else 0)
    if case == "ties":
        assert len(np.unique(allp["interest"])) < n // 2


def test_remove_near_nodata_matches_restatement():
    raw = texture(60, 64, 4)
    raw[20:24, 30:33] = 0
    img = of.normalize(raw)
    pts, _ = of.detect(img, 0)
    for radius in (1, 2, 3):
        got = of.remove_near_nodata(raw, pts, 0.0, radius)
        same(got, ref.remove_near_nodata(raw, [tuple(p.item()) for p in pts], 0.0, radius))


def test_describe_matches_restatement():
    """points in four tiles given out of tile order (the partition swaps them), at the borders, with orientations and
    non-integer coordinates (the crop round trip rounds them)"""
    img = of.normalize(texture(1100, 1060, 5, cell=5))
    pts = np.zeros(7, of.POINT)
    pts["x"] = [1040.25, 3.5, 1030.0, 500.75, 0.0, 1059.9, 1023.999]
    pts["y"] = [10.0, 1090.0, 1070.5, 20.125, 0.0, 1099.5, 517.3]
    pts["ix"], pts["iy"] = pts["x"].astype(np.int32), pts["y"].astype(np.int32)
    pts["scale"] = [1.5, 2.34375, 1.875, 5.722046, 1.2, 3.662109, 4.577636]
    pts["orientation"] = [0, 0.5, -1.0, 0, 2.5, -3.0, 0.25]
    got, desc = of.describe(img, pts)
    want, wdesc = ref.describe(img, [tuple(p.item()) for p in pts])
    same(got, want)
    assert desc.tobytes() == np.array(wdesc, np.float32).tobytes()
