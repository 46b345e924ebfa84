"""The ipfind entry points without a device: argument checks come before the device lookup, valid calls answer
VWB200_ENODEVICE; the per-tile point counts and ipfind's ip_per_image conversion; the Harris taps, which the host computes,
equal the oracle's; and the oracle itself on small images (crop origins, partition order, culling and its ties)."""
import ctypes as C

import numpy as np
import pytest

EARG, ENODEVICE = -1, -6


@pytest.fixture(scope="module")
def v():
    import visionworkbench_b200 as v
    v.api._ipf()
    return v


@pytest.fixture(scope="module")
def ora():
    from oracle import ipfind
    return ipfind


def test_rejections(v):
    L = v.lib()
    img = np.zeros((8, 8), np.float32)
    out = np.zeros((8, 8), np.float32)
    pts = np.zeros(4, v.api._IPF_POINT)
    n = C.c_longlong(0)
    assert L.vwb200_ipfind_normalize(None, 8, 8, 8, 0, 0.0, out.ctypes.data, 8, 0, None) == EARG
    assert L.vwb200_ipfind_normalize(img.ctypes.data, 8, 8, 7, 0, 0.0, out.ctypes.data, 8, 0, None) == EARG
    assert L.vwb200_ipfind_normalize(img.ctypes.data, 8, 8, 8, 0, 0.0, img.ctypes.data + 4, 8, 0, None) == EARG
    assert L.vwb200_ipfind_detect(img.ctypes.data, 8, 8, 8, 1024, -1, pts.ctypes.data, 4, C.byref(n), 0, None) == EARG
    assert L.vwb200_ipfind_detect(img.ctypes.data, 8, 8, 8, 1024, 5, None, 4, C.byref(n), 0, None) == EARG
    assert L.vwb200_ipfind_detect(img.ctypes.data, 8, 8, 8, 1024, 5, pts.ctypes.data, 4, None, 0, None) == EARG
    n.value = 2
    assert L.vwb200_ipfind_remove_near_nodata(img.ctypes.data, 8, 8, 8, 0.0, -1, pts.ctypes.data, C.byref(n), 0, None) == EARG
    bad = pts.copy()
    bad["scale"] = 0
    d = np.zeros((4, 180), np.float32)
    assert L.vwb200_ipfind_describe(img.ctypes.data, 8, 8, 8, 1024, bad.ctypes.data, 4, d.ctypes.data, 0, None) == EARG
    if v.device_count() > 0:
        return
    assert L.vwb200_ipfind_normalize(img.ctypes.data, 8, 8, 8, 0, 0.0, out.ctypes.data, 8, 0, None) == ENODEVICE
    assert L.vwb200_ipfind_detect(img.ctypes.data, 8, 8, 8, 1024, 5, pts.ctypes.data, 4, C.byref(n), 0, None) == ENODEVICE
    n.value = 2
    assert L.vwb200_ipfind_remove_near_nodata(img.ctypes.data, 8, 8, 8, 0.0, 1, pts.ctypes.data, C.byref(n), 0, None) == ENODEVICE
    good = pts.copy()
    good["scale"] = 1
    assert L.vwb200_ipfind_describe(img.ctypes.data, 8, 8, 8, 1024, good.ctypes.data, 4, d.ctypes.data, 0, None) == ENODEVICE


def test_gaussian_taps_match_oracle(v, ora):
    got = v.ipfind_gaussian_taps()
    assert got.tobytes() == ora.gaussian_taps().tobytes()
    assert abs(got.sum() - 1) < 1e-12 and np.all(got == got[::-1])


def test_tile_counts(v):
    assert v.tile_num_ip(1024, 1024, 250) == 250
    assert v.tile_num_ip(1, 1030, 250) == 1                       # a 1-pixel sliver: ceil(0.245...) = 1
    assert v.tile_num_ip(6, 1024, 250) == 2                       # ceil(6 / 1024 * 250) = ceil(1.46) = 2
    assert v.tile_num_ip(2048, 2048, 10, tile_size=2048) == 10
    assert v.tile_num_ip(1024, 1024, 10, tile_size=2048) == 3      # ceil(0.25 * 10)
    assert v.tile_num_ip(5, 5, 0) == 0
    assert v.detection_tile_count(1025, 1030) == 4 and v.detection_tile_count(1, 4096, 256) == 4
    # ipfind.cc:255-262 uses the unclamped tile size
    assert v.ip_per_tile_for_image(1000, 8192, 8192, 256) == 1
    assert v.ip_per_tile_for_image(1000, 8192, 8192, 1024) == 16
    assert v.ip_per_tile_for_image(5000, 3000, 2000) == 874


def _texture(h, w, seed=0):
    rng = np.random.default_rng(seed)
    base = rng.random((h // 4 + 3, w // 4 + 3))
    img = np.kron(base, np.ones((4, 4)))[:h, :w]
    img = (img + np.roll(img, 1, 0) + np.roll(img, 1, 1) + np.roll(img, (1, 1), (0, 1))) / 4
    return np.floor(img * 255).astype(np.float32)


def test_oracle_detection_order_and_cull(ora):
    img = ora.normalize(_texture(200, 240, 1))
    pts, stats = ora.detect(img, ip_per_tile=0)
    assert len(pts) > 20 and stats[3] == 0
    # unculled: (scale, row, column) order
    key = [(p["scale"], p["iy"], p["ix"]) for p in pts]
    assert key == sorted(key)
    for k in (len(pts), len(pts) - 1, 5, 1):
        kept, st = ora.detect(img, ip_per_tile=k)
        num_ip = max(1, min(int(np.ceil(240 * 200 / 1024 ** 2 * k)), k))
        if len(pts) <= num_ip:
            assert kept.tobytes() == pts.tobytes() and st[3] == 0
        else:   # a stable sort by descending interest, then the first num_ip
            order = sorted(range(len(pts)), key=lambda i: -pts[i]["interest"])[:num_ip]
            assert kept.tobytes() == pts[order].tobytes() and st[3] == 1


def test_oracle_ties_keep_list_order(ora):
    tile = np.zeros((16, 16), np.float32)
    tile[6:9, 6:9] = 1                                              # odd blobs: a strict centre each
    img = np.tile(tile, (12, 12))                                   # equal interests everywhere
    pts, _ = ora.detect(ora.normalize(img), ip_per_tile=0)
    kept, _ = ora.detect(ora.normalize(img), ip_per_tile=400)
    n = len(kept)
    assert len(pts) > n                                            # the cull ran
    interests = pts["interest"]
    assert len(np.unique(interests)) < len(interests) // 2           # with many equal interests
    order = sorted(range(len(pts)), key=lambda i: -pts[i]["interest"])[:n]
    assert kept.tobytes() == pts[order].tobytes()


def test_oracle_describe_partition_and_crop(ora):
    img = ora.normalize(_texture(1100, 1050, 2))
    pts = np.zeros(4, ora.POINT)
    pts["x"] = [1040.25, 3.5, 1030.0, 500.75]
    pts["y"] = [10.0, 1090.0, 1070.5, 20.125]
    pts["scale"] = [1.5, 2.34375, 1.875, 5.722046]
    pts["orientation"] = [0, 0.5, -1.0, 0]
    out, desc = ora.describe(img, pts)
    # one point per tile, given as (1, 0), (0, 1), (1, 1), (0, 0): libstdc++'s bidirectional partition swaps the first
    # point outside the tile with the last one inside, tile by tile, giving (0, 0), (1, 0), (0, 1), (1, 1)
    assert list(out["y"]) == [np.float32(v) for v in (20.125, 10.0, 1090.0, 1070.5)]
    assert list(out["orientation"]) == [np.float32(v) for v in (0, 0, 0.5, -1.0)]
    assert np.allclose(np.linalg.norm(desc, axis=1), 1, atol=1e-5)


def test_oracle_detector_order_survives_partition(ora):
    img = ora.normalize(np.ascontiguousarray(np.kron(np.random.default_rng(4).random((330, 280)), np.ones((4, 4)))[:1300, :1100]))
    pts, _ = ora.detect(img, 30)
    out, _ = ora.describe(img, pts)
    assert out.tobytes() == pts.tobytes()        # integer coordinates, tile-ordered: the partition moves nothing
