"""The interest point matching entry points without a device: vwb200_ip_match refuses bad arguments (VWB200_EARG) and a
Hamming descriptor too long for an exact float sum (VWB200_ENOIMPL) before it looks for a device, and answers
VWB200_ENODEVICE otherwise; vwb200_remove_duplicate_matches is host code and equals the oracle; the .vwip / .match writers and
readers follow MatcherIO.cc's packed little-endian layout byte for byte."""
import ctypes as C
import struct

import numpy as np
import pytest

import ipmatch_reference as ref

EARG, ENOIMPL, ENODEVICE = -1, -4, -6


@pytest.fixture(scope="module")
def v():
    import visionworkbench_b200 as v
    return v


def call(v, metric=0, n1=3, n2=4, dim=5, p1=None, p2=None, d1=True, d2=True, q1=True, q2=True, out=True, first=None, second=None):
    a = np.zeros((max(n1, 1), max(dim, 1)), np.float32)
    b = np.zeros((max(n2, 1), max(dim, 1)), np.float32)
    pa, pb = np.zeros(max(n1, 1), np.uint8), np.zeros(max(n2, 1), np.uint8)
    idx = np.zeros(max(n1, 1), np.int32)
    keep = (a, b, pa, pb, idx)
    rc = v.lib().vwb200_ip_match(metric, a.ctypes.data if d1 else None, pa.ctypes.data if q1 else None, n1, b.ctypes.data if d2 else None,
                                 pb.ctypes.data if q2 else None, n2, dim, dim if p1 is None else p1, dim if p2 is None else p2, 0.5,
                                 idx.ctypes.data if out else None, first(keep) if first else None, second(keep) if second else None, 0, None)
    return rc


def test_rejections(v):
    if v.device_count() > 0:
        pytest.skip("device present: the valid calls would run")
    assert call(v) == ENODEVICE
    assert call(v, metric=2) == EARG
    assert call(v, n1=-1) == EARG and call(v, n2=-1) == EARG and call(v, dim=-1) == EARG
    assert call(v, p1=4) == EARG and call(v, p2=-1) == EARG
    assert call(v, d1=False) == EARG and call(v, d2=False) == EARG and call(v, q1=False) == EARG and call(v, q2=False) == EARG
    assert call(v, out=False) == EARG
    # an empty list needs no pointer; D = 0 needs no descriptors
    assert call(v, n2=0, d2=False, q2=False) == ENODEVICE
    assert call(v, dim=0, d1=False, d2=False) == ENODEVICE
    # outputs overlapping each other or an input
    assert call(v, first=lambda k: k[4].ctypes.data) == EARG
    assert call(v, first=lambda k: k[0].ctypes.data) == EARG
    assert call(v, second=lambda k: k[2].ctypes.data) == EARG
    f = np.zeros(3)
    assert call(v, first=lambda k: f.ctypes.data, second=lambda k: f.ctypes.data + 8) == EARG
    assert call(v, first=lambda k: f.ctypes.data) == ENODEVICE
    # Hamming: 8 dim > 2^24 is not exact in float
    assert call(v, metric=1, dim=(1 << 21) + 1, n1=1, n2=1) == ENOIMPL
    assert call(v, metric=1, dim=1 << 21, n1=1, n2=1) == ENODEVICE


def test_python_errors(v):
    a = np.zeros((3, 4), np.float32)
    with pytest.raises(v.ArgumentErr):
        v.ip_match(a, [0] * 3, np.zeros((2, 5), np.float32), [0] * 2)           # descriptors of unequal length
    with pytest.raises(v.ArgumentErr):
        v.ip_match(a, [0] * 2, a, [0] * 3)                                       # polarities of another length
    with pytest.raises(v.ArgumentErr):
        v.ip_match(a, [0] * 3, a, [0] * 3, metric="cosine")
    with pytest.raises(v.NoImplErr):
        v.ip_match(np.zeros((1, (1 << 21) + 1), np.float32), [0], np.zeros((1, (1 << 21) + 1), np.float32), [0], metric="hamming")


@pytest.mark.parametrize("seed", range(3))
def test_remove_duplicates_on_the_host(v, seed):
    rng = np.random.default_rng(seed)
    xy1 = rng.integers(0, 5, (300, 2)).astype(np.float32) * rng.choice([-1, 1], (300, 2)).astype(np.float32)
    xy2 = rng.integers(0, 7, (300, 2)).astype(np.float32)
    from oracle import ipmatch as om
    got = v.remove_duplicates(xy1, xy2)
    assert got.tolist() == om.remove_duplicates(xy1, xy2).tolist() == ref.remove_duplicates(xy1, xy2).tolist()
    assert v.remove_duplicates(np.zeros((0, 2)), np.zeros((0, 2))).size == 0
    xy2[5, 0] = np.nan
    with pytest.raises(v.ArgumentErr):
        v.remove_duplicates(xy1, xy2)
    with pytest.raises(v.ArgumentErr):
        v.remove_duplicates(xy1, xy2[:10])


def test_remove_duplicates_abi_rejections(v):
    n = C.c_int()
    xy = np.zeros(4, np.float32)
    keep = np.zeros(2, np.int32)
    assert v.lib().vwb200_remove_duplicate_matches(xy.ctypes.data, xy.ctypes.data, -1, keep.ctypes.data, C.byref(n)) == EARG
    assert v.lib().vwb200_remove_duplicate_matches(None, xy.ctypes.data, 2, keep.ctypes.data, C.byref(n)) == EARG
    assert v.lib().vwb200_remove_duplicate_matches(xy.ctypes.data, xy.ctypes.data, 2, keep.ctypes.data, None) == EARG
    assert v.lib().vwb200_remove_duplicate_matches(xy.ctypes.data, xy.ctypes.data, 2, keep.ctypes.data, C.byref(n)) == 0
    assert n.value == 1 and keep[0] == 1


def record(x, y, ix, iy, ori, scale, interest, pol, octave, lvl, desc):
    return struct.pack("<ffiifff?IIQ", x, y, ix, iy, ori, scale, interest, pol, octave, lvl, len(desc)) + struct.pack(f"<{len(desc)}f", *desc)


def points(v):
    return v.interest_points([1.5, -2.25], [3.0, 4.75], [[0.5, 1, 2], [3, 4, 255.5]], polarity=[True, False], scale=[2.0, 1.0],
                             interest=[0.25, 9.0], orientation=[0.1, -0.2], octave=[1, 2], scale_lvl=[3, 4])


def test_vwip_layout(v, tmp_path):
    p = tmp_path / "a.vwip"
    v.write_binary_ip_file(str(p), points(v))
    want = struct.pack("<Q", 2) + record(1.5, 3.0, 1, 3, np.float32(0.1), 2.0, 0.25, True, 1, 3, [0.5, 1, 2]) \
        + record(-2.25, 4.75, -2, 4, np.float32(-0.2), 1.0, 9.0, False, 2, 4, [3, 4, 255.5])
    assert p.read_bytes() == want
    back = v.read_binary_ip_file(str(p))
    assert back.tobytes() == points(v).tobytes()
    assert back["descriptor"].tolist() == [[0.5, 1, 2], [3, 4, 255.5]] and back["polarity"].tolist() == [1, 0]


def test_match_layout(v, tmp_path):
    p = tmp_path / "a__b.match"
    a = points(v)
    b = v.interest_points([7.0, 8.0], [9.0, 10.0], [[1, 2, 3], [4, 5, 6]])
    v.write_binary_match_file(str(p), a, b)
    assert p.read_bytes() == struct.pack("<QQ", 2, 2) + a.tobytes() + b.tobytes()
    assert p.read_bytes()[16:16 + 45 + 12] == record(1.5, 3.0, 1, 3, np.float32(0.1), 2.0, 0.25, True, 1, 3, [0.5, 1, 2])
    ra, rb = v.read_binary_match_file(str(p))
    assert ra.tobytes() == a.tobytes() and rb.tobytes() == b.tobytes()
    e = tmp_path / "empty.match"
    v.write_binary_match_file(str(e), a[:0], b[:0])
    assert e.read_bytes() == struct.pack("<QQ", 0, 0)
    assert all(len(x) == 0 for x in v.read_binary_match_file(str(e)))
    with pytest.raises(IOError):
        v.write_binary_match_file(str(e), a, b[:1])
