"""The CAHV / CAHVOR entry points without a device: vwb200_linearize_camera, vwb200_cahv_epipolar and vwb200_pinhole_to_cahv
are host arithmetic and equal the oracle as raw bits; the device entry points refuse bad arguments (VWB200_EARG), cameras at
different centers (VWB200_ELOGIC) and a CAHVOR destination (VWB200_ENOIMPL) before they look for a device, and return
VWB200_ENODEVICE with valid arguments; the Python layer refuses pinhole / CAHV mixes (NoImplErr); and the text format
round-trips and reads the reference's cahvor.txt."""
import ctypes as C
import os

import numpy as np
import pytest

import cahv_reference as cr
from oracle import cahv as oc
from oracle import triangulate as ot

EARG, ELOGIC, ENOIMPL, ENODEVICE = -1, -3, -4, -6
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def v():
    import visionworkbench_b200 as v
    return v


def st(v, c):
    return v.api.Cahv.from_buffer_copy(oc.to_struct(c))


def same_cam(a, b):
    keys = "CAHV" if a["model"] == 1 else "CAHVOR"
    return a["model"] == b["model"] and all(np.array_equal(np.asarray(a[k]).view(np.uint64), np.asarray(b[k]).view(np.uint64)) for k in keys)


def from_api(s):
    return oc.from_struct(oc.Cahv.from_buffer_copy(s))


CAHVORS = [cr.CAHVOR_TXT, cr.FR_CAHVOR] + [cr.rover(s, 640, 480, left=s % 2 == 1) for s in range(4)] + [cr.rover(9, 64, 48, r=(0.0, -3.0, -4.0))]


@pytest.mark.parametrize("size", [(1, 1), (640, 480), (641, 479), (1023, 1025)])
def test_linearize_equals_oracle(v, size):
    for c in CAHVORS:
        out = v.api.Cahv()
        assert v.lib().vwb200_linearize_camera(C.byref(st(v, c)), (C.c_int32 * 2)(*size), (C.c_int32 * 2)(*size[::-1]), C.byref(out)) == 0
        assert same_cam(from_api(out), oc.linearize(c, size, size[::-1]))


def test_epipolar_equals_oracle(v):
    cams = [cr.FR_CAHV] + [cr.rover(s, 640, 480, center=(0.0, 0.1 * s, 0.0), model=1, left=s == 2) for s in range(4)]
    for a in cams:
        for b in cams:
            e0, e1 = v.api.Cahv(), v.api.Cahv()
            assert v.lib().vwb200_cahv_epipolar(C.byref(st(v, a)), C.byref(st(v, b)), C.byref(e0), C.byref(e1)) == 0
            r0, r1 = oc.epipolar(a, b)
            assert same_cam(from_api(e0), r0) and same_cam(from_api(e1), r1)


def test_pinhole_to_cahv_equals_oracle(v):
    rng = np.random.default_rng(5)
    from scipy.spatial.transform import Rotation
    for k in range(8):
        cam = ot.camera(center=tuple(rng.normal(0, 5, 3)), rotation=Rotation.from_rotvec(rng.normal(0, 0.5, 3)).as_matrix(), fu=400.0 + k,
                        fv=410.0, cu=160.5, cv=-3.0, pixel_pitch=(1.0, 0.1, 0.0125)[k % 3])
        if k % 4 == 3:
            cam.update(u=(0.0, 1.0, 0.0), v=(1.0, 0.0, 0.0), w=(0.0, 0.0, -1.0))
        p = v.api.Pinhole.from_buffer_copy(ot.pinhole(cam))
        out = v.api.Cahv()
        assert v.lib().vwb200_pinhole_to_cahv(C.byref(p), C.byref(out)) == 0
        assert same_cam(from_api(out), oc.from_pinhole(ot.pinhole(cam)))


def test_host_rejections(v):
    L, c, good = v.lib(), v.api.Cahv(), st(v, cr.CAHVOR_TXT)
    sz = (C.c_int32 * 2)(10, 10)
    assert L.vwb200_linearize_camera(None, sz, sz, C.byref(c)) == EARG
    assert L.vwb200_linearize_camera(C.byref(good), None, sz, C.byref(c)) == EARG
    assert L.vwb200_linearize_camera(C.byref(st(v, cr.FR_CAHV)), sz, sz, C.byref(c)) == EARG          # a CAHV camera
    bad = st(v, cr.CAHVOR_TXT)
    bad.model = 7
    assert L.vwb200_linearize_camera(C.byref(bad), sz, sz, C.byref(c)) == EARG
    assert L.vwb200_cahv_epipolar(C.byref(good), C.byref(good), C.byref(c), C.byref(c)) == EARG     # CAHVOR sources
    assert L.vwb200_cahv_epipolar(C.byref(st(v, cr.FR_CAHV)), None, C.byref(c), C.byref(c)) == EARG
    cam = ot.camera(fu=100.0, fv=100.0, pixel_pitch=0.0)
    assert L.vwb200_pinhole_to_cahv(C.byref(v.api.Pinhole.from_buffer_copy(ot.pinhole(cam))), C.byref(c)) == EARG
    cam = ot.camera(fu=100.0, fv=100.0, tsai=(0.1, 0, 0, 0, 0))
    assert L.vwb200_pinhole_to_cahv(C.byref(v.api.Pinhole.from_buffer_copy(ot.pinhole(cam))), C.byref(c)) == EARG
    cam = ot.camera(fu=100.0, fv=100.0, u=(1.0, 1.0, 0.0))
    assert L.vwb200_pinhole_to_cahv(C.byref(v.api.Pinhole.from_buffer_copy(ot.pinhole(cam))), C.byref(c)) == ELOGIC


def test_device_entry_points_without_a_device(v):
    if v.device_count() > 0:
        pytest.skip("a device is present")
    L = v.lib()
    src, dst = cr.rover(1, 40, 30), None
    dst = oc.linearize(src, (40, 30), (40, 30))
    s, d = st(v, src), st(v, dst)
    img = np.zeros((30, 40), np.float32)
    out = np.zeros((30, 40), np.float32)
    ev = (C.c_float * 2)(0, 0)
    args = lambda a, b, pt=0, interp=0, edge=0, w=40: (C.byref(a), C.byref(b), pt, interp, edge, ev, img.ctypes.data, w, 30, 40, 0, 0,
                                                        out.ctypes.data, 40, 30, 40, 0, None)
    assert L.vwb200_cahv_camera_transform(*args(s, d)) == ENODEVICE
    assert L.vwb200_cahv_camera_transform(*args(s, d, pt=5)) == EARG
    assert L.vwb200_cahv_camera_transform(*args(s, d, w=0)) == EARG
    far = st(v, dict(dst, C=(0.0, 0.0, 1.0)))
    assert L.vwb200_cahv_camera_transform(*args(s, far)) == ELOGIC
    assert L.vwb200_cahv_camera_transform(*args(d, s)) == ENOIMPL                                    # CAHVOR destination
    disp = np.zeros((30, 40, 3), np.float32)
    xyz = np.zeros((30, 40, 3))
    err = np.zeros((30, 40))
    c1 = st(v, cr.rover(2, 40, 30, center=(0.0, 1.0, 0.0)))
    tri = lambda pt=1, a=s: L.vwb200_cahv_stereo_triangulate(pt, disp.ctypes.data, 40, 30, 40, 0, 0, 40, 30, C.byref(a), C.byref(c1), 0.0,
                                                             xyz.ctypes.data, 40, 0, None)
    assert tri() == ENODEVICE
    assert tri(pt=3) == EARG
    bad = st(v, src)
    bad.model = 0
    assert tri(a=bad) == EARG
    assert L.vwb200_cahv_stereo_model_points(disp.ctypes.data, 40, 30, 40, C.byref(s), C.byref(c1), 0.0, xyz.ctypes.data, 40, err.ctypes.data,
                                             40, 0, None) == ENODEVICE
    assert L.vwb200_cahv_stereo_model_points(disp.ctypes.data, 40, 30, 40, None, C.byref(c1), 0.0, xyz.ctypes.data, 40, err.ctypes.data,
                                             40, 0, None) == EARG


def test_pinhole_cahv_mix_is_noimpl(v):
    pin = v.PinholeModel((0, 0, 0), np.eye(3), 100, 100, 20, 15)
    cahv = v.CAHVModel.from_pinhole(pin)
    img = np.zeros((30, 40), np.float32)
    with pytest.raises(v.NoImplErr):
        v.camera_transform(img, pin, cahv)
    with pytest.raises(v.NoImplErr):
        v.stereo_triangulate(np.zeros((30, 40, 3), np.float32), cahv, pin)
    with pytest.raises(v.NoImplErr):
        v.epipolar(pin, cahv)


def test_string_read_kat(v):
    c = v.CAHVORModel.read(os.path.join(HERE, "golden", "cahvor.txt"))
    want = {"C": (76, -34, 20), "A": np.array([1, 2, 3.0]) / np.sqrt(14), "H": (1300, 123, 456), "V": (345, 900, 157),
            "O": np.array([2, 3, 4.0]) / np.sqrt(29), "R": (1, -1, 1)}
    for k, w in want.items():
        assert np.allclose(getattr(c, k), w, atol=1e-5), k
    assert c.type() == "CAHVOR"


def test_text_round_trip(v, tmp_path):
    c = v.CAHVORModel(*(cr.rover(3, 640, 480)[k] for k in "CAHVOR"))
    c.write(str(tmp_path / "a.cahvor"))
    r = v.CAHVORModel.read(str(tmp_path / "a.cahvor"))
    assert all(getattr(r, k) == getattr(c, k) for k in "CAHVOR")
    h = v.CAHVModel(*(cr.FR_CAHV[k] for k in "CAHV"))
    h.write(str(tmp_path / "b.cahv"))
    assert all(getattr(v.CAHVModel.read(str(tmp_path / "b.cahv")), k) == getattr(h, k) for k in "CAHV")
    (tmp_path / "c.cahv").write_text("BLAH Camera\nC= 1 2 3\nA =0 0 1\nH = 1 0 0\nV = 0 1 0\n")
    r = v.CAHVModel.read(str(tmp_path / "c.cahv"))
    assert r.C == (1.0, 2.0, 3.0) and r.V == (0.0, 1.0, 0.0)
    (tmp_path / "d.cahv").write_text("C = 1 2 3\nX = 0 0 1\n")
    with pytest.raises(v.IOErr):
        v.CAHVModel.read(str(tmp_path / "d.cahv"))


@pytest.mark.parametrize("text,ok", [
    ("BLAH BLAH I'm a Comment\nC = 1 2 3\nA = 0 0 1\nH = 1 0 0\nV = 0 1 0\n", True),
    ("C=1 2 3 A=0 0 1 H=1 0 0 V=0 1 .5e-3", True),
    ("C = -1.5E+2 2 3\nA = 0 0 1\nH = 1 0 0\nV = 0 1 5.", True),
    ("CC = 1 2 3\nA = 0 0 1\nH = 1 0 0\nV = 0 1 0\n", False),      # the second C is read as the character after the first
    ("C = 1 2 3\nA = 0 0 1\nH = 1 0 0\nV = 0 1 nan\n", False),     # istream >> double takes no nan, inf or hex
    ("C = 1 2 3\nA = 0 0 1\nH = 1 0 0\nV = 0 1 inf\n", False),
    ("C = 1 2 3\nA = 0 0 1\nH = 1 0 0\nV = 0 1 0x10\n", True),     # reads the 0, leaves x10
    ("C = 1 2 3\nA = 0 0 1\nH = 1 0 0\nV = 0 1 1e\n", False),
    ("C = 1 2 3\nA = 0 0 1\nH = 1 0 0\nV = 0 1 1e999\n", False),   # overflow sets failbit
    ("C = 1 2 3\nA = 0 0 1\nH = 1 0 0\nV = 0 1 .\n", False),
    ("C = 1 2 3\nA = 0 0 1\nH = 1 0 0\nV = 0 1\n", False),
    ("no camera here", False),
])
def test_reader_follows_the_stream_grammar(v, tmp_path, text, ok):
    p = str(tmp_path / "c.cahv")
    with open(p, "w") as f:
        f.write(text)
    if ok:
        c = v.CAHVModel.read(p)
        assert len(c.V) == 3 and all(np.isfinite(c.V))
    else:
        with pytest.raises(v.IOErr):
            v.CAHVModel.read(p)
