"""The epipolar entry points without a device: vwb200_pinhole_epipolar is host arithmetic and equals the oracle as raw bits;
vwb200_resize_epipolar_cameras_to_fit and vwb200_camera_transform refuse bad arguments (VWB200_EARG), cameras at different
centers or with a non-orthonormal frame (VWB200_ELOGIC) and the combinations without a device form (VWB200_ENOIMPL) before
they look for a device; with valid arguments and no device the answer is VWB200_ENODEVICE."""
import ctypes as C

import numpy as np
import pytest

from oracle import epipolar as oe
from oracle import triangulate as ot
from test_oracle_epipolar import cam_bits, tilted_rig
from test_oracle_triangulate import STRONG, TSAI, TSAI_K3

EARG, ELOGIC, ENOIMPL, ENODEVICE = -1, -3, -4, -6
GRAY, MASK = 0, 1
BILINEAR, BICUBIC, NEAREST = 0, 1, 2
ZERO, CONSTANT, VALUE = 0, 1, 2


@pytest.fixture(scope="module")
def L():
    import visionworkbench_b200 as v
    return v.lib()


def pin(cam):
    from visionworkbench_b200 import api
    return api.Pinhole.from_buffer_copy(ot.pinhole(cam))


@pytest.mark.parametrize("seed", range(6))
def test_epipolar_equals_oracle(L, seed):
    lenses = (None, TSAI, TSAI_K3, STRONG)
    cams = tilted_rig(40 + seed, lenses[seed % 4], lenses[(seed + 2) % 4], pitch=(1.0, 0.05)[seed % 2], frame=seed % 3 == 1)
    if seed == 5:
        cams[1]["center"] = cams[0]["center"]                     # coincident centers: NaN cameras, no error
    from visionworkbench_b200 import api
    a, b = api.Pinhole(), api.Pinhole()
    assert L.vwb200_pinhole_epipolar(C.byref(pin(cams[0])), C.byref(pin(cams[1])), C.byref(a), C.byref(b)) == 0
    w0, w1 = oe.epipolar(*cams)
    assert cam_bits(oe.from_pinhole(a), w0) and cam_bits(oe.from_pinhole(b), w1)
    assert a.lens == 0 and a.num_lens_params == 0


def test_epipolar_in_place(L):
    """the outputs may be the input cameras themselves"""
    cams = tilted_rig(47, TSAI, None)
    a, b = pin(cams[0]), pin(cams[1])
    assert L.vwb200_pinhole_epipolar(C.byref(a), C.byref(b), C.byref(a), C.byref(b)) == 0
    w0, w1 = oe.epipolar(*cams)
    assert cam_bits(oe.from_pinhole(a), w0) and cam_bits(oe.from_pinhole(b), w1)


def test_epipolar_rejections(L):
    from visionworkbench_b200 import api
    c = pin(ot.camera())
    out = api.Pinhole()
    assert L.vwb200_pinhole_epipolar(None, C.byref(c), C.byref(out), C.byref(out)) == EARG
    assert L.vwb200_pinhole_epipolar(C.byref(c), C.byref(c), None, C.byref(out)) == EARG
    bad = pin(ot.camera(w=(0, 0, 1.01)))
    assert L.vwb200_pinhole_epipolar(C.byref(c), C.byref(bad), C.byref(out), C.byref(out)) == ELOGIC


def transform(L, *, src=None, dst=None, ptype=GRAY, interp=BILINEAR, edge=ZERO, ev=True, inp=True, w=8, h=8, pitch=8, ow=8, oh=8, opitch=8,
              out=None, x0=0, y0=0):
    img = np.zeros((16, 16, 2), np.float32)
    o = np.zeros((16, 16, 2), np.float32)
    src = pin(ot.camera(fu=10, fv=10, tsai=TSAI)) if src is None else src
    dst = pin(ot.camera(fu=12, fv=12)) if dst is None else dst
    e = (C.c_float * 2)(0.0, 0.0) if ev else None
    return L.vwb200_camera_transform(C.byref(src), C.byref(dst), ptype, interp, edge, e, img.ctypes.data if inp else None, w, h, pitch, x0, y0,
                                     o.ctypes.data if out is None else out, ow, oh, opitch, 0, None)


def test_camera_transform_rejections(L):
    img = np.zeros(64, np.float32)
    assert transform(L, inp=False) == EARG
    assert transform(L, ptype=2) == EARG
    assert transform(L, interp=3) == EARG
    assert transform(L, edge=3) == EARG
    assert transform(L, edge=VALUE, ptype=MASK, ev=False) == EARG
    assert transform(L, w=0) == EARG
    assert transform(L, pitch=7) == EARG
    assert transform(L, oh=0) == EARG
    assert transform(L, opitch=7) == EARG
    assert transform(L, x0=2 ** 31 - 4) == EARG
    assert L.vwb200_camera_transform(C.byref(pin(ot.camera())), C.byref(pin(ot.camera())), GRAY, 0, 0, None, img.ctypes.data, 8, 8, 8, 0, 0,
                                     img[4:].ctypes.data, 8, 1, 8, 0, None) == EARG          # out overlaps the image
    assert transform(L, dst=pin(ot.camera(center=(0, 0, 1e-9)))) == ELOGIC
    assert transform(L, dst=pin(ot.camera(u=(0, 1, 0)))) == ELOGIC
    assert transform(L, ptype=MASK, interp=BICUBIC) == ENOIMPL
    assert transform(L, ptype=MASK, interp=NEAREST, edge=VALUE) == ENOIMPL
    assert transform(L, ptype=GRAY, edge=VALUE) == ENOIMPL
    if L.vwb200_device_count() == 0:
        for kw in (dict(), dict(ptype=MASK, edge=VALUE), dict(interp=BICUBIC, edge=CONSTANT)):
            assert transform(L, **kw) == ENODEVICE


def test_resize_rejections(L):
    from visionworkbench_b200 import api
    cams = [pin(c) for c in tilted_rig(3, TSAI, None)]
    epis = [api.Pinhole(), api.Pinhole()]
    assert L.vwb200_pinhole_epipolar(C.byref(cams[0]), C.byref(cams[1]), C.byref(epis[0]), C.byref(epis[1])) == 0
    roi = (C.c_int32 * 4)(0, 0, 64, 48)
    s1, s2 = (C.c_int32 * 2)(), (C.c_int32 * 2)()

    def call(c1=cams[0], c2=cams[1], e1=epis[0], e2=epis[1], r1=roi, r2=roi, a=s1, b=s2):
        return L.vwb200_resize_epipolar_cameras_to_fit(*(None if x is None else C.byref(x) for x in (c1, c2, e1, e2)), r1, r2, a, b, None)

    assert call(c1=None) == EARG
    assert call(a=None) == EARG
    assert call(r2=None) == EARG
    assert call(r1=(C.c_int32 * 4)(5, 0, 4, 10)) == EARG
    assert call(e1=epis[1]) == ELOGIC                                 # cam1 and its epipolar camera at different centers
    if L.vwb200_device_count() == 0:
        assert call() == ENODEVICE


def test_python_surface_without_device():
    import visionworkbench_b200 as v
    c0 = v.PinholeModel((0, 0, 0), np.eye(3), 500, 500, 320, 240, distortion_model=v.TsaiLensDistortion(TSAI))
    c1 = v.PinholeModel((1, 0, 0), np.eye(3), 500, 500, 320, 240)
    e0, e1 = v.epipolar(c0, c1)
    assert isinstance(e0.distortion, v.NullLensDistortion) and e1.camera_center == (1.0, 0.0, 0.0)
    img = np.zeros((4, 5, 2), np.float32)
    with pytest.raises(v.NoImplErr):
        v.epipolar_transformed_images(c0, c1, e0, e1, img, img, (5, 4), (5, 4), left_roi=(1, 0, 5, 4))
    with pytest.raises(v.ArgumentErr):
        v.camera_transform(np.zeros((4, 5, 3), np.float32), c0, e0)
    with pytest.raises(v.LogicErr):
        v.camera_transform(img, c0, e1)
