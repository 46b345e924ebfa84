"""The triangulation entry points refuse bad arguments (VWB200_EARG), non-orthonormal frames (VWB200_ELOGIC) and singular
camera matrices (VWB200_EMATH) before they look for a device, so these run without one; with valid arguments and no device
the answer is VWB200_ENODEVICE."""
import ctypes as C

import numpy as np
import pytest

from oracle import triangulate as ot

EARG, EMATH, ELOGIC, ENODEVICE = -1, -2, -3, -6
I32, F32 = 0, 1


@pytest.fixture(scope="module")
def L():
    import visionworkbench_b200 as v
    return v.lib()


def cam(**kw):
    """the engine's vwb200_pinhole of an oracle camera"""
    from visionworkbench_b200 import api
    return api.Pinhole.from_buffer_copy(ot.pinhole(ot.camera(**kw)))


def no_device(L):
    return L.vwb200_device_count() == 0


def tri(L, *, ptype=F32, inp=None, w=8, h=8, pitch=8, x0=0, y0=0, ow=8, oh=8, c1=None, c2=None, out=None, opitch=8):
    d = np.zeros((16, 16, 3), np.float32)
    o = np.zeros((16, 16, 3))
    c1 = cam() if c1 is None else c1
    c2 = cam(center=(1, 0, 0)) if c2 is None else c2
    return L.vwb200_stereo_triangulate(ptype, d.ctypes.data if inp is None else inp, w, h, pitch, x0, y0, ow, oh,
                                       None if c1 is False else C.byref(c1), None if c2 is False else C.byref(c2), 0.0,
                                       o.ctypes.data if out is None else out, opitch, 0, None)


def tsai_short():
    p = cam(tsai=(0.1, 0, 0, 0, 0))
    p.num_lens_params = 4
    return p


def lens7():
    p = cam()
    p.lens = 7
    return p


def null_with_params():
    p = cam()
    p.num_lens_params = 5
    return p


@pytest.mark.parametrize("kw", [dict(ptype=2), dict(w=0), dict(h=-1), dict(pitch=7), dict(ow=0), dict(oh=0), dict(opitch=7),
                                dict(x0=-1), dict(y0=-1), dict(x0=1), dict(y0=1), dict(ow=9), dict(x0=4, ow=5)],
                         ids=lambda k: ",".join(f"{a}={b}" for a, b in k.items()))
def test_triangulate_rejects(L, kw):
    assert tri(L, **kw) == EARG
    assert L.vwb200_last_error()


@pytest.mark.parametrize("which", ["null1", "null2", "tsai_short", "lens7", "null_with_params"])
def test_triangulate_rejects_cameras(L, which):
    c = {"null1": dict(c1=False), "null2": dict(c2=False), "tsai_short": dict(c2=tsai_short()), "lens7": dict(c1=lens7()),
         "null_with_params": dict(c1=null_with_params())}[which]
    assert tri(L, **c) == EARG


def test_null_pointers_and_overlap(L):
    d = np.zeros((8, 8, 3), np.float32)
    c1, c2 = cam(), cam(center=(1, 0, 0))
    o = np.zeros((8, 8, 3))
    assert L.vwb200_stereo_triangulate(F32, None, 8, 8, 8, 0, 0, 8, 8, C.byref(c1), C.byref(c2), 0.0, o.ctypes.data, 8, 0, None) == EARG
    assert L.vwb200_stereo_triangulate(F32, d.ctypes.data, 8, 8, 8, 0, 0, 8, 8, C.byref(c1), C.byref(c2), 0.0, None, 8, 0, None) == EARG
    big = np.zeros(8 * 8 * 3 * 8, np.uint8)                       # xyz over the disparity's bytes
    assert L.vwb200_stereo_triangulate(F32, big.ctypes.data, 8, 8, 8, 0, 0, 2, 2, C.byref(c1), C.byref(c2), 0.0, big[48:].ctypes.data, 2, 0,
                                       None) == EARG
    assert b"overlaps" in L.vwb200_last_error()
    e = np.zeros((8, 8))
    assert L.vwb200_stereo_model_points(d.ctypes.data, 8, 8, 8, C.byref(c1), C.byref(c2), 0.0, o.ctypes.data, 8, None, 8, 0, None) == EARG
    assert L.vwb200_stereo_model_points(d.ctypes.data, 8, 8, 8, C.byref(c1), C.byref(c2), 0.0, o.ctypes.data, 8, e.ctypes.data, 7, 0, None) == EARG
    assert L.vwb200_stereo_model_points(d.ctypes.data, 0, 8, 8, C.byref(c1), C.byref(c2), 0.0, o.ctypes.data, 8, e.ctypes.data, 8, 0, None) == EARG
    assert L.vwb200_stereo_model_points(d.ctypes.data, 8, 8, 8, C.byref(c1), None, 0.0, o.ctypes.data, 8, e.ctypes.data, 8, 0, None) == EARG
    assert L.vwb200_stereo_model_points(d.ctypes.data, 8, 8, 8, C.byref(c1), C.byref(c2), 0.0, o.ctypes.data, 8, o.ctypes.data + 8, 8, 0,
                                        None) == EARG                # error inside xyz
    assert b"overlap" in L.vwb200_last_error()


def test_camera_logic_and_math_errors(L):
    """the u, v, w asserts of rebuild_camera_matrix (LogicErr) and a singular K or uvw * R^T (MathErr), checked before the
    device, on both the triangulation forms"""
    d = np.zeros((8, 8, 3), np.float32)
    o, e = np.zeros((8, 8, 3)), np.zeros((8, 8))
    good = cam(center=(1, 0, 0))
    cases = [(cam(w=(0, 0, 1.01)), ELOGIC), (cam(u=(1, 0, 0), v=(1e-3, 1, 0), w=(0, 0, 1)), ELOGIC), (cam(fu=0.0), EMATH),
             (cam(rotation=np.zeros((3, 3))), EMATH), (cam(u=(np.nan, 0, 0)), ELOGIC)]
    for bad, rc in cases:
        assert tri(L, c1=bad, c2=good) == rc
        assert L.vwb200_stereo_model_points(d.ctypes.data, 8, 8, 8, C.byref(good), C.byref(bad), 0.0, o.ctypes.data, 8, e.ctypes.data, 8, 0,
                                            None) == rc
    assert tri(L, c1=cam(w=(0, 0, 1.0009)), c2=good) in (0, ENODEVICE)       # a norm within 0.001 of 1 passes


def test_universe_radius_rejects(L):
    p = np.zeros((4, 4, 3))
    o = np.zeros((4, 4, 3))
    org = np.zeros(3)
    ur = L.vwb200_universe_radius
    assert ur(None, 4, 4, 4, org.ctypes.data, 0.0, 1.0, o.ctypes.data, 4, None, None, 0, None) == EARG
    assert ur(p.ctypes.data, 4, 4, 4, None, 0.0, 1.0, o.ctypes.data, 4, None, None, 0, None) == EARG
    assert ur(p.ctypes.data, 0, 4, 4, org.ctypes.data, 0.0, 1.0, o.ctypes.data, 4, None, None, 0, None) == EARG
    assert ur(p.ctypes.data, 4, 4, 3, org.ctypes.data, 0.0, 1.0, o.ctypes.data, 4, None, None, 0, None) == EARG
    for near, far in ((-1.0, 1.0), (0.0, -1.0), (2.0, 1.0), (float("nan"), 1.0)):
        assert ur(p.ctypes.data, 4, 4, 4, org.ctypes.data, near, far, o.ctypes.data, 4, None, None, 0, None) == EARG
    assert ur(p.ctypes.data, 4, 4, 4, org.ctypes.data, 0.0, 1.0, p[1:].ctypes.data, 4, None, None, 0, None) == EARG
    assert ur(p.ctypes.data, 4, 4, 4, org.ctypes.data, 0.0, 1.0, p.ctypes.data, 3, None, None, 0, None) == EARG


def test_no_device_only_after_validation(L):
    if not no_device(L):
        pytest.skip("a device is present: the gpu tests run these calls")
    d = np.zeros((8, 8, 3), np.float32)
    o, e, p = np.zeros((8, 8, 3)), np.zeros((8, 8)), np.zeros((8, 8, 3))
    c1, c2 = cam(), cam(center=(1, 0, 0), tsai=(0.1, 0, 0, 0, 0))
    assert tri(L, c2=c2) == ENODEVICE
    assert L.vwb200_stereo_model_points(d.ctypes.data, 8, 8, 8, C.byref(c1), C.byref(c2), 0.0, o.ctypes.data, 8, e.ctypes.data, 8, 0, None) == ENODEVICE
    assert L.vwb200_universe_radius(p.ctypes.data, 8, 8, 8, np.zeros(3).ctypes.data, 0.0, 1.0, p.ctypes.data, 8, None, None, 0, None) == ENODEVICE
    assert b"no CUDA device" in L.vwb200_last_error()
