"""ctypes binding of the epipolar-rectification oracle (vw_epipolar_oracle.c -> libvwepipolar.so; numpy in, numpy out).
Test infrastructure only, like the rest of oracle/: import it as `oracle.epipolar` from tests/ and tools/, never from the
product package.  Cameras are the dicts of oracle.triangulate (camera(), pinhole()); images and interpolation / edge codes
those of oracle.warp, plus VALUE (ValueEdgeExtension, PixelMask<float> images only)."""
import ctypes as C
import os
import subprocess

import numpy as np

from .triangulate import OracleError, Pinhole, pinhole
from .warp import BILINEAR, ZERO

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libvwepipolar.so")
_SRC = [os.path.join(_HERE, f) for f in ("vw_epipolar_oracle.c", "vw_epipolar_oracle.h", "vw_triangulate_oracle.c", "vw_triangulate_oracle.h",
                                         "vw_warp_oracle.c", "vw_warp_oracle.h", "epipolar.py")]
# the flags of oracle/Makefile: the reference's -O3 -msse4.1, no FMA contraction
_CFLAGS = ["-O3", "-std=c11", "-msse4.1", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter"]
_LIB = None
VALUE = 2


def build(force=False):
    """Compile libvwepipolar.so with gcc (vw_epipolar_oracle.c includes the triangulation and warp oracles' sources)."""
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in _SRC):
        subprocess.check_call(["/usr/bin/gcc"] + _CFLAGS + ["-shared", "-o", _SO, os.path.join(_HERE, "vw_epipolar_oracle.c"), "-lm"])
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        P, I, PH = C.c_void_p, C.c_int, C.POINTER(Pinhole)
        L.vwt_quaternion_round_trip.argtypes = [P, P, P]
        L.vwt_epipolar.argtypes = [PH, PH, PH, PH]
        L.vwt_camera_matrix.argtypes = [PH, P]
        L.vwt_point_to_pixel.argtypes = [PH, P, P]
        L.vwt_camera_transform_point.argtypes = [PH, PH, I, P, P]
        L.vwt_camera_reverse_window.argtypes = [PH, PH, I, I, I, I, P, C.POINTER(C.c_longlong)]
        L.vwt_transformed_bbox_fast.argtypes = [PH, PH, P, P, C.POINTER(C.c_longlong)]
        L.vwt_resize_epipolar.argtypes = [PH, PH, PH, PH, P, P, P, P, C.POINTER(C.c_longlong), C.POINTER(I)]
        L.vww_sample.argtypes = [I, I, P, I, I, P, C.c_longlong, P]
        L.vww_sample.restype = None
        L.vww_sample_masked.argtypes = [I, P, P, I, I, P, C.c_longlong, P]
        L.vww_sample_masked.restype = None
        _LIB = L
    return _LIB


class PointToPixelErr(OracleError):
    """point_to_pixel's check failed; `where` is the first failing pixel / perimeter index (and camera) where known"""

    def __init__(self, where=None):
        super().__init__(-4)
        self.where = where

    def __str__(self):
        return "PinholeModel: Projection into pinhole camera is inaccurate."


def _ok(rc, where=None):
    if rc == -4:
        raise PointToPixelErr(where)
    if rc == -5:
        raise OracleError("the camera transform's cameras are at different centers")
    if rc != 0:
        raise OracleError(rc)


def _buf(a, dtype):
    return np.ascontiguousarray(a, dtype)


def from_pinhole(p):
    """the camera dict of a Pinhole struct"""
    return dict(center=tuple(p.center), rotation=np.array(p.rotation[:]).reshape(3, 3), fu=p.fu, fv=p.fv, cu=p.cu, cv=p.cv,
                u=tuple(p.u_direction), v=tuple(p.v_direction), w=tuple(p.w_direction), pixel_pitch=p.pixel_pitch,
                tsai=tuple(p.lens_params) if p.lens == 1 else None)


def quaternion_round_trip(R):
    """(camera_pose().rotation_matrix(), branch 0 ww / 1 xx / 2 yy / 3 zz, quaternion w, x, y, z)"""
    R = _buf(R, np.float64).reshape(9)
    out, q = np.zeros(9), np.zeros(4)
    b = lib().vwt_quaternion_round_trip(R.ctypes.data, out.ctypes.data, q.ctypes.data)
    return out.reshape(3, 3), b, q


def epipolar(cam0, cam1):
    a, b = Pinhole(), Pinhole()
    _ok(lib().vwt_epipolar(C.byref(pinhole(cam0)), C.byref(pinhole(cam1)), C.byref(a), C.byref(b)))
    return from_pinhole(a), from_pinhole(b)


def camera_matrix(cam):
    out = np.zeros(12)
    _ok(lib().vwt_camera_matrix(C.byref(pinhole(cam)), out.ctypes.data))
    return out.reshape(3, 4)


def point_to_pixel(cam, point):
    """point_to_pixel(point); PointToPixelErr (with the pixel computed in .where) when the check fails"""
    pt = _buf(point, np.float64)
    out = np.zeros(2)
    rc = lib().vwt_point_to_pixel(C.byref(pinhole(cam)), pt.ctypes.data, out.ctypes.data)
    _ok(rc, out)
    return out


def camera_forward(src, dst, p):
    pp, out = _buf(p, np.float64), np.zeros(2)
    _ok(lib().vwt_camera_transform_point(C.byref(pinhole(src)), C.byref(pinhole(dst)), 0, pp.ctypes.data, out.ctypes.data))
    return out


def camera_reverse(src, dst, p):
    pp, out = _buf(p, np.float64), np.zeros(2)
    _ok(lib().vwt_camera_transform_point(C.byref(pinhole(src)), C.byref(pinhole(dst)), 1, pp.ctypes.data, out.ctypes.data))
    return out


def camera_reverse_window(src, dst, window):
    """reverse() of every pixel of window (x0, y0, ow, oh): ((oh, ow, 2) coordinates, first failing (x, y) or None)"""
    x0, y0, ow, oh = (int(v) for v in window)
    out = np.zeros((oh, ow, 2))
    ff = C.c_longlong()
    rc = lib().vwt_camera_reverse_window(C.byref(pinhole(src)), C.byref(pinhole(dst)), x0, y0, ow, oh, out.ctypes.data, C.byref(ff))
    if rc not in (0, -4):
        _ok(rc)
    return out, (None if rc == 0 else (x0 + ff.value % ow, y0 + ff.value // ow))


def transformed_bbox_fast(src, dst, roi):
    """compute_transformed_bbox_fast(roi (x0, y0, x1, y1), CameraTransform(src, dst)): float32 [min x, min y, max x, max y];
    PointToPixelErr with the failing perimeter index"""
    r = np.ascontiguousarray(roi, np.int32)
    bb = np.zeros(4, np.float32)
    k = C.c_longlong()
    rc = lib().vwt_transformed_bbox_fast(C.byref(pinhole(src)), C.byref(pinhole(dst)), r.ctypes.data, bb.ctypes.data, C.byref(k))
    _ok(rc, k.value)
    return bb


def resize_epipolar(cam1, cam2, epi1, epi2, roi1, roi2):
    """resize_epipolar_cameras_to_fit: (epi1, epi2, size1, size2); PointToPixelErr with (camera, perimeter index)"""
    e1, e2 = pinhole(epi1), pinhole(epi2)
    r1, r2 = np.ascontiguousarray(roi1, np.int32), np.ascontiguousarray(roi2, np.int32)
    s1, s2 = np.zeros(2, np.int32), np.zeros(2, np.int32)
    k, cam = C.c_longlong(), C.c_int()
    rc = lib().vwt_resize_epipolar(C.byref(pinhole(cam1)), C.byref(pinhole(cam2)), C.byref(e1), C.byref(e2), r1.ctypes.data, r2.ctypes.data,
                                   s1.ctypes.data, s2.ctypes.data, C.byref(k), C.byref(cam))
    _ok(rc, (cam.value, k.value))
    return from_pinhole(e1), from_pinhole(e2), tuple(int(v) for v in s1), tuple(int(v) for v in s2)


def sample(image, interp, edge, coords, edge_value=(0.0, 0.0)):
    """the interpolation stage at reversed coordinates coords (..., 2): a float32 (rows, cols) image gives float32 (...), a
    PixelMask<float> (rows, cols, 2) image (bilinear only) {value, valid} float32 (..., 2)"""
    img = np.ascontiguousarray(image, np.float32)
    c = np.ascontiguousarray(coords, np.float64)
    n = c.size // 2
    if img.ndim == 2:
        out = np.zeros(c.shape[:-1], np.float32)
        lib().vww_sample(int(interp), int(edge), img.ctypes.data, img.shape[1], img.shape[0], c.ctypes.data, n, out.ctypes.data)
    else:
        assert img.ndim == 3 and img.shape[2] == 2 and interp == BILINEAR, (img.shape, interp)
        ev = np.ascontiguousarray(edge_value, np.float32)
        out = np.zeros(c.shape, np.float32)
        lib().vww_sample_masked(int(edge), ev.ctypes.data, img.ctypes.data, img.shape[1], img.shape[0], c.ctypes.data, n, out.ctypes.data)
    return out


def camera_transform(image, src, dst, window, interp=BILINEAR, edge=ZERO, edge_value=(0.0, 0.0)):
    """camera_transform(image, src, dst) over window (x0, y0, ow, oh): the TransformView of CameraTransform(src, dst) (camera
    dicts of oracle.triangulate), its reverse() restated in vw_triangulate_oracle.c.  PointToPixelErr (.where: the first
    failing (x, y) in row-major order) where the reference throws."""
    coords, fail = camera_reverse_window(src, dst, window)
    if fail is not None:
        raise PointToPixelErr(fail)
    return sample(image, interp, edge, coords, edge_value)
