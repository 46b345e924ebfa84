"""ctypes binding of the CAHV / CAHVOR camera oracle (vw_cahv_oracle.c -> libvwcahv.so; numpy in, numpy out).
Test infrastructure only, like the rest of oracle/: import it as `oracle.cahv` from tests/ and tools/, never from the product
package.  A camera is a dict {"model": 1 CAHV | 2 CAHVOR, "C", "A", "H", "V"[, "O", "R"]}; sampling is oracle.epipolar's."""
import ctypes as C
import os
import subprocess

import numpy as np

from .triangulate import Pinhole

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libvwcahv.so")
_SRC = [os.path.join(_HERE, f) for f in ("vw_cahv_oracle.c", "vw_cahv_oracle.h", "vw_epipolar_oracle.c", "vw_epipolar_oracle.h",
                                         "vw_triangulate_oracle.c", "vw_triangulate_oracle.h", "vw_warp_oracle.c", "vw_warp_oracle.h", "cahv.py")]
# the flags of oracle/Makefile: the reference's -O3 -msse4.1, no FMA contraction
_CFLAGS = ["-O3", "-std=c11", "-msse4.1", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter"]
_LIB = None
CAHV, CAHVOR = 1, 2


class Cahv(C.Structure):
    _fields_ = [("model", C.c_int)] + [(k, C.c_double * 3) for k in "CAHVOR"]


def build(force=False):
    """Compile libvwcahv.so with gcc (vw_cahv_oracle.c includes the epipolar, triangulation and warp oracles' sources)."""
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in _SRC):
        subprocess.check_call(["/usr/bin/gcc"] + _CFLAGS + ["-shared", "-o", _SO, os.path.join(_HERE, "vw_cahv_oracle.c"), "-lm"])
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        P, I, CH = C.c_void_p, C.c_int, C.POINTER(Cahv)
        L.vwc_pixel_to_vector.argtypes = [CH, P, P, C.POINTER(I), C.POINTER(I)]
        L.vwc_point_to_pixel.argtypes = [CH, P, P]
        L.vwc_epipolar.argtypes = [CH, CH, CH, CH]
        L.vwc_linearize.argtypes = [CH, P, P, CH]
        L.vwc_from_pinhole.argtypes = [C.POINTER(Pinhole), CH]
        L.vwc_camera_reverse_window.argtypes = [CH, CH, I, I, I, I, P]
        L.vwc_stereo_triangulate.argtypes = [I, P, I, I, I, I, I, I, CH, CH, C.c_double, P, C.POINTER(C.c_longlong)]
        L.vwc_stereo_model.argtypes = [P, I, I, CH, CH, C.c_double, P, P, P, C.POINTER(C.c_longlong)]
        _LIB = L
    return _LIB


def cam(C_, A, H, V, O=None, R=None):
    d = {"model": CAHV if O is None else CAHVOR, "C": C_, "A": A, "H": H, "V": V}
    if O is not None:
        d["O"], d["R"] = O, R
    return d


def to_struct(c):
    s = Cahv()
    s.model = c["model"]
    for k in "CAHVOR":
        if k in c:
            getattr(s, k)[:] = [float(x) for x in c[k]]
    return s


def from_struct(s):
    d = {"model": s.model}
    for k in ("CAHV" if s.model == CAHV else "CAHVOR"):
        d[k] = tuple(getattr(s, k)[:])
    return d


def _check(rc):
    if rc:
        raise ValueError(f"oracle returned {rc}")


def pixel_to_vector(c, pix):
    """(direction, exit code, Newton passes)"""
    out, code, it = np.zeros(3), C.c_int(0), C.c_int(0)
    p = np.asarray(pix, np.float64)
    _check(lib().vwc_pixel_to_vector(C.byref(to_struct(c)), p.ctypes.data, out.ctypes.data, C.byref(code), C.byref(it)))
    return out, code.value, it.value


def point_to_pixel(c, point):
    out, p = np.zeros(2), np.asarray(point, np.float64)
    _check(lib().vwc_point_to_pixel(C.byref(to_struct(c)), p.ctypes.data, out.ctypes.data))
    return out


def epipolar(c0, c1):
    a, b = Cahv(), Cahv()
    _check(lib().vwc_epipolar(C.byref(to_struct(c0)), C.byref(to_struct(c1)), C.byref(a), C.byref(b)))
    return from_struct(a), from_struct(b)


def linearize(c, in_size, out_size):
    o = Cahv()
    _check(lib().vwc_linearize(C.byref(to_struct(c)), (C.c_int * 2)(*in_size), (C.c_int * 2)(*out_size), C.byref(o)))
    return from_struct(o)


def from_pinhole(pin_struct):
    o = Cahv()
    _check(lib().vwc_from_pinhole(C.byref(pin_struct), C.byref(o)))
    return from_struct(o)


def reverse_window(src, dst, x0, y0, ow, oh):
    coords = np.zeros((oh, ow, 2))
    _check(lib().vwc_camera_reverse_window(C.byref(to_struct(src)), C.byref(to_struct(dst)), x0, y0, ow, oh, coords.ctypes.data))
    return coords


def camera_transform(image, src, dst, x0, y0, ow, oh, interp=0, edge=0, edge_value=(0.0, 0.0)):
    """camera_transform(image, src, dst) over the window: float32 (rows, cols) or PixelMask<float> (rows, cols, 2)"""
    from . import epipolar as oe
    coords = reverse_window(src, dst, x0, y0, ow, oh)
    img = np.ascontiguousarray(image, np.float32)
    h, w = img.shape[:2]
    n = ow * oh
    if img.ndim == 3:
        out = np.zeros((oh, ow, 2), np.float32)
        ev = np.asarray(edge_value, np.float32)
        oe.lib().vww_sample_masked(edge, ev.ctypes.data, img.ctypes.data, w, h, coords.ctypes.data, n, out.ctypes.data)
    else:
        out = np.zeros((oh, ow), np.float32)
        oe.lib().vww_sample(interp, edge, img.ctypes.data, w, h, coords.ctypes.data, n, out.ctypes.data)
    return out


def stereo_triangulate(disp, c1, c2, x0=0, y0=0, ow=None, oh=None, angle_tol=0.0):
    """form (a): (xyz (oh, ow, 3), Newton passes)"""
    d = np.ascontiguousarray(disp)
    h, w = d.shape[:2]
    ow = w - x0 if ow is None else ow
    oh = h - y0 if oh is None else oh
    xyz, it = np.zeros((oh, ow, 3)), C.c_longlong(0)
    _check(lib().vwc_stereo_triangulate(0 if d.dtype == np.int32 else 1, d.ctypes.data, w, h, x0, y0, ow, oh, C.byref(to_struct(c1)),
                                        C.byref(to_struct(c2)), float(angle_tol), xyz.ctypes.data, C.byref(it)))
    return xyz, it.value


def stereo_model(disp, c1, c2, angle_tol=0.0):
    """form (b): (xyz, error, stats [points, divergent, max error, error sum], Newton passes)"""
    d = np.ascontiguousarray(disp, np.float32)
    h, w = d.shape[:2]
    xyz, err, st, it = np.zeros((h, w, 3)), np.zeros((h, w)), np.zeros(4), C.c_longlong(0)
    _check(lib().vwc_stereo_model(d.ctypes.data, w, h, C.byref(to_struct(c1)), C.byref(to_struct(c2)), float(angle_tol), xyz.ctypes.data,
                                  err.ctypes.data, st.ctypes.data, C.byref(it)))
    return xyz, err, st, it.value
