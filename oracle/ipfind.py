"""ctypes binding of the ipfind oracle (vw_ipfind_oracle.c -> libvwipfind.so; numpy in, numpy out).
Test infrastructure only, like the rest of oracle/: import it as `oracle.ipfind` from tests/ and tools/, never from the
product package.  Points are structured arrays of POINT (the InterestPoint fields the path reads or writes)."""
import ctypes as C
import math
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libvwipfind.so")
_SRC = [os.path.join(_HERE, f) for f in ("vw_ipfind_oracle.c", "vw_ipfind_oracle.h", "ipfind.py")]
# the flags of oracle/Makefile: the reference's -O3 -msse4.1, no FMA contraction
_CFLAGS = ["-O3", "-std=c11", "-msse4.1", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter"]
_LIB = None
POINT = np.dtype([("x", "<f4"), ("y", "<f4"), ("ix", "<i4"), ("iy", "<i4"), ("scale", "<f4"), ("interest", "<f4"),
                  ("orientation", "<f4")])
DESC = 180


class OracleError(RuntimeError):
    pass


def build(force=False):
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in _SRC):
        subprocess.check_call(["/usr/bin/gcc"] + _CFLAGS + ["-shared", "-o", _SO, os.path.join(_HERE, "vw_ipfind_oracle.c"), "-lm"])
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        P, I, LL = C.c_void_p, C.c_int, C.c_longlong
        L.vwf_normalize.argtypes = [P, I, I, I, C.c_double, P]
        L.vwf_gaussian_taps.argtypes = [P]
        L.vwf_gaussian_taps.restype = None
        L.vwf_detect.argtypes = [P, I, I, I, I, C.POINTER(C.c_void_p), C.POINTER(LL), P]
        L.vwf_remove_near_nodata.argtypes = [P, I, I, C.c_double, I, P, LL]
        L.vwf_remove_near_nodata.restype = LL
        L.vwf_describe.argtypes = [P, I, I, I, P, LL, P]
        L.vwf_integral.argtypes = [P, I, I, P]
        L.vwf_integral.restype = None
        L.vwf_box_filter.argtypes = [P, I, I, I, P, P, P, P, P, P]
        L.vwf_box_filter.restype = None
        L.vwf_free.argtypes = [P]
        L.vwf_free.restype = None
        _LIB = L
    return _LIB


def _img(a):
    a = np.ascontiguousarray(a, np.float32)
    if a.ndim != 2:
        raise ValueError("a 2-D image")
    return a


def integral(image):
    """IntegralImage: (rows + 1, cols + 1) float32"""
    a = _img(image)
    out = np.zeros((a.shape[0] + 1, a.shape[1] + 1), np.float32)
    lib().vwf_integral(a.ctypes.data, a.shape[1], a.shape[0], out.ctypes.data)
    return out


def box_filter(integral_image, boxes):
    """box_filter(integral, filter): boxes are (start x, start y, size x, size y, weight); (rows, cols) float32"""
    I = np.ascontiguousarray(integral_image, np.float32)
    h, w = I.shape[0] - 1, I.shape[1] - 1
    cols = [np.ascontiguousarray([b[k] for b in boxes], np.int32) for k in range(4)]
    wt = np.ascontiguousarray([b[4] for b in boxes], np.float32)
    out = np.zeros((h, w), np.float32)
    lib().vwf_box_filter(I.ctypes.data, w, h, len(boxes), cols[0].ctypes.data, cols[1].ctypes.data, cols[2].ctypes.data,
                         cols[3].ctypes.data, wt.ctypes.data, out.ctypes.data)
    return out


def normalize(image, nodata=None):
    a = _img(image)
    out = np.empty_like(a)
    if lib().vwf_normalize(a.ctypes.data, a.shape[1], a.shape[0], nodata is not None, 0.0 if nodata is None else float(nodata),
                           out.ctypes.data):
        raise OracleError("normalize: NaN / inf input or no valid pixel")
    return out


def gaussian_taps():
    k = np.zeros(9, np.float64)
    lib().vwf_gaussian_taps(k.ctypes.data)
    return k


def detect(image, ip_per_tile=250, tile_size=1024):
    """points and stats (tiles, raw extrema, kept after the thresholds, culled tiles)"""
    a = _img(image)
    p, n, st = C.c_void_p(), C.c_longlong(), np.zeros(5, np.int64)
    if lib().vwf_detect(a.ctypes.data, a.shape[1], a.shape[0], int(tile_size), int(ip_per_tile), C.byref(p), C.byref(n), st.ctypes.data):
        raise OracleError("detect failed")
    pts = np.zeros(n.value, POINT)
    if n.value:
        C.memmove(pts.ctypes.data, p.value, n.value * POINT.itemsize)
    lib().vwf_free(p)
    return pts, [int(v) for v in st[:4]]


def remove_near_nodata(raw, points, nodata=0.0, radius=1):
    a = _img(raw)
    pts = np.array(points, POINT)
    n = lib().vwf_remove_near_nodata(a.ctypes.data, a.shape[1], a.shape[0], float(nodata), int(radius), pts.ctypes.data, len(pts))
    return pts[:n].copy()


def describe(image, points, tile_size=1024):
    """(points in describe_interest_points' order with the crop round trip's x / y, (n, 180) float32 descriptors)"""
    a = _img(image)
    pts = np.array(points, POINT)
    desc = np.zeros((len(pts), DESC), np.float32)
    if lib().vwf_describe(a.ctypes.data, a.shape[1], a.shape[0], int(tile_size), pts.ctypes.data, len(pts), desc.ctypes.data):
        raise OracleError("describe: a point outside every tile")
    return pts, desc


def ip_per_tile_for(ip_per_image, w, h, tile_size=1024):
    """ipfind.cc:255-262 with the unclamped tile size"""
    num_tiles = w * h / float(tile_size * tile_size)
    return max(1, int(math.ceil(ip_per_image / num_tiles)))


def ipfind(image, ip_per_tile=250, ip_per_image=0, nodata=None, nodata_radius=1, tile_size=1024):
    """ipfind.cc:253-401 (iagd, sgrad): (points, descriptors)"""
    raw = _img(image)
    if ip_per_image > 0:
        ip_per_tile = ip_per_tile_for(ip_per_image, raw.shape[1], raw.shape[0], tile_size)
    img = normalize(raw, nodata)
    pts, _ = detect(img, ip_per_tile, tile_size)
    if len(pts) == 0:
        return pts, np.zeros((0, DESC), np.float32)
    if nodata_radius > 0:
        pts = remove_near_nodata(raw, pts, 0.0 if nodata is None else nodata, nodata_radius)
    return describe(img, pts, tile_size)
