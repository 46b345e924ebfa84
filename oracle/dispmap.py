"""ctypes binding of the disparity-map oracle (vw_dispmap_oracle.c -> libvwdispmap.so; numpy in, numpy out).
Test infrastructure only, like the rest of oracle/: import it as `oracle.dispmap` from tests/ and tools/, never from the
product package."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libvwdispmap.so")
_SRC = [os.path.join(_HERE, f) for f in ("vw_dispmap_oracle.c", "vw_dispmap_oracle.h", "dispmap.py")]
# the flags of oracle/Makefile: the reference's -O3 -msse4.1, no FMA contraction
_CFLAGS = ["-O3", "-std=c11", "-msse4.1", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter"]
_LIB = None

LAZY, EXPLICIT = 0, 1


def build(force=False):
    """Compile libvwdispmap.so with gcc."""
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in _SRC):
        subprocess.check_call(["/usr/bin/gcc"] + _CFLAGS + ["-shared", "-o", _SO, os.path.join(_HERE, "vw_dispmap_oracle.c"), "-lm"])
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        P, I = C.c_void_p, C.c_int
        _LIB.vwd_subsample.argtypes = [I, P, I, I, P]
        _LIB.vwd_upsample.argtypes = [I, P, I, I, P]
        _LIB.vwd_range.argtypes = [I, P, I, I, P]
        _LIB.vwd_range_mask.argtypes = [I, P, I, I, P, P, P]
        _LIB.vwd_transform.argtypes = [I, I, P, I, I, I, P, I, I, P]
    return _LIB


def _disp(d):
    d = np.ascontiguousarray(d)
    assert d.ndim == 3 and d.shape[2] == 3 and d.dtype in (np.int32, np.float32), (d.shape, d.dtype)
    return d, 0 if d.dtype == np.int32 else 1


def disparity_subsample(disparity):
    d, t = _disp(disparity)
    h, w = d.shape[:2]
    out = np.zeros((1 + (h - 1) // 2, 1 + (w - 1) // 2, 3), d.dtype)
    lib().vwd_subsample(t, d.ctypes.data, w, h, out.ctypes.data)
    return out


def disparity_upsample(disparity):
    d, t = _disp(disparity)
    h, w = d.shape[:2]
    out = np.zeros((2 * h, 2 * w, 3), d.dtype)
    lib().vwd_upsample(t, d.ctypes.data, w, h, out.ctypes.data)
    return out


def get_disparity_range(disparity):
    """(min dx, min dy, max dx, max dy) as a float32 array"""
    d, t = _disp(disparity)
    r = np.zeros(4, np.float32)
    lib().vwd_range(t, d.ctypes.data, d.shape[1], d.shape[0], r.ctypes.data)
    return r


def disparity_range_mask(disparity, min, max):
    d, t = _disp(disparity)
    mn, mx = np.asarray(min, d.dtype).reshape(2), np.asarray(max, d.dtype).reshape(2)
    out = np.zeros_like(d)
    lib().vwd_range_mask(t, d.ctypes.data, d.shape[1], d.shape[0], mn.ctypes.data, mx.ctypes.data, out.ctypes.data)
    return out


def transform_disparities(mode, matrix, disparity, do_round=False, origin=(0, 0)):
    """mode LAZY: `matrix` is the inverse homography the reference's reverse() applies; EXPLICIT: the homography itself,
    with the subregion's origin and optional rounding"""
    d, t = _disp(disparity)
    m = np.ascontiguousarray(np.asarray(matrix, np.float64).reshape(9))
    out = np.zeros_like(d)
    lib().vwd_transform(t, int(mode), m.ctypes.data, int(bool(do_round)), int(origin[0]), int(origin[1]), d.ctypes.data,
                        d.shape[1], d.shape[0], out.ctypes.data)
    return out
