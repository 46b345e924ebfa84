"""ctypes binding of the image-warp oracle (vw_warp_oracle.c -> libvwwarp.so; numpy in, numpy out).
Test infrastructure only, like the rest of oracle/: import it as `oracle.warp` from tests/ and tools/, never from the
product package."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libvwwarp.so")
_SRC = [os.path.join(_HERE, f) for f in ("vw_warp_oracle.c", "vw_warp_oracle.h", "warp.py")]
# the flags of oracle/Makefile: the reference's -O3 -msse4.1, no FMA contraction
_CFLAGS = ["-O3", "-std=c11", "-msse4.1", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter"]
_LIB = None

HOMOGRAPHY, DISPARITY = 0, 1
BILINEAR, BICUBIC, NEAREST = 0, 1, 2
ZERO, CONSTANT = 0, 1


def build(force=False):
    """Compile libvwwarp.so with gcc."""
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in _SRC):
        subprocess.check_call(["/usr/bin/gcc"] + _CFLAGS + ["-shared", "-o", _SO, os.path.join(_HERE, "vw_warp_oracle.c"), "-lm"])
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        P, I = C.c_void_p, C.c_int
        _LIB.vww_transform.argtypes = [I, I, I, P, P, I, I, P, I, I, I, I, P, I, I]
        _LIB.vww_transform.restype = None
    return _LIB


def transform(image, kind, interp, edge, window, matrix=None, disparity=None):
    """the TransformView pixels of window (x0, y0, ow, oh) as a float32 (oh, ow) array.  kind HOMOGRAPHY: `matrix` is the one
    reverse() applies (inverse(H)); kind DISPARITY: `disparity` is a float32 (rows, cols, 3) {dx, dy, valid} raster."""
    img = np.ascontiguousarray(image, np.float32)
    assert img.ndim == 2, img.shape
    x0, y0, ow, oh = (int(v) for v in window)
    m = np.ascontiguousarray(np.asarray(matrix if matrix is not None else np.eye(3), np.float64).reshape(9))
    if kind == DISPARITY:
        d = np.ascontiguousarray(disparity, np.float32)
        assert d.ndim == 3 and d.shape[2] == 3, d.shape
        dptr, dw, dh = d.ctypes.data, d.shape[1], d.shape[0]
    else:
        d, dptr, dw, dh = None, None, 0, 0
    out = np.zeros((oh, ow), np.float32)
    lib().vww_transform(int(kind), int(interp), int(edge), m.ctypes.data, img.ctypes.data, img.shape[1], img.shape[0], dptr, dw, dh,
                        x0, y0, out.ctypes.data, ow, oh)
    return out
