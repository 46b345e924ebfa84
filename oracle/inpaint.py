"""ctypes binding of the hole-filling oracle (vw_inpaint_oracle.c -> libvwinpaint.so; numpy in, numpy out).
Test infrastructure only, like the rest of oracle/: import it as `oracle.inpaint` from tests/ and tools/, never from the
product package."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libvwinpaint.so")
_SRC = [os.path.join(_HERE, f) for f in ("vw_inpaint_oracle.c", "vw_inpaint_oracle.h", "inpaint.py")]
# the flags of oracle/Makefile: the reference's -O3 -msse4.1, no FMA contraction
_CFLAGS = ["-O3", "-std=c11", "-msse4.1", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter"]
_LIB = None


def build(force=False):
    """Compile libvwinpaint.so with gcc."""
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in _SRC):
        subprocess.check_call(["/usr/bin/gcc"] + _CFLAGS + ["-shared", "-o", _SO, os.path.join(_HERE, "vw_inpaint_oracle.c"), "-lm"])
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        P, I = C.c_void_p, C.c_int
        _LIB.vwi_fill_holes_grass.argtypes = [I, P, I, I, I, I, I, I, I, P, P]
        _LIB.vwi_fill_holes_grass.restype = I
    return _LIB


def fill_holes_grass(disparity, hole_fill_len, window=None, stats=False):
    """fill_holes_grass(disparity, hole_fill_len) rasterised over window (x0, y0, ow, oh) (None: the whole image).
    disparity: an int32 or float32 (rows, cols, 3) {dx, dy, valid} array; returns a new (oh, ow, 3) array of its dtype, and
    with stats=True also (holes in the tile, holes filled, largest 10 * max_distance^2)."""
    d = np.ascontiguousarray(disparity)
    assert d.ndim == 3 and d.shape[2] == 3 and d.dtype in (np.int32, np.float32), (d.shape, d.dtype)
    h, w = d.shape[:2]
    x0, y0, ow, oh = (0, 0, w, h) if window is None else (int(v) for v in window)
    out = np.zeros((oh, ow, 3), d.dtype)
    st = np.zeros(3, np.int32)
    rc = lib().vwi_fill_holes_grass(0 if d.dtype == np.int32 else 1, d.ctypes.data, w, h, int(hole_fill_len), x0, y0, ow, oh,
                                    out.ctypes.data, st.ctypes.data)
    if rc != 0:
        raise ValueError(f"fill_holes_grass oracle: bad window {(x0, y0, ow, oh)} or len {hole_fill_len} for {w} x {h}")
    return (out, tuple(int(v) for v in st)) if stats else out
