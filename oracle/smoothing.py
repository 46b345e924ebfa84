"""ctypes binding of the disparity smoothing oracle (vw_smoothing_oracle.c -> libvwsmoothing.so; numpy in, numpy out).
Test infrastructure only, like the rest of oracle/: import it as `oracle.smoothing` from tests/ and tools/, never from the
product package.  The library links the main oracle (libvworacle.so) for derivative_filter's separable convolution."""
import ctypes as C
import os
import subprocess

import numpy as np

from . import binding

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libvwsmoothing.so")
_SRC = [os.path.join(_HERE, f) for f in ("vw_smoothing_oracle.c", "vw_smoothing_oracle.h", "vw_oracle.h", "smoothing.py")]
# the flags of oracle/Makefile: the reference's -O3 -msse4.1, no FMA contraction
_CFLAGS = ["-O3", "-std=c11", "-msse4.1", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter"]
_LIB = None


def build(force=False):
    """Compile libvwsmoothing.so with gcc (after the main oracle, which it links)."""
    main = binding.build()
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in _SRC + [main]):
        subprocess.check_call(["/usr/bin/gcc"] + _CFLAGS + ["-shared", "-o", _SO, os.path.join(_HERE, "vw_smoothing_oracle.c"),
                                                           "-L", _HERE, "-lvworacle", "-Wl,-rpath,$ORIGIN", "-lm"])
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
    return _LIB


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def destructive_median(values):
    """math::destructive_median (Math/Functors.h:393-398) of a sequence of doubles"""
    v = np.ascontiguousarray(values, np.float64).copy()
    f = lib().vwo_destructive_median
    f.restype = C.c_double
    f.argtypes = [C.c_void_p, C.c_int]
    return f(_p(v), len(v))


def _disp3(disparity):
    d = np.ascontiguousarray(disparity, np.float32).copy()
    assert d.ndim == 3 and d.shape[2] == 3
    return d


def disparity_median_filter(disparity, kernel_size):
    """disparity_median_filter (Stereo/Algorithms.cc:26-67) on a copy of disparity (float32 (h, w, 3) {dx, dy, valid}),
    in place and in raster order like the reference; returns the copy."""
    d = _disp3(disparity)
    f = lib().vwo_disparity_median_filter
    f.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
    rc = f(_p(d), d.shape[1], d.shape[0], d.shape[1], int(kernel_size))
    if rc:
        raise ValueError(rc)
    return d


def texture_measure(image, kernel_size=9, gradient_weight=0.5, stddev_weight=0.5):
    """texture_measure (Stereo/Algorithms.h:144-209) of a float image; returns float32 of the same shape"""
    a = _f32(image)
    out = np.empty_like(a)
    f = lib().vwo_texture_measure
    f.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_void_p]
    rc = f(_p(a), a.shape[1], a.shape[0], a.shape[1], int(kernel_size), float(gradient_weight), float(stddev_weight), _p(out))
    if rc:
        raise ValueError(rc)
    return out


def texture_preserving_disparity_filter(disparity, texture_image, texture_max=0.15, max_kernel_size=11):
    """texture_preserving_disparity_filter<float> (Stereo/Algorithms.h:213-281) on a copy of disparity, in place and in
    raster order like the reference; returns the copy."""
    d = _disp3(disparity)
    t = _f32(texture_image)
    assert t.shape == d.shape[:2]
    f = lib().vwo_texture_preserving_disparity_filter
    f.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_int]
    rc = f(_p(d), d.shape[1], d.shape[0], d.shape[1], _p(t), t.shape[1], float(texture_max), int(max_kernel_size))
    if rc:
        raise ValueError(rc)
    return d
