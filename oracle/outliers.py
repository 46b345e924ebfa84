"""ctypes binding of the outlier-filter oracle (vw_outlier_oracle.c -> libvwoutliers.so; numpy in, numpy out).
Test infrastructure only, like the rest of oracle/: import it as `oracle.outliers` from tests/ and tools/, never from the
product package."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libvwoutliers.so")
_SRC = [os.path.join(_HERE, f) for f in ("vw_outlier_oracle.c", "vw_outlier_oracle.h", "outliers.py")]
# the flags of oracle/Makefile: the reference's -O3 -msse4.1, no FMA contraction
_CFLAGS = ["-O3", "-std=c11", "-msse4.1", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter"]
_LIB = None

THRESH, MEAN, STDDEV = 0, 1, 2


def build(force=False):
    """Compile libvwoutliers.so with gcc."""
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in _SRC):
        subprocess.check_call(["/usr/bin/gcc"] + _CFLAGS + ["-shared", "-o", _SO, os.path.join(_HERE, "vw_outlier_oracle.c"), "-lm"])
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.vwo_outlier_filter.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                            C.c_double, C.c_double, C.c_double, C.c_void_p]
    return _LIB


def outlier_filter(method, cleanup, disparity, half_h, half_v, pixel_threshold=0.0, rejection_threshold=0.0, max_mean_diff=0.0):
    """one of the six filters on an int32 or float32 (rows, cols, 3) {dx, dy, valid} array; returns a new array"""
    d = np.ascontiguousarray(disparity)
    assert d.ndim == 3 and d.shape[2] == 3 and d.dtype in (np.int32, np.float32), (d.shape, d.dtype)
    out = np.zeros_like(d)
    rc = lib().vwo_outlier_filter(int(method), int(bool(cleanup)), 0 if d.dtype == np.int32 else 1, d.ctypes.data, d.shape[1], d.shape[0],
                                  int(half_h), int(half_v), float(pixel_threshold), float(rejection_threshold), float(max_mean_diff),
                                  out.ctypes.data)
    if rc:
        raise ValueError(rc)
    return out


def rm_outliers_using_thresh(d, half_h_kernel, half_v_kernel, pixel_threshold, rejection_threshold):
    return outlier_filter(THRESH, 0, d, half_h_kernel, half_v_kernel, pixel_threshold, rejection_threshold)


def disparity_cleanup_using_thresh(d, h_half_kernel, v_half_kernel, pixel_threshold, rejection_threshold):
    return outlier_filter(THRESH, 1, d, h_half_kernel, v_half_kernel, pixel_threshold, rejection_threshold)


def rm_outliers_using_mean(d, half_h_kernel, half_v_kernel, max_mean_diff):
    return outlier_filter(MEAN, 0, d, half_h_kernel, half_v_kernel, max_mean_diff=max_mean_diff)


def disparity_cleanup_using_mean(d, h_half_kernel, v_half_kernel, max_mean_diff):
    return outlier_filter(MEAN, 1, d, h_half_kernel, v_half_kernel, max_mean_diff=max_mean_diff)


def rm_outliers_using_stddev(d, half_h_kernel, half_v_kernel, pixel_threshold, rejection_threshold):
    return outlier_filter(STDDEV, 0, d, half_h_kernel, half_v_kernel, pixel_threshold, rejection_threshold)


def disparity_cleanup_using_stddev(d, h_half_kernel, v_half_kernel, pixel_threshold, rejection_threshold):
    return outlier_filter(STDDEV, 1, d, h_half_kernel, v_half_kernel, pixel_threshold, rejection_threshold)
