"""ctypes binding of the interest point matching oracle (vw_ipmatch_oracle.c -> libvwipmatch.so; numpy in, numpy out).
Test infrastructure only, like the rest of oracle/: import it as `oracle.ipmatch` from tests/ and tools/, never from the
product package."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libvwipmatch.so")
_SRC = [os.path.join(_HERE, f) for f in ("vw_ipmatch_oracle.c", "vw_ipmatch_oracle.h", "ipmatch.py")]
# the flags of oracle/Makefile: the reference's -O3 -msse4.1, no FMA contraction
_CFLAGS = ["-O3", "-std=c11", "-msse4.1", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter"]
_LIB = None
L2, HAMMING = 0, 1


class OracleError(RuntimeError):
    def __init__(self, code, msg=""):
        super().__init__(f"{msg} (oracle code {code})" if msg else f"oracle code {code}")
        self.code = code


class BadByteValue(OracleError):
    """a Hamming descriptor value outside (-1, 256) or NaN: `where` = (list 0 / 1, row, k)"""

    def __init__(self, where):
        super().__init__(-1, f"Hamming value outside (-1, 256) at desc{where[0] + 1}[{where[1]}][{where[2]}]")
        self.where = where


def build(force=False):
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in _SRC):
        subprocess.check_call(["/usr/bin/gcc"] + _CFLAGS + ["-shared", "-o", _SO, os.path.join(_HERE, "vw_ipmatch_oracle.c"), "-lm"])
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        P, I = C.c_void_p, C.c_int
        L.vwm_l2.argtypes = [P, P, I]
        L.vwm_l2.restype = C.c_float
        L.vwm_hamming.argtypes = [P, P, I]
        L.vwm_hamming.restype = C.c_float
        L.vwm_match.argtypes = [I, P, P, I, P, P, I, I, C.c_double, P, P, P, C.POINTER(I), C.POINTER(C.c_longlong)]
        L.vwm_remove_duplicates.argtypes = [P, P, I, P, C.POINTER(I)]
        _LIB = L
    return _LIB


def l2(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return np.float32(lib().vwm_l2(a.ctypes.data, b.ctypes.data, len(a)))


def hamming(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return np.float32(lib().vwm_hamming(a.ctypes.data, b.ctypes.data, len(a)))


def match(desc1, pol1, desc2, pol2, threshold=0.5, metric=L2):
    """InterestPointMatcherSimple: (int32 index per ip1, float64 first_pick, float64 second_pick).  BadByteValue for a Hamming
    value outside (-1, 256); OracleError(-4) for 8 dim > 2^24.  Empty lists give index -1 and picks 1e100."""
    d1, d2 = np.ascontiguousarray(desc1, np.float32), np.ascontiguousarray(desc2, np.float32)
    n1, n2 = len(d1), len(d2)
    dim = d1.shape[1] if d1.ndim == 2 and n1 else (d2.shape[1] if d2.ndim == 2 else 0)
    p1, p2 = np.ascontiguousarray(np.asarray(pol1).astype(bool), np.uint8), np.ascontiguousarray(np.asarray(pol2).astype(bool), np.uint8)
    idx, first, second = np.full(n1, -1, np.int32), np.full(n1, 1e100), np.full(n1, 1e100)
    bl, be = C.c_int(), C.c_longlong()
    rc = lib().vwm_match(int(metric), d1.ctypes.data, p1.ctypes.data, n1, d2.ctypes.data, p2.ctypes.data, n2, dim, float(threshold),
                         idx.ctypes.data, first.ctypes.data, second.ctypes.data, C.byref(bl), C.byref(be))
    if rc == -1:
        raise BadByteValue((bl.value, be.value // dim, be.value % dim))
    if rc != 0:
        raise OracleError(rc)
    return idx, first, second


def remove_duplicates(xy1, xy2):
    a, b = np.ascontiguousarray(xy1, np.float32).reshape(-1, 2), np.ascontiguousarray(xy2, np.float32).reshape(-1, 2)
    keep = np.zeros(len(a), np.int32)
    k = C.c_int()
    if lib().vwm_remove_duplicates(a.ctypes.data, b.ctypes.data, len(a), keep.ctypes.data, C.byref(k)) != 0:
        raise OracleError(-1, "NaN coordinate")
    return keep[:k.value].copy()
