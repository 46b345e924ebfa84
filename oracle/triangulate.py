"""ctypes binding of the triangulation oracle (vw_triangulate_oracle.c -> libvwtriangulate.so; numpy in, numpy out).
Test infrastructure only, like the rest of oracle/: import it as `oracle.triangulate` from tests/ and tools/, never from the
product package.  A camera is a dict of the PinholeModel constructor parameters: center, rotation (3 x 3), fu, fv, cu, cv,
and optionally u, v, w (the unit axes by default), pixel_pitch (1) and tsai (k1, k2, p1, p2, k3; None for the NULL lens)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libvwtriangulate.so")
_SRC = [os.path.join(_HERE, f) for f in ("vw_triangulate_oracle.c", "vw_triangulate_oracle.h", "triangulate.py")]
# the flags of oracle/Makefile: the reference's -O3 -msse4.1, no FMA contraction
_CFLAGS = ["-O3", "-std=c11", "-msse4.1", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter"]
_LIB = None
DBL_MAX = float(np.finfo(np.float64).max)


class Pinhole(C.Structure):
    """vwt_pinhole / vwb200_pinhole"""
    _fields_ = [("center", C.c_double * 3), ("rotation", C.c_double * 9), ("fu", C.c_double), ("fv", C.c_double), ("cu", C.c_double),
                ("cv", C.c_double), ("u_direction", C.c_double * 3), ("v_direction", C.c_double * 3), ("w_direction", C.c_double * 3),
                ("pixel_pitch", C.c_double), ("lens", C.c_int), ("num_lens_params", C.c_int), ("lens_params", C.c_double * 5)]


def camera(center=(0, 0, 0), rotation=None, fu=1.0, fv=1.0, cu=0.0, cv=0.0, u=(1, 0, 0), v=(0, 1, 0), w=(0, 0, 1), pixel_pitch=1.0, tsai=None):
    return dict(center=center, rotation=np.eye(3) if rotation is None else rotation, fu=fu, fv=fv, cu=cu, cv=cv, u=u, v=v, w=w,
                pixel_pitch=pixel_pitch, tsai=tsai)


def pinhole(cam):
    """the Pinhole struct of a camera dict"""
    p = Pinhole()
    p.center[:] = [float(x) for x in cam["center"]]
    p.rotation[:] = [float(x) for x in np.asarray(cam["rotation"], np.float64).reshape(9)]
    p.fu, p.fv, p.cu, p.cv = (float(cam[k]) for k in ("fu", "fv", "cu", "cv"))
    p.u_direction[:] = [float(x) for x in cam.get("u", (1, 0, 0))]
    p.v_direction[:] = [float(x) for x in cam.get("v", (0, 1, 0))]
    p.w_direction[:] = [float(x) for x in cam.get("w", (0, 0, 1))]
    p.pixel_pitch = float(cam.get("pixel_pitch", 1.0))
    t = cam.get("tsai")
    p.lens, p.num_lens_params = (0, 0) if t is None else (1, 5)
    if t is not None:
        p.lens_params[:] = [float(x) for x in t]
    return p


def build(force=False):
    """Compile libvwtriangulate.so with gcc."""
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in _SRC):
        subprocess.check_call(["/usr/bin/gcc"] + _CFLAGS + ["-shared", "-o", _SO, os.path.join(_HERE, "vw_triangulate_oracle.c"), "-lm"])
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        P, I, D, PH = C.c_void_p, C.c_int, C.c_double, C.POINTER(Pinhole)
        L.vwt_camera_inverse.argtypes = [PH, P]
        L.vwt_inverse3.argtypes = [P, P]
        L.vwt_tsai_undistort.argtypes = [PH, P, P, C.POINTER(I), C.POINTER(I)]
        L.vwt_pixel_to_vector.argtypes = [PH, P, P]
        L.vwt_triangulate.argtypes = [PH, PH, D, P, P, P, P]
        L.vwt_stereo_triangulate.argtypes = [I, P, I, I, I, I, I, I, PH, PH, D, P]
        L.vwt_stereo_model.argtypes = [P, I, I, PH, PH, D, P, P, P]
        L.vwt_universe_radius.argtypes = [P, I, I, P, D, D, P, P]
        _LIB = L
    return _LIB


class OracleError(ValueError):
    def __init__(self, rc):
        super().__init__({-1: "bad argument", -2: "Matrix is singular in inverse()", -3: "u, v, w are not orthonormal"}.get(rc, rc))
        self.rc = rc


def _ok(rc):
    if rc != 0:
        raise OracleError(rc)


def _buf(a, dtype):
    return np.ascontiguousarray(a, dtype)


def inverse3(m):
    out = np.zeros(9)
    m = _buf(m, np.float64).reshape(9)
    _ok(lib().vwt_inverse3(m.ctypes.data, out.ctypes.data))
    return out.reshape(3, 3)


def camera_inverse(cam):
    out = np.zeros(9)
    _ok(lib().vwt_camera_inverse(C.byref(pinhole(cam)), out.ctypes.data))
    return out.reshape(3, 3)


def tsai_undistort(cam, p):
    """(undistorted point, exit code, iterations): exit 0 converged, 1 bad determinant, 2 NaN |F|, 3 out of iterations,
    4 fu or fv < 1e-300"""
    p = _buf(p, np.float64)
    out = np.zeros(2)
    ex, it = C.c_int(), C.c_int()
    _ok(lib().vwt_tsai_undistort(C.byref(pinhole(cam)), p.ctypes.data, out.ctypes.data, C.byref(ex), C.byref(it)))
    return out, ex.value, it.value


def pixel_to_vector(cam, pix):
    pix = _buf(pix, np.float64)
    out = np.zeros(3)
    _ok(lib().vwt_pixel_to_vector(C.byref(pinhole(cam)), pix.ctypes.data, out.ctypes.data))
    return out


def triangulate(cam1, cam2, pix1, pix2, angle_tol=0.0):
    """StereoModel(cam1, cam2, angle_tol)(pix1, pix2, errorVec): (point, errorVec)"""
    a, b = _buf(pix1, np.float64), _buf(pix2, np.float64)
    xyz, err = np.zeros(3), np.zeros(3)
    _ok(lib().vwt_triangulate(C.byref(pinhole(cam1)), C.byref(pinhole(cam2)), float(angle_tol), a.ctypes.data, b.ctypes.data,
                              xyz.ctypes.data, err.ctypes.data))
    return xyz, err


def stereo_triangulate(disparity, cam1, cam2, window=None, angle_tol=0.0):
    """stereo_triangulate(disparity, cam1, cam2) over window (x0, y0, ow, oh) (None: the whole image): (oh, ow, 3) float64"""
    d = np.ascontiguousarray(disparity)
    assert d.ndim == 3 and d.shape[2] == 3 and d.dtype in (np.int32, np.float32), (d.shape, d.dtype)
    h, w = d.shape[:2]
    x0, y0, ow, oh = (0, 0, w, h) if window is None else (int(v) for v in window)
    out = np.zeros((oh, ow, 3))
    _ok(lib().vwt_stereo_triangulate(0 if d.dtype == np.int32 else 1, d.ctypes.data, w, h, x0, y0, ow, oh, C.byref(pinhole(cam1)),
                                     C.byref(pinhole(cam2)), float(angle_tol), out.ctypes.data))
    return out


def stereo_model(disparity, cam1, cam2, angle_tol=0.0):
    """StereoModel(cam1, cam2, angle_tol)(disparity, error) of a float32 (rows, cols, 3) disparity: (xyz, error, stats) with
    stats = dict(points, divergent, max_error, error_sum) (the error sum in raster order)"""
    d = _buf(disparity, np.float32)
    h, w = d.shape[:2]
    xyz, err, st = np.zeros((h, w, 3)), np.zeros((h, w)), np.zeros(4)
    _ok(lib().vwt_stereo_model(d.ctypes.data, w, h, C.byref(pinhole(cam1)), C.byref(pinhole(cam2)), float(angle_tol), xyz.ctypes.data,
                               err.ctypes.data, st.ctypes.data))
    return xyz, err, dict(points=int(st[0]), divergent=int(st[1]), max_error=float(st[2]), error_sum=float(st[3]))


def universe_radius(points, origin, near=0.0, far=DBL_MAX):
    """UniverseRadiusFunc(origin, near, far) over a (rows, cols, 3) float64 point image: (points, rejected, total)"""
    p = _buf(points, np.float64)
    o = _buf(origin, np.float64)
    out = np.zeros_like(p)
    cnt = np.zeros(2, np.int64)
    _ok(lib().vwt_universe_radius(p.ctypes.data, p.shape[1], p.shape[0], o.ctypes.data, float(near), float(far), out.ctypes.data,
                                  cnt.ctypes.data))
    return out, int(cnt[0]), int(cnt[1])
