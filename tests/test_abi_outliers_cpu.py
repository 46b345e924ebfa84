"""vwb200_outlier_filter without a GPU: every invalid call returns VWB200_EARG (with the reference's message for zero half
kernels) before the library looks for a device, and a valid call returns VWB200_ENODEVICE when there is none.  Plus the
C++ shim (include/vwb200/DisparityOutliers.h): it compiles as C++14 against the VW stand-ins, and on a GPU machine it
reproduces the oracle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

EARG, ENODEVICE = -1, -6
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "build", "test_outliers_shim")


@pytest.fixture(scope="module")
def v():
    from visionworkbench_b200 import build
    build.build()
    import visionworkbench_b200 as v
    return v


def call(v, prm, ptype=1, w=8, h=6, pitch=8, opitch=8, same_buffer=False, null_in=False):
    buf = np.zeros((h, max(pitch, 1), 3), np.float32)
    out = buf if same_buffer else np.zeros((h, max(opitch, 1), 3), np.float32)
    return v.lib().vwb200_outlier_filter(None if prm is None else C.byref(prm), ptype, None if null_in else buf.ctypes.data, w, h, pitch,
                                         out.ctypes.data, opitch, 0, None)


def P(v, method=1, cleanup=0, hh=1, hv=1):
    return v.api.OutlierParams(method, cleanup, hh, hv, 3.0, 0.5, 2.0)


def test_invalid_calls_return_earg_before_the_device(v):
    bad = {
        "null params": lambda: call(v, None),
        "null input": lambda: call(v, P(v), null_in=True),
        "method -1": lambda: call(v, P(v, method=-1)),
        "method 3": lambda: call(v, P(v, method=3)),
        "cleanup 2": lambda: call(v, P(v, cleanup=2)),
        "pixel type 2": lambda: call(v, P(v), ptype=2),
        "pixel type -1": lambda: call(v, P(v), ptype=-1),
        "half_h 0": lambda: call(v, P(v, hh=0)),
        "half_v -1": lambda: call(v, P(v, method=2, hv=-1)),
        "negative width": lambda: call(v, P(v), w=-1),
        "pitch below width": lambda: call(v, P(v), pitch=7, opitch=8),
        "opitch below width": lambda: call(v, P(v), opitch=7),
        "in place": lambda: call(v, P(v), same_buffer=True),
    }
    for name, f in bad.items():
        assert f() == EARG, name
    call(v, P(v, method=1, hh=0))
    assert v.lib().vwb200_last_error() == b"RmOutliersUsingMeanFunc: half kernel sizes must be non-zero."
    for m in (0, 2):
        call(v, P(v, method=m, hv=0))
        assert v.lib().vwb200_last_error() == b"RmOutliersFunc: half kernel sizes must be non-zero."


def test_valid_calls_need_a_device(v):
    if v.device_count() > 0:
        pytest.skip("device present: the GPU tests cover valid calls")
    for method in (0, 1, 2):
        for cleanup in (0, 1):
            for ptype in (0, 1):
                assert call(v, P(v, method, cleanup, 2, 3), ptype=ptype) == ENODEVICE
    with pytest.raises(v.NoDeviceErr):
        v.rm_outliers_using_stddev(np.zeros((4, 5, 3), np.float32), 1, 1, 2.0, 0.5)


def test_python_refuses_other_dtypes_and_shapes(v):
    for bad in (np.zeros((4, 5, 3), np.float64), np.zeros((4, 5, 3), np.int64), np.zeros((4, 5, 2), np.float32), np.zeros((4, 5), np.int32)):
        with pytest.raises(v.ArgumentErr):
            v.rm_outliers_using_mean(bad, 1, 1, 2.0)


def _build_shim():
    from visionworkbench_b200 import build
    import oracle.outliers
    build.build()
    oracle.outliers.build()
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpp", "test_outliers_shim.cpp")
    deps = [src] + [os.path.join(ROOT, "include", "vwb200", f) for f in ("DisparityOutliers.h", "PyramidCorrelationView.h", "vw_standin.h")]
    deps += [os.path.join(ROOT, "visionworkbench_b200", "libvwb200.so"), os.path.join(ROOT, "oracle", "libvwoutliers.so")]
    if not os.path.exists(EXE) or any(os.path.getmtime(d) > os.path.getmtime(EXE) for d in deps):
        subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), src, "-o", EXE,
                               "-L", os.path.join(ROOT, "visionworkbench_b200"), "-lvwb200",
                               "-L", os.path.join(ROOT, "oracle"), "-lvwoutliers", "-lpthread",
                               "-Wl,-rpath," + os.path.join(ROOT, "visionworkbench_b200"), "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    return EXE


def test_outliers_shim_compiles_as_cxx14_and_fails_loudly_without_a_device():
    exe = _build_shim()
    import visionworkbench_b200 as v
    if v.device_count() > 0:
        pytest.skip("device present: covered by the gpu test")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 3, r.stdout + r.stderr
    assert "no CUDA device" in r.stdout


@pytest.mark.gpu
def test_outliers_shim_matches_oracle():
    r = subprocess.run([_build_shim()], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "outliers shim: 0 float, 0 int mismatches" in r.stdout, r.stdout
