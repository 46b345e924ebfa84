"""The C++ smoothing shim (include/vwb200/DisparitySmoothing.h): compiles against the VW stand-ins as C++14, keeps the
reference's signatures and its shallow `disparity_out = disparity_in`, and (on the GPU box) reproduces the oracle."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "build", "test_smoothing_shim")


def _build():
    from visionworkbench_b200 import build
    import oracle.smoothing
    build.build()
    oracle.smoothing.build()
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpp", "test_smoothing_shim.cpp")
    deps = [src] + [os.path.join(ROOT, "include", "vwb200", f) for f in ("DisparitySmoothing.h", "PyramidCorrelationView.h", "vw_standin.h")]
    deps += [os.path.join(ROOT, "visionworkbench_b200", "libvwb200.so"), os.path.join(ROOT, "oracle", "libvwsmoothing.so")]
    if not os.path.exists(EXE) or any(os.path.getmtime(d) > os.path.getmtime(EXE) for d in deps):
        subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), src, "-o", EXE,
                               "-L", os.path.join(ROOT, "visionworkbench_b200"), "-lvwb200",
                               "-L", os.path.join(ROOT, "oracle"), "-lvwsmoothing", "-lvworacle", "-lpthread",
                               "-Wl,-rpath," + os.path.join(ROOT, "visionworkbench_b200"), "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    return EXE


def test_smoothing_shim_compiles_as_cxx14_and_fails_loudly_without_a_device():
    exe = _build()
    import visionworkbench_b200 as v
    if v.device_count() > 0:
        pytest.skip("device present: covered by the gpu test")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 3, r.stdout + r.stderr
    assert "no CUDA device" in r.stdout


@pytest.mark.gpu
def test_smoothing_shim_matches_oracle():
    r = subprocess.run([_build()], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 texture, 0 texture-filter, 0 median mismatches" in r.stdout and "aliasing kept" in r.stdout, r.stdout
