"""The CAHV / CAHVOR overloads of the C++ shim (include/vwb200/CameraTransform.h, StereoView.h): they compile as C++14 against
the VW stand-ins and call linearize_camera, epipolar, camera_transform, linearize_camera_transform,
epipolar_transformed_cahv_images, stereo_triangulate and StereoModel with the reference's argument lists; the host-only calls
match the oracle without a device, the device calls fail loudly without one, and on a GPU machine every call reproduces the
oracle."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "build", "test_cahv_shim")


def _build_shim():
    from visionworkbench_b200 import build
    import oracle.cahv
    build.build()
    oracle.cahv.build()
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpp", "test_cahv_shim.cpp")
    deps = [src] + [os.path.join(ROOT, "include", "vwb200", f) for f in ("CameraTransform.h", "ImageTransform.h", "StereoView.h",
                                                                         "DisparityResampling.h", "PyramidCorrelationView.h", "vw_standin.h")]
    deps += [os.path.join(ROOT, "include", "vwb200.h"), os.path.join(ROOT, "visionworkbench_b200", "libvwb200.so"),
             os.path.join(ROOT, "oracle", "libvwcahv.so")]
    if not os.path.exists(EXE) or any(os.path.getmtime(d) > os.path.getmtime(EXE) for d in deps):
        subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), src, "-o", EXE,
                               "-L", os.path.join(ROOT, "visionworkbench_b200"), "-lvwb200",
                               "-L", os.path.join(ROOT, "oracle"), "-lvwcahv", "-lpthread",
                               "-Wl,-rpath," + os.path.join(ROOT, "visionworkbench_b200"), "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    return EXE


def test_cahv_shim_compiles_as_cxx14_and_fails_loudly_without_a_device():
    exe = _build_shim()
    import visionworkbench_b200 as v
    if v.device_count() > 0:
        pytest.skip("device present: covered by the gpu test")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 3, r.stdout + r.stderr
    assert "no CUDA device" in r.stdout


@pytest.mark.gpu
def test_cahv_shim_matches_oracle():
    r = subprocess.run([_build_shim()], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "cahv shim: 0 mismatches" in r.stdout, r.stdout
