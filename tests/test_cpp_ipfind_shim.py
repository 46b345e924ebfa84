"""The C++ shim include/vwb200/InterestPointDetector.h: it compiles as C++14 against the VW stand-ins and runs
detect_interest_points (IntegralAutoGainDetector), remove_ip_near_nodata and describe_interest_points
(SGradDescriptorGenerator) with the reference's argument lists; without a device it fails loudly, and on a GPU machine it
reproduces the oracle bit for bit."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "build", "test_ipfind_shim")


def _build_shim():
    from visionworkbench_b200 import build
    import oracle.ipfind
    build.build()
    oracle.ipfind.build()
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpp", "test_ipfind_shim.cpp")
    deps = [src] + [os.path.join(ROOT, "include", "vwb200", f) for f in ("InterestPointDetector.h", "PyramidCorrelationView.h", "vw_standin.h")]
    deps += [os.path.join(ROOT, "include", "vwb200.h"), os.path.join(ROOT, "visionworkbench_b200", "libvwb200.so"),
             os.path.join(ROOT, "oracle", "libvwipfind.so")]
    if not os.path.exists(EXE) or any(os.path.getmtime(d) > os.path.getmtime(EXE) for d in deps):
        subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), src, "-o", EXE,
                               "-L", os.path.join(ROOT, "visionworkbench_b200"), "-lvwb200",
                               "-L", os.path.join(ROOT, "oracle"), "-lvwipfind", "-lpthread",
                               "-Wl,-rpath," + os.path.join(ROOT, "visionworkbench_b200"), "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    return EXE


def test_ipfind_shim_compiles_as_cxx14_and_fails_loudly_without_a_device():
    exe = _build_shim()
    import visionworkbench_b200 as v
    if v.device_count() > 0:
        pytest.skip("device present: covered by the gpu test")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 3, r.stdout + r.stderr
    assert "no CUDA device" in r.stdout


@pytest.mark.gpu
def test_ipfind_shim_matches_oracle():
    r = subprocess.run([_build_shim()], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ipfind shim: 0 mismatches" in r.stdout, r.stdout
