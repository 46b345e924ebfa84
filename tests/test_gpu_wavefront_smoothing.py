"""The device's disparity smoothing against the oracle, bit for bit with -0.0 == +0.0: the CPU matrix of
test_oracle_smoothing.py (where the oracle is checked against the restatement of the reference), larger rasters where
many rows of the wavefront are in flight, host and device paths, a non-dense pitch, a non-default stream, and the texture
chain of tools/correlate.cc:234-247.

The module sorts after the ones that trace kernels with torch.profiler in the pytest process (test_gpu_value_domain.py
last): in a whole-suite run with it placed before them, those modules' profiler sessions recorded no kernel at all."""
import os
import subprocess
import sys

import numpy as np
import pytest

import smoothing_reference as S
from test_oracle_smoothing import INVALID, KERNELS, SHAPE, hand_disparity, HAND_MEDIAN, HAND_TEXTURE, median_case, same, \
    so, texture_case, texture_image  # noqa: F401  (so: the smoothing oracle fixture)

pytestmark = pytest.mark.gpu
SWEEP = "smooth_sweep_kernel"


@pytest.fixture(scope="module")
def vwb():
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "GPU tests need a CUDA device: the engine has no CPU path"
    return v


def median(vwb, d, k):
    out = d.copy()
    assert vwb.disparity_median_filter(out, k) is out
    return out


def texture_filter(vwb, d, t, tmax, maxk):
    out = d.copy()
    assert vwb.texture_preserving_disparity_filter(out, t, tmax, maxk) is out
    return out


@pytest.mark.parametrize("integer", [False, True])
@pytest.mark.parametrize("k", KERNELS)
@pytest.mark.parametrize("invalid", INVALID)
def test_median_matrix(vwb, so, invalid, k, integer):
    d = median_case(invalid, k, integer)
    assert same(median(vwb, d, k), so.disparity_median_filter(d, k))


@pytest.mark.parametrize("shape,k", [((5, 6), 7), ((1, 30), 3), ((30, 1), 3), ((7, 7), 7), ((8, 9), 8), ((40, 70), 31), ((64, 33), 24)])
def test_median_small_and_wide_windows(vwb, so, shape, k):
    d = S.random_disparity(7 + shape[0] * 31 + shape[1], shape, 0.2, integer=k > 20)
    assert same(median(vwb, d, k), so.disparity_median_filter(d, k))


def test_hand_case(vwb):
    d = hand_disparity()
    got = median(vwb, d, 3)
    assert np.array_equal(got[..., 0], HAND_MEDIAN) and np.array_equal(got[..., 1], HAND_MEDIAN / 2)
    got = texture_filter(vwb, d, np.zeros((5, 5), np.float32), 1.0, 3)
    assert np.array_equal(got[..., 0], HAND_TEXTURE)


@pytest.mark.parametrize("k", [1, 2, 3, 4, 5, 9, 15, 31])
@pytest.mark.parametrize("shape", [(17, 21), (1, 12), (12, 1), (3, 2), (45, 70)])
def test_texture_measure_matrix(vwb, so, shape, k):
    img = texture_image(k * 13 + shape[0], shape)
    for gw, sw in ((0.5, 0.5), (1.0, 0.0), (0.3, 2.5)):
        assert same(vwb.texture_measure(img, k, gw, sw), so.texture_measure(img, k, gw, sw)), (gw, sw)


@pytest.mark.parametrize("tmax,maxk", [(0.15, 11), (0.15, 13), (0.15, 12), (0.2, 3), (0.05, 7), (0.0, 11), (-1.0, 11), (0.15, 2),
                                       (0.15, 31)])
@pytest.mark.parametrize("invalid", INVALID)
def test_texture_filter_matrix(vwb, so, invalid, tmax, maxk):
    d, t = texture_case(200 + int(invalid * 10) + maxk, SHAPE, invalid)
    assert same(texture_filter(vwb, d, t, tmax, maxk), so.texture_preserving_disparity_filter(d, t, tmax, maxk))


# ---- many rows in flight ---------------------------------------------------------------------------------------------------
LARGE_MEDIAN = [((2048, 2048), 3), ((2048, 2048), 5), ((2048, 2048), 11), ((1024, 4096), 3), ((1024, 4096), 5), ((160, 1024), 31)]


@pytest.mark.parametrize("shape,k", LARGE_MEDIAN)
def test_median_large(vwb, so, shape, k):
    d = S.random_disparity(shape[0] + k, shape, 0.1, integer=k == 5)
    want = so.disparity_median_filter(d, k)
    assert same(median(vwb, d, k), want)


@pytest.mark.parametrize("shape", [(2048, 2048), (1024, 4096)])
def test_texture_filter_large(vwb, so, shape):
    d, t = texture_case(shape[1], shape, 0.1)
    assert same(texture_filter(vwb, d, t, 0.15, 13), so.texture_preserving_disparity_filter(d, t, 0.15, 13))


def test_texture_measure_large(vwb, so):
    img = texture_image(5, (1024, 2048))
    assert same(vwb.texture_measure(img, 15), so.texture_measure(img, 15))


# ---- host / device, pitch, stream ---------------------------------------------------------------------------------------
def test_device_path_pitch_and_stream(vwb, so):
    import torch
    d = S.random_disparity(11, (300, 257), 0.2)
    t = texture_case(12, (300, 257), 0.0)[1]
    img = texture_image(13, (300, 257))
    wide = np.zeros((300, 300, 3), np.float32)                        # a non-dense pitch on the host: a column slice
    wide[:, :257] = d
    view = wide[:, :257]
    vwb.disparity_median_filter(view, 5)
    want = so.disparity_median_filter(d, 5)
    assert same(view, want) and not wide[:, 257:].any()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        big = torch.zeros((300, 301, 3), dtype=torch.float32, device="cuda")
        dd = big[:, 3:260]                                            # non-dense pitch on the device
        dd.copy_(torch.from_numpy(d))
        assert vwb.disparity_median_filter(dd, 5) is dd
        tt = torch.from_numpy(t).cuda()
        d2 = torch.from_numpy(d).cuda()
        vwb.texture_preserving_disparity_filter(d2, tt, 0.15, 11)
        tm = vwb.texture_measure(torch.from_numpy(img).cuda(), 9)
    s.synchronize()
    assert same(dd.cpu().numpy(), want) and not big[:, :3].any() and not big[:, 260:].any()
    assert same(d2.cpu().numpy(), so.texture_preserving_disparity_filter(d, t, 0.15, 11))
    assert same(tm.cpu().numpy(), so.texture_measure(img, 9))
    tpad = np.zeros((300, 280), np.float32)
    tpad[:, :257] = t
    got = texture_filter(vwb, d, tpad[:, :257], 0.15, 11)             # a texture with a non-dense pitch
    assert same(got, so.texture_preserving_disparity_filter(d, t, 0.15, 11))


def test_texture_chain_of_correlate(vwb, so):
    """tools/correlate.cc:234-247: texture_measure of the left image with texture_smooth_range 15, then
    texture_preserving_disparity_filter of the disparity with 0.85 of the largest texture and max_kernel_size 13"""
    left = texture_image(21, (512, 640))
    left[100:300, 200:500] = 128.0                                    # a flat area: the texture filter smooths there
    d = S.random_disparity(22, (512, 640), 0.1)
    tex = vwb.texture_measure(left, 15)
    assert same(tex, so.texture_measure(left, 15))
    tmax = np.float32(0.85) * tex.max()
    got = texture_filter(vwb, d, tex, tmax, 13)
    want = so.texture_preserving_disparity_filter(d, tex, tmax, 13)
    assert same(got, want)
    assert (got != d).any(-1).sum() > 1000


# Traced in a process of its own, so that its profiler sessions neither depend on nor add to the ones of the rest of the suite.
TRACE_SCRIPT = """
import numpy as np, torch
import smoothing_reference as S
import visionworkbench_b200 as v
from kernel_trace import KernelTrace
from test_oracle_smoothing import texture_case


class SmoothingTrace(KernelTrace):
    def hot(self):
        return {n for n in self.raw if "smooth_sweep_kernel" in n or "texture_measure_kernel" in n}


torch.cuda.init()
d = torch.from_numpy(S.random_disparity(31, (256, 512), 0.1)).cuda()
d2, t = texture_case(32, (256, 512), 0.1)
d2, t = torch.from_numpy(d2).cuda(), torch.from_numpy(t).cuda()
calls = [("MedianOp", lambda: v.disparity_median_filter(d.clone(), 11)),
         ("TextureFilterOp", lambda: v.texture_preserving_disparity_filter(d2.clone(), t, 0.15, 13)),
         ("texture_measure_kernel", lambda: v.texture_measure(t, 9))]
for name, fn in calls:
    fn()
    tr = SmoothingTrace()
    tr.run(fn)
    print(name, "RAN" if any(name in n for n in tr.raw) else "MISSING", sorted(set(tr.raw)))
"""


def test_wavefront_kernel_ran(vwb):
    """each filter ran its own kernel: the median and the texture filter the wavefront sweep with their operation,
    texture_measure its tiled kernel (tests/kernel_trace.py, device tensors on the current stream)"""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here]), PYTHONNOUSERSITE="1")
    r = subprocess.run([sys.executable, "-c", TRACE_SCRIPT], cwd=here, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln for ln in r.stdout.splitlines() if ln.split(" ")[0] in ("MedianOp", "TextureFilterOp", "texture_measure_kernel")]
    assert len(lines) == 3 and all(" RAN " in ln for ln in lines), r.stdout
    assert any("smooth_sweep_kernel" in ln for ln in lines[:2]), r.stdout
