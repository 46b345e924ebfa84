"""The device's neighbourhood outlier filters (vwb200_outlier_filter: rm_outliers_using_{thresh,mean,stddev} and
disparity_cleanup_using_* on int32 and float32 disparities) against the oracle, bit for bit (floats as raw bits): the CPU
matrix of test_oracle_outliers.py, where the oracle is checked against the restatement of the reference, its hand cases,
4096^2 rasters, host and device paths with padded pitches and two streams, the existing integer thresh entry points, a
view's float output, the window limits and the kernel each filter ran.

The module sorts after the ones that trace kernels with torch.profiler in the pytest process."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import outlier_reference as R
from test_oracle_outliers import HALVES, INVALID, METHODS, SMALL, TYPES, check_all, hand_float_tie, hand_quantile_index, \
    hand_stddev_floor, hand_truncated_row, matrix_case, ou, params, same, stddev_wide_cases  # noqa: F401  (ou: oracle fixture)

pytestmark = pytest.mark.gpu
EARG, ENOIMPL = -1, -4


@pytest.fixture(scope="module")
def vwb():
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "GPU tests need a CUDA device: the engine has no CPU path"
    return v


def engine(vwb, method, cleanup, d, hx, hy, pt=0.0, rt=0.0, mmd=0.0):
    return vwb.outlier_filter(method, cleanup, d, hx, hy, pt, rt, mmd)


def check_engine(vwb, ou, d, hx, hy, i):
    for method in METHODS:
        p = params(method, i)
        for cleanup in (False, True):
            got = engine(vwb, method, cleanup, d, hx, hy, **p)
            want = ou.outlier_filter(method, cleanup, d, hx, hy, p["pt"], p["rt"], p["mmd"])
            assert same(got, want), (method, cleanup, np.argwhere((got != want).any(-1))[:5])


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
@pytest.mark.parametrize("half", HALVES, ids=lambda h: f"{h[0]}x{h[1]}")
@pytest.mark.parametrize("invalid", INVALID)
def test_matrix(vwb, ou, invalid, half, dtype):
    i = HALVES.index(half) + INVALID.index(invalid)
    check_engine(vwb, ou, matrix_case(invalid, half, dtype), half[0], half[1], i)
    # a raster wider and taller than one tile of the kernel, with its partial tiles
    check_engine(vwb, ou, matrix_case(invalid, half, dtype, shape=(45, 77)), half[0], half[1], i)


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
@pytest.mark.parametrize("shape,half", SMALL)
def test_small_and_thin_images(vwb, ou, shape, half, dtype):
    d = R.random_disparity(31 + shape[0] * 10 + shape[1], shape, 0.2, dtype)
    check_engine(vwb, ou, d, half[0], half[1], shape[0] + shape[1])


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
def test_hand_cases(vwb, ou, dtype):
    for make, fn in ((hand_truncated_row, vwb.rm_outliers_using_mean), (hand_quantile_index, vwb.rm_outliers_using_mean)):
        d, (hx, hy), mmd = make(dtype)
        got = fn(d, hx, hy, mmd)
        assert same(got, ou.rm_outliers_using_mean(d, hx, hy, mmd)) and got[d.shape[0] // 2, d.shape[1] // 2, 2] == 1
    if dtype == np.float32:
        d, (hx, hy), mmd = hand_float_tie()
        got = vwb.rm_outliers_using_mean(d, hx, hy, mmd)
        assert same(got, ou.rm_outliers_using_mean(d, hx, hy, mmd)) and got[1, 1, 2] == 0
    d = hand_stddev_floor(dtype)
    for pt, rt, kept in ((2.0, 4.0, 1), (1.99, 4.0, 0), (2.0, 0.0, 0)):
        got = vwb.rm_outliers_using_stddev(d, 1, 1, pt, rt)
        assert same(got, ou.rm_outliers_using_stddev(d, 1, 1, pt, rt)) and got[1, 1, 2] == kept
    d = R.random_disparity(5, (6, 7), 0.0, dtype)
    d[2, 3] = (7, -3, 0)
    for method in METHODS:
        for cleanup in (False, True):
            got = engine(vwb, method, cleanup, d, 1, 1, 1e9, 0.0, 1e9)
            assert same(got, d)


@pytest.mark.parametrize("case", range(3))
def test_stddev_wide_window(vwb, ou, case):
    d, (hx, hy), _ = stddev_wide_cases()[case]
    for cleanup in (False, True):
        for pt, rt in ((1.0, 0.5), (2.0, 0.1)):
            assert same(engine(vwb, R.STDDEV, cleanup, d, hx, hy, pt, rt), ou.outlier_filter(R.STDDEV, cleanup, d, hx, hy, pt, rt))


def realistic(seed, n, dtype):
    """a smooth disparity field with speckle (isolated wild values) and holes (invalid blobs)"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:n, 0:n].astype(np.float32)
    dx = 20 * np.sin(xx / 300) + 0.004 * yy + 0.3 * rng.standard_normal((n, n), np.float32)
    dy = 2 * np.cos(yy / 500) + 0.2 * rng.standard_normal((n, n), np.float32)
    speck = rng.random((n, n)) < 0.02
    dx[speck] += rng.uniform(-60, 60, int(speck.sum())).astype(np.float32)
    v = np.ones((n, n), np.float32)
    for _ in range(300):
        cy, cx, r = rng.integers(0, n), rng.integers(0, n), rng.integers(2, 25)
        v[max(cy - r, 0):cy + r, max(cx - r, 0):cx + r] = 0
    v[rng.random((n, n)) < 0.05] = 0
    d = np.stack([dx, dy, v], -1)
    return np.rint(d).astype(np.int32) if dtype == np.int32 else d.astype(np.float32)


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
def test_4096_rasters(vwb, ou, dtype):
    import torch
    d = realistic(11, 4096, dtype)
    t = torch.from_numpy(d).cuda()
    for method, kw in ((R.THRESH, dict(pt=3.0, rt=0.5)), (R.MEAN, dict(mmd=3.0)), (R.STDDEV, dict(pt=2.0, rt=0.5))):
        for cleanup in (False, True):
            got = engine(vwb, method, cleanup, t, 3, 2, **kw).cpu().numpy()
            want = ou.outlier_filter(method, cleanup, d, 3, 2, kw.get("pt", 0.0), kw.get("rt", 0.0), kw.get("mmd", 0.0))
            assert same(got, want), (method, cleanup)
            assert (got != d).any(-1).sum() > 10000


# ---- the C ABI: host and device inputs, padded pitches, NULL and side streams ------------------------------------------------
SENTINEL = -7777


def padded(d, pad):
    """d inside a wider (rows, cols + pad, 3) buffer whose padding holds the sentinel"""
    b = np.full((d.shape[0], d.shape[1] + pad, 3), SENTINEL, d.dtype)
    b[:, :d.shape[1]] = d
    return b


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
def test_abi_places_pitches_streams(vwb, ou, dtype):
    import torch
    L = vwb.lib()
    d = R.random_disparity(404, (37, 45), 0.2, dtype)
    side = torch.cuda.Stream()
    for method in METHODS:
        for cleanup in (0, 1):
            p = params(method, 3)
            want = ou.outlier_filter(method, cleanup, d, 2, 3, p["pt"], p["rt"], p["mmd"])
            prm = vwb.api.OutlierParams(method, cleanup, 2, 3, p["pt"], p["rt"], p["mmd"])
            ptype = 0 if dtype == np.int32 else 1
            for dev in (0, 1):
                for ipad, opad in ((0, 0), (3, 0), (0, 5), (2, 7)):
                    for stream in ((None, side) if dev else (None,)):
                        src, dst = padded(d, ipad), padded(np.zeros_like(d), opad)
                        if dev:
                            src, dst = torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda()
                        sp = C.c_void_p(stream.cuda_stream) if stream is not None else None
                        ptr = (lambda x: x.data_ptr()) if dev else (lambda x: x.ctypes.data)
                        torch.cuda.synchronize()             # the uploads are done before the call's stream reads them
                        rc = L.vwb200_outlier_filter(C.byref(prm), ptype, ptr(src), 45, 37, 45 + ipad, ptr(dst), 45 + opad, dev, sp)
                        assert rc == 0, vwb.lib().vwb200_last_error()
                        out = dst.cpu().numpy() if dev else dst
                        assert same(np.ascontiguousarray(out[:, :45]), want), (method, cleanup, dev, ipad, opad, stream)
                        assert (out[:, 45:] == SENTINEL).all(), "the pitch padding was written"
                        src_np = src.cpu().numpy() if dev else src
                        assert same(np.ascontiguousarray(src_np[:, :45]), d), "the input changed"


def test_abi_refuses_in_place(vwb):
    L = vwb.lib()
    d = R.random_disparity(1, (8, 8), 0.0, np.float32)
    prm = vwb.api.OutlierParams(1, 0, 1, 1, 0.0, 0.0, 1.0)
    assert L.vwb200_outlier_filter(C.byref(prm), 1, d.ctypes.data, 8, 8, 8, d.ctypes.data, 8, 0, None) == EARG
    assert L.vwb200_outlier_filter(C.byref(prm), 1, d.ctypes.data, 8, 4, 8, d[3:].ctypes.data, 8, 0, None) == EARG


@pytest.mark.parametrize("cleanup", [False, True])
@pytest.mark.parametrize("half", [(1, 1), (3, 2), (5, 5)])
def test_existing_int_thresh_entry_points(vwb, half, cleanup):
    """the existing integer thresh entry points give what vwb200_outlier_filter gives with VWB200_DISP_I32"""
    d = realistic(21, 300, np.int32)
    old = (vwb.disparity_cleanup_using_thresh if cleanup else vwb.rm_outliers_using_thresh)(d, half[0], half[1], 3.0, 0.5)
    assert same(old, engine(vwb, R.THRESH, cleanup, d, half[0], half[1], 3.0, 0.5))


@pytest.mark.parametrize("name,method", [("mean", R.MEAN), ("stddev", R.STDDEV)])
def test_view_output_filtered(vwb, ou, name, method):
    """a view's PixelMask<Vector2f> output on synthetic imagery, cleaned on the device, equals the oracle"""
    import torch
    from visionworkbench_b200.synth import make_pair
    search, kernel = (-12, -8, 12, 8), (7, 7)
    left, right, lm, rm, _ = make_pair(320, 256, search, seed=9)
    view = vwb.pyramid_correlate(left, right, lm, rm, vwb.PREFILTER_NONE, 0.0, search, kernel, vwb.ABSOLUTE_DIFFERENCE, 0, 0.0, 2.0, 0, 2, 3)
    disp = view.rasterize(None, (0, 0, 320, 256))
    assert disp.dtype == np.float32 and disp[..., 2].mean() > 0.5
    t = torch.from_numpy(disp).cuda()
    if method == R.MEAN:
        got, want = vwb.disparity_cleanup_using_mean(t, 5, 5, 2.0), ou.disparity_cleanup_using_mean(disp, 5, 5, 2.0)
    else:
        got, want = vwb.disparity_cleanup_using_stddev(t, 5, 5, 1.5, 0.5), ou.disparity_cleanup_using_stddev(disp, 5, 5, 1.5, 0.5)
    assert same(got.cpu().numpy(), want)
    # and on the host path
    host = vwb.disparity_cleanup_using_mean(disp, 5, 5, 2.0) if method == R.MEAN else vwb.disparity_cleanup_using_stddev(disp, 5, 5, 1.5, 0.5)
    assert same(host, want)


def largest_half_h(hy, words):
    """the largest half_h whose (32 + 2 hx) x (8 + 2 hy) tile of `words` 4-byte words fits the kernels' 200 KiB"""
    return ((200 * 1024) // (4 * words * (8 + 2 * hy)) - 32) // 2


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
@pytest.mark.parametrize("method", METHODS)
def test_window_limits(vwb, ou, method, dtype):
    """the largest accepted window, and VWB200_ENOIMPL one step above it.  The thresh filters stage two words per pixel
    (validity folded into dx); mean and stddev stage three."""
    words = 2 if method == R.THRESH else 3
    d = R.random_disparity(3, (12, 40), 0.3, dtype)
    for hy in (1, 20):
        hx = largest_half_h(hy, words)
        assert hx > 0
        for cleanup in (False, True):
            got = engine(vwb, method, cleanup, d, hx, hy, 2.0, 0.3, 4.0)
            assert same(got, ou.outlier_filter(method, cleanup, d, hx, hy, 2.0, 0.3, 4.0))
            with pytest.raises(vwb.NoImplErr, match="too large"):
                engine(vwb, method, cleanup, d, hx + 1, hy, 2.0, 0.3, 4.0)


# Traced in a process of its own, so that its profiler sessions neither depend on nor add to the ones of the rest of the suite.
TRACE_SCRIPT = """
import numpy as np, torch
import outlier_reference as R
import visionworkbench_b200 as v
from kernel_trace import KernelTrace


class OutlierTrace(KernelTrace):
    def hot(self):
        return {n for n in self.raw if "outlier" in n or "cleanup_pass2" in n}


torch.cuda.init()
for dt, tn in ((np.int32, "vwb200_dispi"), (np.float32, "DispF")):
    d = torch.from_numpy(R.random_disparity(8, (256, 300), 0.2, dt)).cuda()
    for m in range(3):
        for cleanup in (0, 1):
            fn = lambda: v.outlier_filter(m, cleanup, d, 2, 2, 3.0, 0.5, 3.0)
            fn()
            tr = OutlierTrace()
            tr.run(fn)
            print("CASE", tn, m, cleanup, "|".join(sorted(set(tr.raw))))
"""


def test_kernel_trace():
    """each filter ran its kernel, outlier_pass1_kernel<pixel type, method> and no other pass-1 kernel; the cleanup
    composites add cleanup_pass2_kernel<pixel type>"""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here]), PYTHONNOUSERSITE="1")
    r = subprocess.run([sys.executable, "-c", TRACE_SCRIPT], cwd=here, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    cases = [ln.split(" ", 4)[1:] for ln in r.stdout.splitlines() if ln.startswith("CASE ")]
    assert len(cases) == 12, r.stdout
    for tn, m, cleanup, names in cases:
        names = names.split("|")
        want = re.compile(rf"outlier_pass1_kernel<(vwb200::)?{tn}, (\(int\))?{m}>")
        assert any(want.search(n) for n in names), (tn, m, cleanup, names)
        assert all(want.search(n) or "cleanup_pass2_kernel" in n for n in names), names
        assert any("cleanup_pass2_kernel" in n for n in names) == (cleanup == "1"), names
