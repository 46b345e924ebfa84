"""The device's disparity resampling, range and transform operations (vwb200_disparity_subsample / _upsample,
vwb200_get_disparity_range, vwb200_disparity_range_mask, vwb200_transform_disparities on int32 and float32 disparities)
against the oracle, bit for bit (floats as raw bits, NaN equal to NaN): the CPU matrix of test_oracle_dispmap.py, where the
oracle is checked against the restatement of the reference, 4096^2 and 8192 x 1 / 1 x 8192 rasters, a view's float output,
host and device paths with padded pitches, NULL and side streams, out == in for the per-pixel calls, and the K7 kernel each
call ran.

The module sorts after the ones that trace kernels with torch.profiler in the pytest process."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import dispmap_reference as R
from test_oracle_dispmap import INVALID, MATRICES, SHAPES, TYPES, dm, nan_cases, same, signed_zero_case  # noqa: F401  (dm: fixture)

pytestmark = pytest.mark.gpu
EARG = -1


@pytest.fixture(scope="module")
def vwb():
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "GPU tests need a CUDA device: the engine has no CPU path"
    return v


def bounds(d):
    h, w = d.shape[:2]
    return (((-5, -3), (w + 4, h + 2)), ((0, 0), (w, h)), ((-30, 10), (w - 3, h + 40)))


def check_engine(vwb, dm, d, i):
    """every call on d (numpy, then the same raster as a CUDA tensor) against the oracle"""
    import torch
    for x in (d, torch.from_numpy(d).cuda()):
        host = lambda a: a.cpu().numpy() if hasattr(a, "cpu") else a       # noqa: E731
        assert same(host(vwb.disparity_subsample(x)), dm.disparity_subsample(d))
        assert same(host(vwb.disparity_upsample(x)), dm.disparity_upsample(d))
        assert same(np.array(vwb.get_disparity_range(x), np.float32), dm.get_disparity_range(d))
        for mn, mx in bounds(d):
            assert same(host(vwb.disparity_range_mask(x, mn, mx)), dm.disparity_range_mask(d, mn, mx)), (mn, mx)
        m = MATRICES[i % len(MATRICES)]
        assert same(host(vwb.transform_disparities(x, m)), dm.transform_disparities(dm.LAZY, np.linalg.inv(m), d))
        for do_round in (False, True):
            for origin in ((0, 0), (17, -9)):
                box = (origin[0], origin[1], origin[0] + d.shape[1], origin[1] + d.shape[0])
                got = host(vwb.transform_disparities_explicit(do_round, box, m, x))
                assert same(got, dm.transform_disparities(dm.EXPLICIT, m, d, do_round, origin)), (do_round, origin)


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("invalid", INVALID)
def test_matrix(vwb, dm, invalid, shape, dtype):
    i = SHAPES.index(shape) + INVALID.index(invalid)
    check_engine(vwb, dm, R.random_disparity(1000 + 7 * i, shape, invalid, dtype), i)
    # several tiles of the subsample kernel, with partial ones
    check_engine(vwb, dm, R.random_disparity(2000 + 7 * i, (37 + shape[0], 131 + shape[1]), invalid, dtype), i)


def test_hand_cases(vwb, dm):
    check_engine(vwb, dm, signed_zero_case(), 0)
    a, b = nan_cases()
    check_engine(vwb, dm, a, 1)
    check_engine(vwb, dm, b, 2)
    for dtype in TYPES:
        d = R.random_disparity(77, (9, 11), 0.25, dtype, scale=1e3)
        d[..., :2] = -np.abs(d[..., :2])
        check_engine(vwb, dm, d, 0)
    d = np.zeros((3, 3, 3), np.int32)
    d[...] = (0, 0, 1)
    d[1, 1] = (0, -5, 1)
    for mn in ((-10, 0), (-3, -10)):
        assert same(vwb.disparity_range_mask(d, mn, (10, 10)), dm.disparity_range_mask(d, mn, (10, 10)))
    h = np.zeros((1, 4, 3), np.float32)
    h[0] = [(0.5, -0.5, 1), (1.5, -1.5, 1), (2.5, -2.5, 1), (0.49999997, -0.49999997, 1)]
    assert same(vwb.transform_disparities_explicit(True, (0, 0, 4, 1), np.eye(3), h), dm.transform_disparities(dm.EXPLICIT, np.eye(3), h, True))
    # the range of a raster without a valid pixel, and a NaN met after the first pixel of a large raster
    z = R.random_disparity(3, (300, 500), 1.0, np.float32)
    assert vwb.get_disparity_range(z) == (0.0, 0.0, 0.0, 0.0)
    big = R.random_disparity(4, (300, 500), 0.5, np.float32)
    big[200, 400, :] = (np.nan, np.nan, 1)
    assert same(np.array(vwb.get_disparity_range(big), np.float32), dm.get_disparity_range(big))


def realistic(seed, h, w, dtype):
    """a smooth field with -0.0 / +0.0 zeros, speckle and holes"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    dx = 20 * np.sin(xx / 300) + 0.004 * yy + 0.3 * rng.standard_normal((h, w), np.float32)
    dy = 2 * np.cos(yy / 500) + 0.2 * rng.standard_normal((h, w), np.float32)
    dx[rng.random((h, w)) < 0.01] = -0.0
    dy[rng.random((h, w)) < 0.01] = 0.0
    v = (rng.random((h, w)) >= 0.1).astype(np.float32)
    d = np.stack([dx, dy, v], -1)
    return np.rint(d).astype(np.int32) if dtype == np.int32 else d


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
@pytest.mark.parametrize("shape", [(4096, 4096), (1, 8192), (8192, 1)], ids=["4096^2", "1x8192", "8192x1"])
def test_large_rasters(vwb, dm, shape, dtype):
    import torch
    d = realistic(11 + shape[1], shape[0], shape[1], dtype)
    t = torch.from_numpy(d).cuda()
    assert same(vwb.disparity_subsample(t).cpu().numpy(), dm.disparity_subsample(d))
    assert same(vwb.disparity_upsample(t).cpu().numpy(), dm.disparity_upsample(d))
    assert same(np.array(vwb.get_disparity_range(t), np.float32), dm.get_disparity_range(d))
    mn, mx = (-3, -2), (shape[1] - 5, shape[0] + 1)
    assert same(vwb.disparity_range_mask(t, mn, mx).cpu().numpy(), dm.disparity_range_mask(d, mn, mx))
    m = MATRICES[1]
    assert same(vwb.transform_disparities(t, m).cpu().numpy(), dm.transform_disparities(dm.LAZY, np.linalg.inv(m), d))
    box = (100, -50, 100 + shape[1], -50 + shape[0])
    assert same(vwb.transform_disparities_explicit(True, box, m, t).cpu().numpy(), dm.transform_disparities(dm.EXPLICIT, m, d, True, (100, -50)))


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
@pytest.mark.parametrize("shape", [(70000, 3), (1100000, 1)], ids=["70000x3", "1100000x1"])
def test_tall_rasters(vwb, dm, shape, dtype):
    """more rows than a grid has blocks in y (65535): every kernel deals its rows to the blocks.  1100000 rows give the
    subsample kernel more than 65535 tile rows as well."""
    import torch
    d = R.random_disparity(31 + shape[1], shape, 0.2, dtype)
    t = torch.from_numpy(d).cuda()
    assert same(vwb.disparity_subsample(t).cpu().numpy(), dm.disparity_subsample(d))
    assert same(vwb.disparity_upsample(t).cpu().numpy(), dm.disparity_upsample(d))
    assert same(np.array(vwb.get_disparity_range(t), np.float32), dm.get_disparity_range(d))
    mn, mx = (-20, -8), (shape[1] + 10, shape[0] - 3)
    assert same(vwb.disparity_range_mask(t, mn, mx).cpu().numpy(), dm.disparity_range_mask(d, mn, mx))
    m = MATRICES[1]
    assert same(vwb.transform_disparities(t, m).cpu().numpy(), dm.transform_disparities(dm.LAZY, np.linalg.inv(m), d))
    box = (4, 9, 4 + shape[1], 9 + shape[0])
    assert same(vwb.transform_disparities_explicit(True, box, m, t).cpu().numpy(), dm.transform_disparities(dm.EXPLICIT, m, d, True, (4, 9)))
    # int32 results outside the range (w of the projective matrix crosses zero near row 50000): INT32_MIN on both sides
    if dtype == np.int32 and shape[0] == 70000:
        assert (dm.transform_disparities(dm.EXPLICIT, m, d, True, (4, 9))[..., :2] == -2 ** 31).any()
    # and in place, on the device
    u = t.clone()
    assert vwb.transform_disparities(u, m, out=u) is u
    assert same(u.cpu().numpy(), dm.transform_disparities(dm.LAZY, np.linalg.inv(m), d))


def test_view_output(vwb, dm):
    """a view's PixelMask<Vector2f> output on synthetic imagery, resampled, ranged and transformed on the device"""
    from visionworkbench_b200.synth import make_pair
    search, kernel = (-12, -8, 12, 8), (7, 7)
    left, right, lm, rm, _ = make_pair(320, 256, search, seed=9)
    view = vwb.pyramid_correlate(left, right, lm, rm, vwb.PREFILTER_NONE, 0.0, search, kernel, vwb.ABSOLUTE_DIFFERENCE, 0, 0.0, 2.0, 0, 2, 3)
    disp = view.rasterize(None, (0, 0, 320, 256))
    assert disp.dtype == np.float32 and disp[..., 2].mean() > 0.5
    check_engine(vwb, dm, disp, 1)


# ---- the C ABI: host and device inputs, padded pitches, NULL and side streams, out == in -----------------------------------------
SENTINEL = -7777


def padded(d, pad):
    b = np.full((d.shape[0], d.shape[1] + pad, 3), SENTINEL, d.dtype)
    b[:, :d.shape[1]] = d
    return b


@pytest.mark.parametrize("dtype", TYPES, ids=["i32", "f32"])
def test_abi_places_pitches_streams(vwb, dm, dtype):
    import torch
    L = vwb.lib()
    d = R.random_disparity(404, (37, 45), 0.2, dtype)
    h, w = d.shape[:2]
    pt = 0 if dtype == np.int32 else 1
    side = torch.cuda.Stream()
    mn, mx = np.array([-2, -1], dtype), np.array([w + 3, h - 2], dtype)
    m = np.ascontiguousarray(MATRICES[1].reshape(9))
    box = (C.c_int32 * 4)(5, 6, 5 + w, 6 + h)
    # (name, output shape, call(src, w, h, pitch, dst, opitch, dev, stream), expected)
    calls = [
        ("subsample", (1 + (h - 1) // 2, 1 + (w - 1) // 2), lambda s, ip, o, op, dev, sp: L.vwb200_disparity_subsample(pt, s, w, h, ip, o, op, dev, sp),
         dm.disparity_subsample(d)),
        ("upsample", (2 * h, 2 * w), lambda s, ip, o, op, dev, sp: L.vwb200_disparity_upsample(pt, s, w, h, ip, o, op, dev, sp), dm.disparity_upsample(d)),
        ("range_mask", (h, w), lambda s, ip, o, op, dev, sp: L.vwb200_disparity_range_mask(pt, s, w, h, ip, mn.ctypes.data, mx.ctypes.data, o, op, dev, sp),
         dm.disparity_range_mask(d, mn, mx)),
        ("lazy", (h, w), lambda s, ip, o, op, dev, sp: L.vwb200_transform_disparities(pt, 0, m.ctypes.data, 0, None, s, w, h, ip, o, op, dev, sp),
         dm.transform_disparities(dm.LAZY, m, d)),
        ("explicit", (h, w), lambda s, ip, o, op, dev, sp: L.vwb200_transform_disparities(pt, 1, m.ctypes.data, 1, box, s, w, h, ip, o, op, dev, sp),
         dm.transform_disparities(dm.EXPLICIT, m, d, True, (5, 6))),
    ]
    for name, oshape, call, want in calls:
        for dev in (0, 1):
            for ipad, opad in ((0, 0), (3, 0), (0, 5), (2, 7)):
                for stream in ((None, side) if dev else (None,)):
                    src, dst = padded(d, ipad), padded(np.zeros(oshape + (3,), dtype), opad)
                    if dev:
                        src, dst = torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda()
                    sp = C.c_void_p(stream.cuda_stream) if stream is not None else None
                    ptr = (lambda x: x.data_ptr()) if dev else (lambda x: x.ctypes.data)
                    torch.cuda.synchronize()
                    rc = call(ptr(src), w + ipad, ptr(dst), oshape[1] + opad, dev, sp)
                    assert rc == 0, vwb.lib().vwb200_last_error()
                    out = dst.cpu().numpy() if dev else dst
                    assert same(np.ascontiguousarray(out[:, :oshape[1]]), want), (name, dev, ipad, opad, stream)
                    assert (out[:, oshape[1]:] == SENTINEL).all(), "the pitch padding was written"
                    src_np = src.cpu().numpy() if dev else src
                    assert same(np.ascontiguousarray(src_np[:, :w]), d), "the input changed"
        if oshape == (h, w):                                               # the per-pixel calls also run in place
            for dev in (0, 1):
                for ipad in (0, 4):
                    buf = padded(d, ipad)
                    if dev:
                        buf = torch.from_numpy(buf).cuda()
                    ptr = buf.data_ptr() if dev else buf.ctypes.data
                    assert call(ptr, w + ipad, ptr, w + ipad, dev, None) == 0, vwb.lib().vwb200_last_error()
                    got = buf.cpu().numpy() if dev else buf
                    assert same(np.ascontiguousarray(got[:, :w]), want), (name, "in place", dev, ipad)
                    assert (got[:, w:] == SENTINEL).all()
    # get_disparity_range on every place and pitch
    r, flag = (C.c_float * 4)(), C.c_int(-1)
    for dev in (0, 1):
        for ipad in (0, 3):
            src = padded(d, ipad)
            src = torch.from_numpy(src).cuda() if dev else src
            ptr = src.data_ptr() if dev else src.ctypes.data
            assert L.vwb200_get_disparity_range(pt, ptr, w, h, w + ipad, r, C.byref(flag), dev, C.c_void_p(side.cuda_stream) if dev else None) == 0
            assert same(np.array(list(r), np.float32), dm.get_disparity_range(d)) and flag.value == 1
    # python in place
    for x in (d.copy(), torch.from_numpy(d.copy()).cuda()):
        o = vwb.disparity_range_mask(x, mn, mx, out=x)
        got = x.cpu().numpy() if hasattr(x, "cpu") else x
        assert o is x and same(got, dm.disparity_range_mask(d, mn, mx))


def test_abi_refuses_overlap(vwb):
    L = vwb.lib()
    d = R.random_disparity(1, (8, 8), 0.0, np.float32)
    big = np.zeros((16, 16, 3), np.float32)
    assert L.vwb200_disparity_subsample(1, d.ctypes.data, 8, 8, 8, d.ctypes.data, 4, 0, None) == EARG
    assert L.vwb200_disparity_upsample(1, big.ctypes.data, 8, 8, 8, big[2:].ctypes.data, 16, 0, None) == EARG
    m = np.eye(3).reshape(9)
    assert L.vwb200_transform_disparities(1, 0, m.ctypes.data, 0, None, d.ctypes.data, 8, 4, 8, d[2:].ctypes.data, 8, 0, None) == EARG
    assert L.vwb200_transform_disparities(1, 0, m.ctypes.data, 0, None, d.ctypes.data, 4, 4, 8, d.ctypes.data, 4, 0, None) == EARG


# Traced in a process of its own, so that its profiler sessions neither depend on nor add to the ones of the rest of the suite.
TRACE_SCRIPT = """
import numpy as np, torch
import dispmap_reference as R
import visionworkbench_b200 as v
from kernel_trace import KernelTrace


class K7Trace(KernelTrace):
    def hot(self):
        return {n for n in self.raw if "k7_" in n}


torch.cuda.init()
m = np.array([[0.98, 0.03, 12.5], [-0.02, 1.01, -7.25], [1.5e-5, -2e-5, 1.0]])
for dt, tn in ((np.int32, "vwb200_dispi"), (np.float32, "DispF")):
    d = torch.from_numpy(R.random_disparity(8, (256, 300), 0.2, dt)).cuda()
    calls = {"subsample": lambda: v.disparity_subsample(d), "upsample": lambda: v.disparity_upsample(d),
             "range": lambda: v.get_disparity_range(d), "range_mask": lambda: v.disparity_range_mask(d, (0, 0), (300, 256)),
             "lazy": lambda: v.transform_disparities(d, m), "explicit": lambda: v.transform_disparities_explicit(True, (0, 0, 300, 256), m, d)}
    for name, fn in calls.items():
        fn()
        tr = K7Trace()
        tr.run(fn)
        print("CASE", tn, name, "|".join(sorted(set(tr.raw))))
"""

WANT = {"subsample": r"k7_subsample_kernel<(vwb200::)?{tn}>", "upsample": r"k7_upsample_kernel<(vwb200::)?{tn}>",
        "range": r"k7_range_kernel<(vwb200::)?{tn}>", "range_mask": r"k7_pixel_kernel<(vwb200::)?{tn}, .*RangeMaskOp",
        "lazy": r"k7_pixel_kernel<(vwb200::)?{tn}, .*TransformLazyOp", "explicit": r"k7_pixel_kernel<(vwb200::)?{tn}, .*TransformExplicitOp"}


def test_kernel_trace():
    """each call ran its K7 kernel (get_disparity_range also its final step)"""
    import re
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here]), PYTHONNOUSERSITE="1")
    r = subprocess.run([sys.executable, "-c", TRACE_SCRIPT], cwd=here, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    cases = [ln.split(" ", 3)[1:] for ln in r.stdout.splitlines() if ln.startswith("CASE ")]
    assert len(cases) == 12, r.stdout
    for tn, name, names in cases:
        names = names.split("|")
        assert any(re.search(WANT[name].format(tn=tn), n) for n in names), (tn, name, names)
        assert any("k7_range_final_kernel" in n for n in names) == (name == "range"), names
