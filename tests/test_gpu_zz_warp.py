"""The device's image warp (vwb200_transform_image / transform with HomographyTransform or DisparityTransform) against the
oracle, bit for bit (floats as raw bits, NaN equal to NaN, 0.0f outside the contract's domain on both sides): the CPU matrix of
test_oracle_warp.py, where the oracle is checked against the restatement of the reference, 4096^2 rasters for each
interpolation, 1 x 70000 / 70000 x 1 / 1 x 600000 windows, host and device paths with padded pitches on NULL and side
streams, window crops against crops of the whole window, the correlate.cc chain on 512^2 integer imagery, and the
k8_warp_kernel instantiation each case ran.

The module sorts after the ones that trace kernels with torch.profiler in the pytest process."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import warp_reference as R
from test_oracle_warp import EDGES, INTERPS, KINDS, MATRICES, SHAPES, cases, disparity, image, same, wo  # noqa: F401  (wo: fixture)

pytestmark = pytest.mark.gpu
EARG = -1


@pytest.fixture(scope="module")
def vwb():
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "GPU tests need a CUDA device: the engine has no CPU path"
    return v


def tx_of(vwb, kind, m, d, dev=False):
    """the Python transform object for a case.  m is the matrix reverse() applies, so H = inverse(m); HomographyTransform
    inverts H again, and the oracle is given that H_inverse, the matrix the engine applies."""
    import torch
    if kind == R.HOMOGRAPHY:
        return vwb.HomographyTransform(np.linalg.inv(m))
    return vwb.DisparityTransform(torch.from_numpy(d).cuda() if dev else d)


def engine(vwb, im, kind, interp, edge, win, m, d, dev):
    import torch
    tx = tx_of(vwb, kind, m, d, dev)
    x0, y0, ow, oh = win
    x = torch.from_numpy(im).cuda() if dev else im
    got = vwb.transform(x, tx, (x0, y0, x0 + ow, y0 + oh), edge, interp)
    return (got.cpu().numpy() if dev else got), (tx.H_inverse if kind == R.HOMOGRAPHY else None)


def check(vwb, wo, im, kind, interp, edge, win, m, d, label=""):
    for dev in (False, True):
        got, minv = engine(vwb, im, kind, interp, edge, win, m, d, dev)
        want = wo.transform(im, kind, interp, edge, win, matrix=minv, disparity=d)
        assert same(got, want), (label, dev, np.argwhere(~((got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))))[:5])


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("edge", EDGES, ids=["zero", "constant"])
@pytest.mark.parametrize("interp", INTERPS, ids=["bilinear", "bicubic", "nearest"])
@pytest.mark.parametrize("kind", KINDS, ids=["homography", "disparity"])
def test_matrix(vwb, wo, kind, interp, edge, shape):
    for label, im, win, m, d in cases(kind, shape):
        check(vwb, wo, im, kind, interp, edge, win, m, d, label)


@pytest.mark.parametrize("edge", EDGES, ids=["zero", "constant"])
@pytest.mark.parametrize("interp", INTERPS, ids=["bilinear", "bicubic", "nearest"])
def test_special_pixels_and_domain(vwb, wo, interp, edge):
    im = image(5, (21, 34), special=0.08)
    for name in ("identity", "frac_shift", "rot_scale", "near_int", "halves", "w_crosses_0"):
        check(vwb, wo, im, R.HOMOGRAPHY, interp, edge, (-2, -2, 38, 25), MATRICES[name], None, name)
    check(vwb, wo, im, R.DISPARITY, interp, edge, (-2, -2, 38, 25), None, disparity(6, (21, 34), 0.3), "disparity")
    # the out-of-domain rule: a w of 1e-300 (every pixel but the origin leaves the domain or overflows to inf / NaN), and
    # reversed x = 2^30 - 1 (inside) next to 2^30 (outside)
    for H, win in ((np.diag([1, 1, 1e300]), (0, 0, 34, 21)), (np.array([[1, 0, 1 - 2.0 ** 30], [0, 1, 0], [0, 0, 1.0]]), (0, 0, 2, 1))):
        tx = vwb.HomographyTransform(H)
        got = vwb.transform(im, tx, (win[0], win[1], win[0] + win[2], win[1] + win[3]), edge, interp)
        assert same(got, wo.transform(im, R.HOMOGRAPHY, interp, edge, win, matrix=tx.H_inverse))
        assert (got.view(np.uint32) == 0).sum() >= (win[2] * win[3] - 1 if win[2] > 2 else 1)


def smooth_image(seed, h, w):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    return (100 * np.sin(xx / 97) * np.cos(yy / 61) + 5 * rng.standard_normal((h, w), np.float32)).astype(np.float32)


@pytest.mark.parametrize("interp", INTERPS, ids=["bilinear", "bicubic", "nearest"])
def test_4096_rasters(vwb, wo, interp):
    import torch
    n = 4096
    im = smooth_image(40 + interp, n, n)
    t = torch.from_numpy(im).cuda()
    H = np.array([[1.01, 0.02, -12.5], [-0.015, 0.995, 7.25], [2e-6, -3e-6, 1.0]])
    tx = vwb.HomographyTransform(H)
    got = vwb.transform(t, tx, None, vwb.EDGE_CONSTANT if interp == R.BICUBIC else vwb.EDGE_ZERO, interp).cpu().numpy()
    assert same(got, wo.transform(im, R.HOMOGRAPHY, interp, R.CONSTANT if interp == R.BICUBIC else R.ZERO, (0, 0, n, n), matrix=tx.H_inverse))
    # window crops are crops of the whole window (every pixel depends on its own coordinates only)
    for x0, y0, ow, oh in ((0, 0, 33, 7), (1000, 2047, 517, 301), (4000, 4090, 96, 6), (-5, 4093, 4101, 3)):
        c = vwb.transform(t, tx, (x0, y0, x0 + ow, y0 + oh), vwb.EDGE_CONSTANT if interp == R.BICUBIC else vwb.EDGE_ZERO, interp).cpu().numpy()
        ix0, iy0 = max(x0, 0), max(y0, 0)
        ix1, iy1 = min(x0 + ow, n), min(y0 + oh, n)
        assert same(c[iy0 - y0:iy1 - y0, ix0 - x0:ix1 - x0], got[iy0:iy1, ix0:ix1]), (x0, y0, ow, oh)
    if interp == R.BILINEAR:                                              # and a DisparityTransform over the whole raster
        d = disparity(41, (n, n), 0.1)
        got = vwb.transform(t, vwb.DisparityTransform(torch.from_numpy(d).cuda()), None, vwb.EDGE_ZERO, interp).cpu().numpy()
        assert same(got, wo.transform(im, R.DISPARITY, interp, R.ZERO, (0, 0, n, n), disparity=d))


@pytest.mark.parametrize("win", [(0, 0, 70000, 1), (0, 0, 1, 70000), (-3, -300000, 1, 600000)], ids=["1x70000", "70000x1", "600000x1"])
@pytest.mark.parametrize("kind", KINDS, ids=["homography", "disparity"])
def test_thin_windows(vwb, wo, kind, win):
    """600000 rows are more row tiles than a grid has blocks in y (65535 x 8 rows): the kernel deals them to the blocks"""
    im = image(50, (37, 53))
    m, d = (MATRICES["rot_scale"], None) if kind == R.HOMOGRAPHY else (None, disparity(51, (40, 60), 0.2))
    for interp in INTERPS:
        check(vwb, wo, im, kind, interp, R.CONSTANT, win, m, d, interp)


# ---- the C ABI: host and device rasters, padded pitches, NULL and side streams --------------------------------------------------
SENTINEL = -7777.0


def padded(a, pad):
    b = np.full((a.shape[0], a.shape[1] + pad) + a.shape[2:], SENTINEL, a.dtype)
    b[:, :a.shape[1]] = a
    return b


@pytest.mark.parametrize("kind", KINDS, ids=["homography", "disparity"])
def test_abi_places_pitches_streams(vwb, wo, kind):
    import torch
    L = vwb.lib()
    im = image(60, (29, 41))
    d = disparity(61, (25, 44), 0.3)
    m = MATRICES["projective"]
    side = torch.cuda.Stream()
    x0, y0, ow, oh = -4, 3, 47, 30
    for interp in INTERPS:
        for edge in EDGES:
            p = vwb.WarpParams(kind, interp, edge)
            p.matrix[:] = list(m.reshape(9))
            want = wo.transform(im, kind, interp, edge, (x0, y0, ow, oh), matrix=m, disparity=d)
            for dev in (0, 1):
                for ipad, dpad, opad in ((0, 0, 0), (3, 0, 0), (0, 2, 5), (2, 7, 1)):
                    for stream in ((None, side) if dev else (None,)):
                        src, dsp, dst = padded(im, ipad), padded(d, dpad), padded(np.zeros((oh, ow), np.float32), opad)
                        if dev:
                            src, dsp, dst = (torch.from_numpy(a).cuda() for a in (src, dsp, dst))
                        ptr = (lambda a: a.data_ptr()) if dev else (lambda a: a.ctypes.data)
                        sp = C.c_void_p(stream.cuda_stream) if stream is not None else None
                        torch.cuda.synchronize()
                        rc = L.vwb200_transform_image(C.byref(p), ptr(src), 41, 29, 41 + ipad, ptr(dsp) if kind else None, 44, 25, 44 + dpad,
                                                      x0, y0, ptr(dst), ow, oh, ow + opad, dev, sp)
                        assert rc == 0, L.vwb200_last_error()
                        out = dst.cpu().numpy() if dev else dst
                        assert same(np.ascontiguousarray(out[:, :ow]), want), (interp, edge, dev, ipad, dpad, opad, stream)
                        assert (out[:, ow:] == SENTINEL).all(), "the pitch padding was written"
                        src_np = src.cpu().numpy() if dev else src
                        assert same(np.ascontiguousarray(src_np[:, :41]), im), "the input changed"


def test_abi_refuses_overlap(vwb):
    L = vwb.lib()
    im = np.zeros((8, 8), np.float32)
    p = vwb.WarpParams(0, 0, 0)
    p.matrix[:] = list(np.eye(3).reshape(9))
    assert L.vwb200_transform_image(C.byref(p), im.ctypes.data, 8, 8, 8, None, 0, 0, 0, 0, 0, im[4:].ctypes.data, 8, 4, 8, 0, None) == EARG


def test_correlate_chain(vwb, wo):
    """tools/correlate.cc with a match file: the right image pre-aligned by transform(right, HomographyTransform(alignment))
    (nearest-pixel here, so the imagery stays integral and the exact block-matching paths apply), calc_disparity, and
    transform_disparities(disparity, HomographyTransform(alignment)), on the device and on the oracles"""
    import torch

    import oracle
    import oracle.dispmap as dm
    from visionworkbench_b200.synth import make_rasters
    search, kernel = (16, 12), (7, 7)
    left, right = make_rasters(500, 500, search, kernel, seed=12)
    alignment = np.array([[1.002, 0.004, -1.5], [-0.003, 0.998, 1.25], [1e-6, -2e-6, 1.0]])
    tx = vwb.HomographyTransform(alignment)
    for dev in (False, True):
        r = torch.from_numpy(right).cuda() if dev else right
        aligned = vwb.transform(r, tx, None, vwb.EDGE_ZERO, vwb.INTERP_NEAREST)
        lt = torch.from_numpy(left).cuda() if dev else left
        disp = vwb.calc_disparity(vwb.ABSOLUTE_DIFFERENCE, lt, aligned, search, kernel)
        final = vwb.transform_disparities(disp, alignment)
        a_ref = wo.transform(right, R.HOMOGRAPHY, R.NEAREST, R.ZERO, (0, 0, right.shape[1], right.shape[0]), matrix=tx.H_inverse)
        assert np.all(a_ref == np.rint(a_ref))
        d_ref = oracle.calc_disparity(0, left, a_ref, search, kernel)
        f_ref = dm.transform_disparities(dm.LAZY, np.linalg.inv(alignment), d_ref)
        host = (lambda a: a.cpu().numpy()) if dev else (lambda a: a)
        assert same(host(aligned), a_ref)
        assert np.array_equal(host(disp), d_ref)
        assert np.array_equal(host(final), f_ref)
        assert d_ref[..., 2].mean() > 0.5


# Traced in a process of its own, so that its profiler sessions neither depend on nor add to the ones of the rest of the suite.
TRACE_SCRIPT = """
import numpy as np, torch
import visionworkbench_b200 as v
from kernel_trace import KernelTrace


class K8Trace(KernelTrace):
    def hot(self):
        return {n for n in self.raw if "k8_" in n}


torch.cuda.init()
im = torch.rand(200, 300, device="cuda")
d = torch.zeros(200, 300, 3, device="cuda")
d[..., 2] = 1
for kind, tx in ((0, v.HomographyTransform(np.array([[1.0, 0.01, 2.5], [0, 1, -1.5], [1e-5, 0, 1]]))), (1, v.DisparityTransform(d))):
    for interp in (0, 1, 2):
        for edge in (0, 1):
            fn = lambda: v.transform(im, tx, None, edge, interp)
            fn()
            tr = K8Trace()
            tr.run(fn)
            print("CASE", kind, interp, edge, "|".join(sorted(set(tr.raw))))
"""


def test_kernel_trace():
    """each case ran the k8_warp_kernel<Kind, Interp, Edge> instantiation of its arguments, and only that one"""
    import re
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here]), PYTHONNOUSERSITE="1")
    r = subprocess.run([sys.executable, "-c", TRACE_SCRIPT], cwd=here, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    cases_ = [ln.split(" ", 4)[1:] for ln in r.stdout.splitlines() if ln.startswith("CASE ")]
    assert len(cases_) == 12, r.stdout
    for kind, interp, edge, names in cases_:
        k8 = {n for n in names.split("|") if "k8_warp_kernel" in n}
        want = re.compile(rf"k8_warp_kernel<\(?(int\)?)?{kind}, \(?(int\)?)?{interp}, \(?(int\)?)?{edge}>")
        assert len(k8) == 1 and want.search(next(iter(k8))), (kind, interp, edge, names)
