"""Epipolar rectification on the device against the oracle, bit for bit (floats and doubles as raw bits, NaN equal to NaN):
camera_transform through K8's camera kind for NULL / TSAI / TSAI-with-k3 source cameras into epipolar and Tsai destination
cameras, pixel pitches and u, v, w frames, every float interpolation x edge, PixelMask<float> bilinear x zero / constant /
value edges with 0-100 % invalid pixels and NaN values, 1 x 1 to 8192^2, whole / interior / edge / 1-pixel / outside windows,
host and device rasters with padded pitches on the NULL and a side stream; resize_epipolar_cameras_to_fit over square,
non-square and 1-pixel ROIs; PointToPixelErr with the oracle's first failing pixel; which kernel each case ran; and the chain
epipolar -> resize -> epipolar_transformed_images -> pyramid_correlate -> stereo_triangulate on a rendered plane."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
from scipy import ndimage
from scipy.spatial.transform import Rotation

from oracle import epipolar as oe
from oracle import triangulate as ot
from test_oracle_epipolar import cam_bits
from test_oracle_triangulate import STRONG, TSAI, TSAI_K3, api_cam

pytestmark = pytest.mark.gpu
BILINEAR, BICUBIC, NEAREST = 0, 1, 2
ZERO, CONSTANT, VALUE = 0, 1, 2


@pytest.fixture(scope="module")
def vwb():
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "GPU tests need a CUDA device: the engine has no CPU path"
    return v


def same32(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != np.float32 or b.dtype != np.float32:
        return False
    return bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


def rig(seed, w, h, lens0, lens1=None, pitch=1.0, frame=False):
    """two seeded cameras about 1 apart over a w x h image (f about 0.9 w), small tilts; frame=True: a non-identity u, v, w
    frame on the first"""
    rng = np.random.default_rng(seed)
    cams = []
    for k, lens in enumerate((lens0, lens1)):
        R = Rotation.from_rotvec(rng.normal(0, 0.04, 3)).as_matrix()
        f = max(w, 4) * rng.uniform(0.85, 0.95) * pitch
        c = ot.camera(center=(k * rng.uniform(0.8, 1.2), rng.normal(0, 0.05), rng.normal(0, 0.05)), rotation=R, fu=f, fv=f * rng.uniform(0.98, 1.02),
                      cu=(w / 2 + rng.normal(0, 1)) * pitch, cv=(h / 2 + rng.normal(0, 1)) * pitch, pixel_pitch=pitch, tsai=lens)
        if frame and k == 0:
            c.update(u=(0.0, 1.0, 0.0), v=(1.0, 0.0, 0.0), w=(0.0, 0.0, -1.0), rotation=R @ np.array([[0, 1, 0], [1, 0, 0], [0, 0, -1.0]]))
        cams.append(c)
    return cams


def image(w, h, seed, masked=False, invalid=0.0):
    rng = np.random.default_rng(seed)
    v = (rng.random((h, w)) * 200 - 50).astype(np.float32)
    v[rng.random((h, w)) < 0.02] = np.nan
    if not masked:
        return v
    m = np.zeros((h, w, 2), np.float32)
    m[..., 0] = v
    m[..., 1] = (rng.random((h, w)) >= invalid).astype(np.float32)
    m[..., 1][rng.random((h, w)) < 0.05] = 0.5                    # any non-zero valid word counts as valid
    return m


def engine(vwb, img, src, dst, win, interp, edge, ev=(0.0, 0.0), dev=False, pad=0, stream=False):
    import torch
    x0, y0, ow_, oh_ = win
    x = img
    if dev:
        t = torch.from_numpy(img).cuda()
        if pad:
            big = torch.zeros((t.shape[0], t.shape[1] + pad) + tuple(t.shape[2:]), device="cuda")
            big[:, :t.shape[1]] = t
            t = big[:, :img.shape[1]]
        x = t
    s = torch.cuda.Stream() if stream else None
    with torch.cuda.stream(s) if s is not None else torch.cuda.device(0):
        got = vwb.camera_transform(x, api_cam(vwb, src), api_cam(vwb, dst), bbox=(x0, y0, x0 + ow_, y0 + oh_), edge=edge, interp=interp,
                                   edge_value=ev)
    if s is not None:
        s.synchronize()
    return got.cpu().numpy() if dev else got


def check(vwb, img, src, dst, win, interp, edge, ev=(0.0, 0.0), variants=((False, 0, False), (True, 3, False), (True, 0, True)), label=""):
    """the engine equals the oracle on every variant (device?, pitch padding, side stream?); where the oracle throws
    PointToPixelErr, the engine does too, naming the same first failing pixel"""
    try:
        want = oe.camera_transform(img, src, dst, win, interp, edge, ev)
    except oe.PointToPixelErr as e:
        for dev, pad, stream in variants:
            with pytest.raises(vwb.PointToPixelErr) as g:
                engine(vwb, img, src, dst, win, interp, edge, ev, dev, pad, stream)
            assert failing_pixel(g.value) == tuple(e.where), (label, win, str(g.value), e.where)
        return None
    for dev, pad, stream in variants:
        got = engine(vwb, img, src, dst, win, interp, edge, ev, dev, pad, stream)
        assert same32(got, want), (label, win, dev, pad, stream)
    return want


def failing_pixel(err):
    return tuple(int(v) for v in re.search(r"first failing pixel \((-?\d+), (-?\d+)\)", str(err)).groups())


def windows(w, h):
    out = [(0, 0, w, h), (w - 1, h - 1, 1, 1), (-3, -2, 5, 4), (w // 3, h // 3, max(1, w // 2), max(1, h // 2)), (w + 40, -30, 7, 5)]
    return out


SIZES = [(1, 1), (1, 9), (9, 1), (23, 17), (97, 61)]
LENSES = {"null": None, "tsai": TSAI, "tsai_k3": TSAI_K3}


@pytest.mark.parametrize("lens", list(LENSES))
@pytest.mark.parametrize("w,h", SIZES, ids=lambda s: str(s))
def test_float_matrix(vwb, w, h, lens):
    for k, (interp, edge) in enumerate([(i, e) for i in (BILINEAR, BICUBIC, NEAREST) for e in (ZERO, CONSTANT)]):
        cams = rig(10 * k + w + h, w, h, LENSES[lens], TSAI, pitch=(1.0, 0.01, 4.0)[k % 3], frame=k % 2 == 1)
        epis = oe.epipolar(*cams)
        img = image(w, h, k + w)
        for win in windows(w, h):
            check(vwb, img, cams[0], epis[0], win, interp, edge, label=(interp, edge), variants=((k % 2 == 0, k % 3, False),))
        check(vwb, img, cams[1], epis[1], (0, 0, w, h), interp, edge, label=("right", interp, edge))
        # a Tsai destination (camera_transform is general): back from the epipolar camera into the source camera
        check(vwb, img, epis[0], dict(cams[0]), (0, 0, w, h), interp, edge, variants=((True, 0, False),), label=("inverse", interp, edge))


@pytest.mark.parametrize("edge", [ZERO, CONSTANT, VALUE], ids=["zero", "constant", "value"])
@pytest.mark.parametrize("w,h", SIZES, ids=lambda s: str(s))
def test_masked_matrix(vwb, w, h, edge):
    for k, invalid in enumerate((0.0, 0.1, 0.5, 1.0)):
        cams = rig(100 + 7 * k + w, w, h, (None, TSAI, TSAI_K3, TSAI)[k], None, pitch=(1.0, 0.5)[k % 2], frame=k == 2)
        epis = oe.epipolar(*cams)
        img = image(w, h, 50 + k, masked=True, invalid=invalid)
        ev = ((0.0, 0.0), (3.25, 1.0), (-1.0, 0.0), (np.nan, 1.0))[k]
        for win in windows(w, h):
            check(vwb, img, cams[0], epis[0], win, BILINEAR, edge, ev, variants=((k % 2 == 1, 2 * (k % 2), False),), label=(invalid, edge))
        check(vwb, img, cams[0], epis[0], (0, 0, w, h), BILINEAR, edge, ev, label=(invalid, edge, "all paths"))


def test_integral_points(vwb):
    """a destination equal to the source maps many pixels exactly onto themselves (about 38 % here): the interpolations'
    integral shortcuts, where a masked valid word becomes 0 / 1"""
    cam = ot.camera(fu=20, fv=20, cu=8, cv=6)
    for masked in (False, True):
        img = image(16, 12, 3, masked=masked, invalid=0.3)
        for interp in ((BILINEAR,) if masked else (BILINEAR, BICUBIC, NEAREST)):
            want = check(vwb, img, cam, cam, (0, 0, 16, 12), interp, ZERO)
            if masked:
                assert set(np.unique(want[..., 1])) <= {0.0, 1.0}


def test_8192(vwb):
    """an 8192^2 image, Tsai source into its epipolar camera, bilinear: the whole device result against oracle strips (each
    output pixel depends only on its own coordinates)"""
    import torch
    n = 8192
    cams = rig(8192, n, n, TSAI, None)
    epi = oe.epipolar(*cams)[0]
    rng = np.random.default_rng(1)
    img = (rng.random((n, n), dtype=np.float32) * 255).astype(np.float32)
    got = vwb.camera_transform(torch.from_numpy(img).cuda(), api_cam(vwb, cams[0]), api_cam(vwb, epi)).cpu().numpy()
    for y0 in (0, 4090, n - 12):
        want = oe.camera_transform(img, cams[0], epi, (0, y0, n, 12))
        assert same32(got[y0:y0 + 12], want), y0
    assert np.count_nonzero(got) > 0.5 * n * n


@pytest.mark.parametrize("rois", [((0, 0, 97, 61), (0, 0, 97, 61)), ((0, 0, 120, 40), (0, 0, 33, 90)), ((0, 0, 1, 1), (0, 0, 1, 1)),
                                  ((3, 4, 50, 20), (0, 0, 64, 64))], ids=["square", "non_square", "one_pixel", "offset"])
def test_resize(vwb, rois):
    for k, lenses in enumerate(((None, None), (TSAI, TSAI_K3), (TSAI_K3, None))):
        cams = rig(300 + k, 97, 61, *lenses, pitch=(1.0, 0.02, 1.0)[k], frame=k == 1)
        epis = oe.epipolar(*cams)
        want = oe.resize_epipolar(*cams, *epis, *rois)
        e1, e2, s1, s2 = vwb.resize_epipolar_cameras_to_fit(*(api_cam(vwb, c) for c in cams + list(epis)), *rois)
        assert cam_bits(oe.from_pinhole(e1._struct()), want[0]) and cam_bits(oe.from_pinhole(e2._struct()), want[1]), (k, rois)
        assert (s1, s2) == want[2:], (k, rois, s1, s2, want[2:])
        # the engine's own epipolar cameras give the same
        g1, g2 = vwb.epipolar(*(api_cam(vwb, c) for c in cams))
        assert vwb.resize_epipolar_cameras_to_fit(api_cam(vwb, cams[0]), api_cam(vwb, cams[1]), g1, g2, *rois)[2:] == want[2:]


def test_point_to_pixel_error(vwb):
    """a strongly distorted Tsai source and a window far outside its image: PointToPixelErr naming the oracle's first failing
    pixel, from the host and the device; the resize of such a ROI fails the same way"""
    import torch
    src = ot.camera(fu=300, fv=300, cu=320, cv=240, tsai=STRONG)
    dst = ot.camera(fu=300, fv=300, cu=320, cv=240)
    win = (100, 200, 900, 60)
    _, fail = oe.camera_reverse_window(src, dst, win)
    assert fail is not None
    img = image(640, 480, 1)
    for x in (img, torch.from_numpy(img).cuda()):
        with pytest.raises(vwb.PointToPixelErr) as e:
            vwb.camera_transform(x, api_cam(vwb, src), api_cam(vwb, dst), bbox=(100, 200, 1000, 260))
        assert "Projection into pinhole camera is inaccurate" in str(e.value)
        assert failing_pixel(e.value) == tuple(fail), (str(e.value), fail)
    # inside the image the same cameras work
    check(vwb, img, src, dst, (250, 180, 140, 120), BILINEAR, ZERO, variants=((True, 0, False),))
    with pytest.raises(oe.PointToPixelErr):
        oe.transformed_bbox_fast(dst, src, (0, 0, 2000, 1500))
    with pytest.raises(vwb.PointToPixelErr):
        vwb.resize_epipolar_cameras_to_fit(api_cam(vwb, dst), api_cam(vwb, dst), api_cam(vwb, src), api_cam(vwb, src), (0, 0, 2000, 1500),
                                           (0, 0, 10, 10))


# Traced in a process of its own, so that its profiler sessions neither depend on nor add to the ones of the rest of the suite.
TRACE_SCRIPT = """
import numpy as np, torch
import visionworkbench_b200 as v
from kernel_trace import KernelTrace


class K8Trace(KernelTrace):
    def hot(self):
        return {n for n in self.raw if "k8_" in n}


torch.cuda.init()
c0 = v.PinholeModel((0, 0, 0), np.eye(3), 300, 300, 150, 100, distortion_model=v.TsaiLensDistortion((-0.12, 0.03, 1e-3, -2e-3, 0)))
c1 = v.PinholeModel((1, 0, 0), np.eye(3), 300, 300, 150, 100)
e0, e1 = v.epipolar(c0, c1)
gray, masked = torch.rand(200, 300, device="cuda"), torch.rand(200, 300, 2, device="cuda")
cases = [(0, i, e, lambda i=i, e=e: v.camera_transform(gray, c0, e0, interp=i, edge=e)) for i in (0, 1, 2) for e in (0, 1)]
cases += [(1, 0, e, lambda e=e: v.camera_transform(masked, c0, e0, edge=e, edge_value=(1.0, 1.0))) for e in (0, 1, 2)]
cases += [(2, 0, 0, lambda: v.resize_epipolar_cameras_to_fit(c0, c1, e0, e1, (0, 0, 300, 200), (0, 0, 300, 200)))]
for m, i, e, fn in cases:
    fn()
    tr = K8Trace()
    tr.run(fn)
    print("CASE", m, i, e, "|".join(sorted(set(tr.raw))))
"""


def test_kernel_trace():
    """gray cases ran k8_warp_kernel<2, interp, edge>, masked ones k8_warp_kernel<3, 0, edge>, the resize two
    k8_camera_bbox_kernel passes, and nothing else of K8"""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here]), PYTHONNOUSERSITE="1")
    r = subprocess.run([sys.executable, "-c", TRACE_SCRIPT], cwd=here, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    cases = [ln.split(" ", 4)[1:] for ln in r.stdout.splitlines() if ln.startswith("CASE ")]
    assert len(cases) == 10, r.stdout
    for m, interp, edge, names in cases:
        k8 = {n for n in names.split("|") if "k8_" in n}
        if m == "2":
            assert k8 and all("k8_camera_bbox_kernel" in n for n in k8), names
            continue
        want = re.compile(rf"k8_warp_kernel<\(?(int\)?)?{2 + int(m)}, \(?(int\)?)?{interp}, \(?(int\)?)?{edge}>")
        assert len(k8) == 1 and want.search(next(iter(k8))), (m, interp, edge, names)


# ---- end to end ------------------------------------------------------------------------------------------------------------

def tsai_undistort_np(x, y, k, iters=30):
    """Newton's method on the normalised Tsai model, vectorised (rendering only; not the reference's loop)"""
    k1, k2, p1, p2, k3 = k
    u, v = x.copy(), y.copy()
    for _ in range(iters):
        r2 = u * u + v * v
        rd = 1 + k1 * r2 + k2 * r2 * r2 + k3 * r2 ** 3
        fx = u * rd + 2 * p1 * u * v + p2 * (r2 + 2 * u * u) - x
        fy = v * rd + p1 * (r2 + 2 * v * v) + 2 * p2 * u * v - y
        a = k1 + 2 * k2 * r2 + 3 * k3 * r2 * r2
        j00 = rd + 2 * u * u * a + 2 * p1 * v + 6 * p2 * u
        j01 = 2 * u * v * a + 2 * p1 * u + 2 * p2 * v
        j10 = 2 * u * v * a + 2 * p1 * u + 2 * p2 * v
        j11 = rd + 2 * v * v * a + 6 * p1 * v + 2 * p2 * u
        det = j00 * j11 - j01 * j10
        u, v = u - (j11 * fx - j01 * fy) / det, v - (j00 * fy - j10 * fx) / det
    return u, v


def render_plane(cam, w, h, texture, cell, plane):
    """ray-cast every pixel centre of a Tsai pinhole camera (identity frame) onto the plane z = a + b x and sample the texture"""
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    xn, yn = (xs - cam["cu"]) / cam["fu"], (ys - cam["cv"]) / cam["fv"]
    un, vn = tsai_undistort_np(xn, yn, cam["tsai"])
    R = np.asarray(cam["rotation"])
    d = np.stack([un, vn, np.ones_like(un)], -1) @ R.T                # world direction R (u, v, 1) (pixel_to_vector, unnormalised)
    C = np.asarray(cam["center"])
    a, b = plane
    t = (a + b * C[0] - C[2]) / (d[..., 2] - b * d[..., 0])
    X, Y = C[0] + t * d[..., 0], C[1] + t * d[..., 1]
    return ndimage.map_coordinates(texture, [Y / cell + texture.shape[0] / 2, X / cell + texture.shape[1] / 2], order=1).astype(np.float32)


def test_end_to_end_plane(vwb):
    """two Tsai cameras over a textured plane z = 10 + 0.05 x: after epipolar rectification the correlator needs only +-2 rows
    of vertical search; at least 95 % of the valid pixels have |dy| <= 1, and at least 95 % of the triangulated points lie
    within 0.4 (4 % of the range; half a pixel of disparity is 0.25) of the plane"""
    w, h = 320, 240
    rng = np.random.default_rng(2024)
    texture = ndimage.gaussian_filter(rng.random((800, 800)), 1.2) * 255
    plane = (10.0, 0.05)
    cams = []
    for k, centre in enumerate(((0.0, 0.0, 0.0), (0.5, 0.02, 0.01))):
        R = Rotation.from_rotvec(rng.normal(0, 0.02, 3)).as_matrix()
        cams.append(ot.camera(center=centre, rotation=R, fu=400.0, fv=402.0, cu=160.0 + k, cv=120.0 - k, tsai=(TSAI, TSAI_K3)[k]))
    imgs = [render_plane(c, w, h, texture, 0.02, plane) for c in cams]
    masked = []
    for im in imgs:
        m = np.ones((h, w, 2), np.float32)
        m[..., 0] = im
        masked.append(m)
    c0, c1 = (api_cam(vwb, c) for c in cams)
    e0, e1 = vwb.epipolar(c0, c1)
    e0, e1, s0, s1 = vwb.resize_epipolar_cameras_to_fit(c0, c1, e0, e1, (0, 0, w, h), (0, 0, w, h))
    L, R = vwb.epipolar_transformed_images(c0, c1, e0, e1, masked[0], masked[1], s0, s1, (0.0, 0.0))
    assert L.shape == (s0[1], s0[0], 2) and R.shape == (s1[1], s1[0], 2)
    lm, rm = (np.where(x[..., 1] != 0, 255, 0).astype(np.uint8) for x in (L, R))
    view = vwb.pyramid_correlate(np.ascontiguousarray(L[..., 0]), np.ascontiguousarray(R[..., 0]), lm, rm, vwb.PREFILTER_NONE, 0.0,
                                 (-40, -2, 0, 2), (9, 9), vwb.ABSOLUTE_DIFFERENCE, 0, 0.0, 2.0, 0, 0, 2)
    d = view.rasterize(None, (0, 0, s0[0], s0[1]))
    valid = d[..., 2] != 0
    assert valid.mean() > 0.4, valid.mean()
    assert np.mean(np.abs(d[..., 1][valid]) <= 1) >= 0.95
    xyz = vwb.stereo_triangulate(d, e0, e1)
    p = xyz[valid]
    p = p[np.any(p != 0, axis=1)]
    err = np.abs(p[:, 2] - (plane[0] + plane[1] * p[:, 0]))
    assert len(p) > 0.3 * s0[0] * s0[1] and np.mean(err <= 0.4) >= 0.95, (len(p), np.percentile(err, [50, 95]))
