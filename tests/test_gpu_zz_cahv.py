"""CAHV / CAHVOR cameras on the device against the oracle (oracle/vw_cahv_oracle.c), bit for bit (floats and doubles as raw
bits, NaN equal to NaN): camera_transform from CAHV and CAHVOR sources (rover cameras, the reference's cahvor.txt camera,
strongly distorted and left-handed ones; the transform runs only the source's point_to_pixel, which has no Newton loop) into
linearized and epipolar CAHV cameras, every float interpolation x
edge and PixelMask<float> bilinear x zero / constant / value edges with 0-100 % invalid pixels, 1 x 1 to 4096^2 and 8192^2,
whole / interior / edge / 1-pixel / outside windows, host and device rasters with padded pitches on the NULL and a side stream;
stereo_triangulate on both disparity types and stereo_model_points with its statistics for each CAHV / CAHVOR pairing,
with CAHVOR rays that reach every Newton exit (converged, deriv <= 0 and 20 passes); which
kernel each call ran; and the chain linearize -> epipolar -> epipolar_transformed_cahv_images -> pyramid_correlate ->
stereo_triangulate on a rendered plane."""
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy import ndimage

from cahv_reference import CAHVOR_TXT, rover
from oracle import cahv as oc

pytestmark = pytest.mark.gpu
BILINEAR, BICUBIC, NEAREST = 0, 1, 2
ZERO, CONSTANT, VALUE = 0, 1, 2


@pytest.fixture(scope="module")
def vwb():
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "GPU tests need a CUDA device: the engine has no CPU path"
    return v


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    u = np.uint32 if a.dtype == np.float32 else np.uint64
    return bool(np.all((a.view(u) == b.view(u)) | (np.isnan(a) & np.isnan(b))))


def api(vwb, c):
    if c["model"] == 1:
        return vwb.CAHVModel(c["C"], c["A"], c["H"], c["V"])
    return vwb.CAHVORModel(c["C"], c["A"], c["H"], c["V"], c["O"], c["R"])


def image(w, h, seed, masked=False, invalid=0.0):
    rng = np.random.default_rng(seed)
    v = (rng.random((h, w)) * 200 - 50).astype(np.float32)
    if not masked:
        return v
    m = np.empty((h, w, 2), np.float32)
    m[..., 0] = v
    m[..., 1] = (rng.random((h, w)) >= invalid).astype(np.float32)
    if h * w > 4:
        m[0, 0, 0] = np.nan
    return m


def sources(w, h):
    """(name, src camera, dst CAHV camera) over a w x h image"""
    out = []
    src = rover(1, w, h)
    out.append(("cahvor-linearized", src, oc.linearize(src, (w, h), (w, h))))
    cahv = rover(2, w, h, model=1)
    e0, _ = oc.epipolar(cahv, rover(3, w, h, center=(0.0, 0.5, 0.0), model=1))
    out.append(("cahv-epipolar", cahv, e0))
    strong = rover(4, w, h, r=(0.0, -3.0, -4.0))                     # deriv <= 0 towards the corners
    out.append(("cahvor-strong", strong, oc.linearize(rover(4, w, h), (w, h), (w, h))))
    wild = rover(5, w, h, r=(-0.9, 40.0, 900.0), left=True)          # left-handed, slow or no convergence
    out.append(("cahvor-wild", wild, dict(oc.linearize(rover(5, w, h), (w, h), (w, h)), C=wild["C"])))
    out.append(("cahvor-txt", CAHVOR_TXT, oc.linearize(CAHVOR_TXT, (w, h), (w, h))))
    return out


def run(vwb, img, src, dst, win, interp, edge, dev=False, pad=0, side=False, ev=(0.0, 0.0)):
    import torch
    x0, y0, ow, oh = win
    masked = img.ndim == 3
    ref = oc.camera_transform(img, src, dst, x0, y0, ow, oh, interp, edge, ev)
    arg = img
    if dev:
        t = torch.from_numpy(img).cuda()
        if pad:
            big = torch.zeros((img.shape[0], img.shape[1] + pad) + img.shape[2:], dtype=torch.float32, device="cuda")
            big[:, :img.shape[1]] = t
            t = big[:, :img.shape[1]]
        arg = t
    kw = dict(bbox=(x0, y0, x0 + ow, y0 + oh), edge=edge, interp=interp, edge_value=ev if masked else None)
    if side:
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            got = vwb.camera_transform(arg, api(vwb, src), api(vwb, dst), **kw)
        s.synchronize()
    else:
        got = vwb.camera_transform(arg, api(vwb, src), api(vwb, dst), **kw)
    if dev:
        got = got.cpu().numpy()
    assert same(got, ref), (win, interp, edge, dev, pad, side)


@pytest.mark.parametrize("w,h", [(1, 1), (7, 5), (64, 48), (333, 257)])
def test_camera_transform_every_mode(vwb, w, h):
    for k, (name, src, dst) in enumerate(sources(w, h)):
        gray = image(w, h, 10 + k)
        for interp in (BILINEAR, BICUBIC, NEAREST):
            for edge in (ZERO, CONSTANT):
                run(vwb, gray, src, dst, (0, 0, w, h), interp, edge)
        for inv in (0.0, 0.3, 1.0):
            m = image(w, h, 20 + k, True, inv)
            for edge in (ZERO, CONSTANT, VALUE):
                run(vwb, m, src, dst, (0, 0, w, h), BILINEAR, edge, ev=(7.5, 1.0))


def test_camera_transform_windows_and_staging(vwb):
    w, h = 300, 200
    for name, src, dst in sources(w, h):
        gray, m = image(w, h, 3), image(w, h, 4, True, 0.2)
        for win in ((0, 0, w, h), (40, 30, 100, 80), (w - 10, h - 7, 30, 20), (123, 45, 1, 1), (-500, -400, 60, 50), (5000, 10, 20, 20)):
            run(vwb, gray, src, dst, win, BICUBIC, CONSTANT)
            run(vwb, m, src, dst, win, BILINEAR, VALUE, ev=(1.0, 0.0))
        for dev, pad, side in ((True, 0, False), (True, 3, False), (True, 5, True), (False, 0, True)):
            run(vwb, gray, src, dst, (10, 10, 200, 150), BILINEAR, ZERO, dev, pad, side)
            run(vwb, m, src, dst, (10, 10, 200, 150), BILINEAR, ZERO, dev, pad, side)


@pytest.mark.parametrize("n", [1024, 4096])
def test_camera_transform_large(vwb, n):
    src = rover(7, n, n)
    dst = oc.linearize(src, (n, n), (n, n))
    run(vwb, image(n, n, 8, True, 0.1), src, dst, (0, 0, n, n), BILINEAR, VALUE, dev=True, ev=(0.0, 0.0))
    run(vwb, image(n, n, 9), rover(9, n, n, model=1), oc.epipolar(rover(9, n, n, model=1), rover(10, n, n, (0, 1, 0), model=1))[0],
        (0, 0, n, n), BICUBIC, CONSTANT, dev=True)


def test_camera_transform_8192(vwb):
    n = 8192
    src = rover(11, n, n)
    dst = oc.linearize(src, (n, n), (n, n))
    run(vwb, image(n, n, 12, True, 0.05), src, dst, (0, 0, n, n), BILINEAR, ZERO, dev=True)


def test_center_mismatch_is_logic_err(vwb):
    src = rover(1, 50, 40)
    dst = dict(oc.linearize(src, (50, 40), (50, 40)), C=(0.0, 0.0, 1e-9))
    with pytest.raises(vwb.LogicErr):
        vwb.camera_transform(image(50, 40, 1), api(vwb, src), api(vwb, dst))
    with pytest.raises(vwb.NoImplErr):                               # a CAHVOR destination
        vwb.camera_transform(image(50, 40, 1), api(vwb, dst), api(vwb, src))


def disparity(w, h, seed, kind, invalid=0.1):
    rng = np.random.default_rng(seed)
    if kind == "i32":
        d = np.zeros((h, w, 3), np.int32)
        d[..., 0] = rng.integers(-40, -5, (h, w))
        d[..., 1] = rng.integers(-2, 3, (h, w))
    else:
        d = np.zeros((h, w, 3), np.float32)
        d[..., 0] = rng.uniform(-40, -5, (h, w))
        d[..., 1] = rng.uniform(-2, 2, (h, w))
    d[..., 2] = rng.random((h, w)) >= invalid
    if kind == "f32" and h * w > 8:
        d[0, 1, 0] = np.nan
        d[0, 2, :2] = -1e8
    return d


def pairs(w, h):
    out = []
    for m0 in (1, 2):
        for m1 in (1, 2):
            out.append((rover(30 + m0, w, h, model=m0), rover(40 + m1, w, h, center=(0.0, -0.4, 0.01), model=m1)))
    out.append((rover(50, w, h, r=(0.0, -3.0, -4.0)), rover(51, w, h, center=(0.0, -0.4, 0.0), r=(-0.9, 40.0, 900.0), left=True)))
    return out


@pytest.mark.parametrize("w,h", [(1, 1), (37, 29), (500, 300)])
def test_stereo_triangulate(vwb, w, h):
    import torch
    for c0, c1 in pairs(w, h):
        for kind in ("i32", "f32"):
            d = disparity(w, h, w + h, kind)
            for win in ((0, 0, w, h), (w // 3, h // 4, max(1, w // 2), max(1, h // 2)), (w - 1, h - 1, 1, 1)):
                x0, y0, ow, oh = win
                ref, it = oc.stereo_triangulate(d, c0, c1, x0, y0, ow, oh)
                got = vwb.stereo_triangulate(d, api(vwb, c0), api(vwb, c1), bbox=(x0, y0, x0 + ow, y0 + oh))
                assert same(got, ref), (kind, win)
                s = vwb.last_triangulation_stats()
                assert s["cahvor_iterations"] == it and s["tsai_iterations"] == 0, (kind, win, s)
            got = vwb.stereo_triangulate(torch.from_numpy(d).cuda(), api(vwb, c0), api(vwb, c1), angle_tol=1e-3).cpu().numpy()
            assert same(got, oc.stereo_triangulate(d, c0, c1, angle_tol=1e-3)[0])


@pytest.mark.parametrize("w,h", [(3, 2), (400, 256)])
def test_stereo_model_points(vwb, w, h):
    for c0, c1 in pairs(w, h):
        d = disparity(w, h, 7, "f32", 0.25)
        xyz, err, st, it = oc.stereo_model(d, c0, c1)
        gx, ge = vwb.stereo_model_points(d, api(vwb, c0), api(vwb, c1))
        assert same(gx, xyz) and same(ge, err)
        s = vwb.last_triangulation_stats()
        assert (s["points"], s["divergent"], s["max_error"], s["cahvor_iterations"]) == (st[0], st[1], st[2], it)
        assert abs(s["error_sum"] - st[3]) <= 1e-12 * max(1.0, abs(st[3])) and s["tsai_iterations"] == 0


TRACE_SCRIPT = """
import numpy as np, torch
import visionworkbench_b200 as v
from kernel_trace import KernelTrace
from cahv_reference import rover
from oracle import cahv as oc


class Trace(KernelTrace):
    def hot(self):
        return {n for n in self.raw if "k8_" in n or "k10_" in n}


def api(c):
    return v.CAHVModel(c["C"], c["A"], c["H"], c["V"]) if c["model"] == 1 else v.CAHVORModel(c["C"], c["A"], c["H"], c["V"], c["O"], c["R"])


torch.cuda.init()
src = rover(1, 300, 200)
dst = oc.linearize(src, (300, 200), (300, 200))
gray, masked = torch.rand(200, 300, device="cuda"), torch.rand(200, 300, 2, device="cuda")
di = torch.zeros(200, 300, 3, dtype=torch.int32, device="cuda")
df = torch.zeros(200, 300, 3, dtype=torch.float32, device="cuda")
di[..., 2] = 1
df[..., 2] = 1
c1 = rover(2, 300, 200, center=(0, -0.4, 0))
cases = [("w4", i, e, lambda i=i, e=e: v.camera_transform(gray, api(src), api(dst), interp=i, edge=e)) for i in (0, 1, 2) for e in (0, 1)]
cases += [("w5", 0, e, lambda e=e: v.camera_transform(masked, api(src), api(dst), edge=e, edge_value=(1.0, 1.0))) for e in (0, 1, 2)]
cases += [("ti", 0, 0, lambda: v.stereo_triangulate(di, api(src), api(c1))), ("tf", 0, 0, lambda: v.stereo_triangulate(df, api(src), api(c1))),
          ("tm", 0, 0, lambda: v.stereo_model_points(df, api(src), api(c1)))]
for m, i, e, fn in cases:
    fn()
    tr = Trace()
    tr.run(fn)
    print("CASE", m, i, e, "|".join(sorted(set(tr.raw))))
"""


def test_kernel_trace_per_camera_type():
    """each CAHV call ran only its own instantiation: k8_warp_kernel<4, interp, edge> / <5, 0, edge>, and
    k10_triangulate_kernel<CahvCam, T, MODEL, true>"""
    import re
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here]), PYTHONNOUSERSITE="1")
    r = subprocess.run([sys.executable, "-c", TRACE_SCRIPT], cwd=here, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    cases = [ln.split(" ", 4)[1:] for ln in r.stdout.splitlines() if ln.startswith("CASE ")]
    assert len(cases) == 12, r.stdout
    n = r"\(?(int\)?)?"
    for m, interp, edge, names in cases:
        hot = {x for x in names.split("|") if "k8_" in x or "k10_" in x}
        assert len(hot) == 1, (m, names)
        name = next(iter(hot))
        if m in ("w4", "w5"):
            assert re.search(rf"k8_warp_kernel<{n}{m[1]}, {n}{interp}, {n}{edge}>", name), (m, interp, edge, name)
        else:
            t = {"ti": "vwb200_dispi", "tf": "DispF", "tm": "DispF"}[m]
            model = "true" if m == "tm" else "false"
            assert "k10_triangulate_kernel<" in name, (m, name)
            args = name.split("<", 1)[1].split(">")[0].replace("(bool)1", "true").replace("(bool)0", "false").split(", ")
            assert args[0].endswith("CahvCam") and args[1].endswith(t) and args[2:] == [model, "true"], (m, name)


# ---- end to end ------------------------------------------------------------------------------------------------------------

def rays(c, w, h):
    """CAHVOR pixel_to_vector of every pixel, vectorised (rendering only; not the reference's evaluation order)"""
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    A, H, V = (np.asarray(c[k]) for k in "AHV")
    rr = np.cross(V[None, None] - ys[..., None] * A, H[None, None] - xs[..., None] * A)
    rr /= np.linalg.norm(rr, axis=-1, keepdims=True)
    if np.dot(np.cross(V, H), A) < 0:
        rr = -rr
    O, R = np.asarray(c["O"]), np.asarray(c["R"])
    om = rr @ O
    lam = rr - om[..., None] * O
    tau = np.sum(lam * lam, -1) / (om * om)
    k1, k3, k5 = 1 + R[0], R[1] * tau, R[2] * tau * tau
    u = 1 - (R[0] + k3 + k5)
    for _ in range(20):
        u = u - (((k5 * u * u + k3) * u * u + k1) * u - 1) / ((5 * k5 * u * u + 3 * k3) * u * u + k1)
    d = rr - (1 - u)[..., None] * lam
    return d / np.linalg.norm(d, axis=-1, keepdims=True)


def test_end_to_end_plane(vwb):
    """a CAHVOR pair 0.5 apart over the textured plane x = 10 + 0.05 y: linearize, epipolar, rectify, correlate with +-2 rows of
    vertical search and triangulate through the epipolar CAHV cameras.  The correlator's disparities are integers, so a point's
    depth is known to one pixel of disparity, z^2 / (f * baseline) (about 0.7 here): at least 95 % of the valid points lie
    within that of the plane, and at least 95 % of the valid pixels have |dy| <= 1"""
    w, h = 320, 240
    rng = np.random.default_rng(2026)
    texture = ndimage.gaussian_filter(rng.random((800, 800)), 1.2) * 255
    a, b = 10.0, 0.05
    cams = [rover(60, w, h, tilt=0.01), rover(61, w, h, center=(0.0, 0.5, 0.0), tilt=0.01)]
    imgs = []
    for c in cams:
        d = rays(c, w, h)
        C = np.asarray(c["C"])
        t = (a + b * C[1] - C[0]) / (d[..., 0] - b * d[..., 1])
        Y, Z = C[1] + t * d[..., 1], C[2] + t * d[..., 2]
        im = ndimage.map_coordinates(texture, [Z / 0.02 + 400, Y / 0.02 + 400], order=1).astype(np.float32)
        m = np.ones((h, w, 2), np.float32)
        m[..., 0] = im
        imgs.append(m)
    api_c = [api(vwb, c) for c in cams]
    lin = [vwb.linearize_camera(c, (w, h), (w, h)) for c in api_c]
    e0, e1 = vwb.epipolar(lin[0], lin[1])
    L, R = vwb.epipolar_transformed_cahv_images(api_c[0], api_c[1], e0, e1, imgs[0], imgs[1], (0.0, 0.0))
    lm, rm = (np.where(x[..., 1] != 0, 255, 0).astype(np.uint8) for x in (L, R))
    view = vwb.pyramid_correlate(np.ascontiguousarray(L[..., 0]), np.ascontiguousarray(R[..., 0]), lm, rm, vwb.PREFILTER_NONE, 0.0,
                                 (-40, -2, 40, 2), (9, 9), vwb.ABSOLUTE_DIFFERENCE, 0, 0.0, 2.0, 0, 0, 2)
    d = view.rasterize(None, (0, 0, w, h))
    valid = d[..., 2] != 0
    assert valid.mean() > 0.4, valid.mean()
    assert np.mean(np.abs(d[..., 1][valid]) <= 1) >= 0.95
    xyz = vwb.stereo_triangulate(d, e0, e1)
    p = xyz[valid]
    p = p[np.any(p != 0, axis=1)]
    f = np.linalg.norm(np.cross(e0.A, e0.H))
    tol = a * a / (f * 0.5)
    err = p[:, 0] - (a + b * p[:, 1])
    print("signed depth error percentiles (1, 50, 99):", np.percentile(err, [1, 50, 99]), "tolerance", tol)
    assert np.mean(np.abs(err) <= tol) >= 0.95, np.percentile(np.abs(err), [50, 90, 95, 99])
