"""Stereo triangulation on the device (k10_triangulate.cu) against the oracle (oracle/vw_triangulate_oracle.c), bit for bit
(raw bits, NaN == NaN): stereo_triangulate (both pixel types) over whole, interior, edge and 1-pixel windows, StereoModel on a
float disparity with its statistics, universe radius in and out of place; NULL and TSAI lenses (with and without k3, at
strengths that reach every Newton-Raphson exit), pixel pitches, non-identity u, v, w frames, arbitrary rotations, angle_tol 0
and custom, identical cameras, 0-100 % invalid pixels, 1 x 1 to 4096^2, host and device rasters with padded pitches on NULL
and side streams, a view's output and a fill_holes_grass output as input, and which K10 kernel each case ran."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import triangulate as ot
from test_oracle_triangulate import STRONG, TSAI, TSAI_K3, api_cam, disparity_field, rig, same

pytestmark = pytest.mark.gpu
I32, F32 = 0, 1


@pytest.fixture(scope="module")
def vwb():
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "GPU tests need a CUDA device: the engine has no CPU path"
    return v


def windows(w, h):
    out = [None, (w - 1, h - 1, 1, 1), (0, 0, 1, 1)]
    if w > 6 and h > 6:
        out += [(2, 3, w - 5, h - 6), (0, h // 2, w, h - h // 2), (w // 3, 0, w - w // 3, 3)]
    return out


def check_a(vwb, d, cams, window=None, angle_tol=0.0, devs=(False, True), label=""):
    import torch
    want = ot.stereo_triangulate(d, cams[0], cams[1], window, angle_tol)
    a, b = api_cam(vwb, cams[0]), api_cam(vwb, cams[1])
    x0, y0, ow, oh = window if window is not None else (0, 0, d.shape[1], d.shape[0])
    for dev in devs:
        x = torch.from_numpy(d).cuda() if dev else d
        got = vwb.stereo_triangulate(x, a, b, (x0, y0, x0 + ow, y0 + oh), angle_tol)
        got = got.cpu().numpy() if dev else got
        assert same(got, want), (label, window, dev, np.argwhere(np.any(~eq(got, want), axis=2))[:5])
    return want


def check_b(vwb, d, cams, angle_tol=0.0, devs=(False, True), label=""):
    import torch
    xyz, err, st = ot.stereo_model(d, cams[0], cams[1], angle_tol)
    a, b = api_cam(vwb, cams[0]), api_cam(vwb, cams[1])
    for dev in devs:
        x = torch.from_numpy(d).cuda() if dev else d
        gx, ge = vwb.stereo_model_points(x, a, b, angle_tol)
        gx, ge = (gx.cpu().numpy(), ge.cpu().numpy()) if dev else (gx, ge)
        assert same(gx, xyz) and same(ge, err), (label, dev)
        s = vwb.last_triangulation_stats()
        assert (s["points"], s["divergent"], s["max_error"]) == (st["points"], st["divergent"], st["max_error"]), (s, st)
        assert abs(s["error_sum"] - st["error_sum"]) <= 1e-12 * abs(st["error_sum"]), (s, st)
        tsai = any(c.get("tsai") is not None for c in cams) and st["points"] + st["divergent"] > 0
        assert (s["tsai_iterations"] > 0) == tsai and s["cahvor_iterations"] == 0, (s, label)
    return xyz, err, st


def eq(a, b):
    return (a == b) | (np.isnan(a) & np.isnan(b))


SIZES = [(1, 1), (1, 9), (9, 1), (23, 17), (50, 147)]
LENSES = {"null": None, "tsai": TSAI, "tsai_k3": TSAI_K3}


@pytest.mark.parametrize("lens", list(LENSES))
@pytest.mark.parametrize("w,h", SIZES, ids=lambda s: str(s))
def test_density_matrix(vwb, w, h, lens):
    for k, dens in enumerate([0.0, 0.1, 0.5, 0.9, 1.0]):
        cams = rig(100 + 7 * k + w, LENSES[lens], pitch=(1.0, 0.01, 7.5)[k % 3], frame=k % 2 == 1)
        for dtype in (np.int32, np.float32):
            d = disparity_field(w, h, dens, dtype, 10 * k + h)
            for win in windows(w, h):
                check_a(vwb, d, cams, win, devs=(True,) if win else (False, True), label=(dens, dtype))
        check_b(vwb, disparity_field(w, h, dens, np.float32, 10 * k + h), cams, devs=(True,), label=dens)


def test_float_versus_double_right_pixel(vwb):
    """form (b) adds the disparity to the column in float, form (a) in double: at x = 1000 with d = 0.1 they differ"""
    cams = [dict(c, cu=1000.0) for c in rig(7, None)]
    d = disparity_field(1200, 3, 0.0, np.float32, 8)
    d[..., 0] = np.float32(-20.1)
    a = check_a(vwb, d, cams)
    b, _, _ = check_b(vwb, d, cams)
    assert not same(a, b)


def test_nr_exits(vwb):
    """each exit of the Tsai Newton-Raphson loop, reached and matched"""
    cams = [dict(c, fu=300.0, fv=300.0, cu=320.0, cv=240.0) for c in rig(11, STRONG)]
    d = disparity_field(64, 48, 0.05, np.float32, 12, lo=-600, hi=600)
    d[5, 5, :2] = (np.inf, 0)                                     # NaN |F|
    d[6, 6] = (614, 234, 1)                                       # right pixel (620, 240): normalised (1, 0), det 0
    check_a(vwb, d, cams)
    check_b(vwb, d, cams)
    exits = set()
    cam = cams[1]
    for j in range(48):
        for i in range(64):
            if d[j, i, 2]:
                exits.add(ot.tsai_undistort(cam, ((i + float(d[j, i, 0])) * cam["pixel_pitch"], (j + float(d[j, i, 1])) * cam["pixel_pitch"]))[1])
    assert exits >= {0, 1, 2, 3}, exits
    tiny = dict(cams[1], fu=1e-301)                              # fu < 1e-300: HUGE_VAL
    check_a(vwb, d, (cams[0], tiny))
    check_b(vwb, d, (cams[0], tiny))


def test_special_values(vwb):
    cams = rig(21, TSAI, pitch=0.5)
    d = disparity_field(40, 30, 0.2, np.float32, 22)
    rng = np.random.default_rng(23)
    pick = rng.random((30, 40)) < 0.3
    d[..., :2][pick] = rng.choice(np.array([np.nan, np.inf, -np.inf, -0.0, 1e30, -1e30, 3.5], np.float32), (pick.sum(), 2))
    d[0, 0] = (-1e8, -1e8, 1)                                    # invalid_pixel() on the right
    d[2, 3, 2] = np.nan                                          # a NaN valid word is valid
    d[2, 4, 2] = -0.0                                            # and -0.0 invalid
    for win in (None, (5, 5, 20, 20)):
        check_a(vwb, d, cams, win)
    check_b(vwb, d, cams)
    di = disparity_field(40, 30, 0.2, np.int32, 24)
    di[..., :2] = rng.integers(-(1 << 31), (1 << 31) - 1, (30, 40, 2))
    di[0, 0] = (-100000000, -100000000, 1)
    check_a(vwb, di, cams)


@pytest.mark.parametrize("tol", [0.0, 0.03, 1e-9])
def test_angle_tol_and_identical_cameras(vwb, tol):
    cams = rig(31, TSAI_K3, frame=True)
    d = disparity_field(60, 40, 0.1, np.float32, 32)
    check_a(vwb, d, cams, angle_tol=tol)
    xyz, _, st = check_b(vwb, d, cams, angle_tol=tol)
    same_cams = (cams[0], cams[0])
    check_a(vwb, d, same_cams, angle_tol=tol)                   # distinct rays from one center meet at the center
    d[..., :2] = 0                                               # one ray twice: parallel, every point (0, 0, 0)
    xyz = check_a(vwb, d, same_cams, angle_tol=tol)
    xyz2, err, st = check_b(vwb, d, same_cams, angle_tol=tol)
    assert (xyz == 0).all() and (xyz2 == 0).all() and (err == 0).all() and st["points"] == (d[..., 2] != 0).sum()


def test_4096(vwb):
    import torch
    n = 4096
    cams = rig(41, TSAI)
    d = disparity_field(n, n, 0.1, np.float32, 42)
    x = torch.from_numpy(d).cuda()
    xyz, err, st = ot.stereo_model(d, cams[0], cams[1])
    gx, ge = vwb.stereo_model_points(x, api_cam(vwb, cams[0]), api_cam(vwb, cams[1]))
    assert same(gx.cpu().numpy(), xyz) and same(ge.cpu().numpy(), err)
    s = vwb.last_triangulation_stats()
    assert (s["points"], s["divergent"], s["max_error"]) == (st["points"], st["divergent"], st["max_error"]), (s, st)
    assert abs(s["error_sum"] - st["error_sum"]) <= 1e-12 * abs(st["error_sum"]), (s, st)
    assert s["tsai_iterations"] > 0 and s["cahvor_iterations"] == 0, s
    got = vwb.stereo_triangulate(x, api_cam(vwb, cams[0]), api_cam(vwb, cams[1]), (1000, 1500, 2024, 2524)).cpu().numpy()
    assert same(got, ot.stereo_triangulate(d, cams[0], cams[1], (1000, 1500, 1024, 1024)))
    pts = torch.from_numpy(xyz).cuda()
    want = ot.universe_radius(xyz, (0.1, -0.2, 3.0), 2.0, 40.0)
    got, rej, tot = vwb.universe_radius(pts, (0.1, -0.2, 3.0), 2.0, 40.0, out=pts)
    assert same(got.cpu().numpy(), want[0]) and (rej, tot) == want[1:] and 0 < rej < tot


def test_view_and_inpaint_output_as_input(vwb):
    """the float disparity the correlation view rasterises, and fill_holes_grass's output, as the triangulation's input"""
    import torch
    from visionworkbench_b200.synth import make_pair
    search, kernel = (-12, -8, 12, 8), (7, 7)
    left, right, lm, rm, _ = make_pair(256, 224, search, seed=5)
    view = vwb.pyramid_correlate(left, right, lm, rm, vwb.PREFILTER_NONE, 0.0, search, kernel, vwb.ABSOLUTE_DIFFERENCE,
                                 0, 0.0, 2.0, 0, 3, 3)
    disp = view.rasterize(None, (0, 0, 256, 224))
    disp = np.ascontiguousarray(disp.cpu().numpy() if hasattr(disp, "cpu") else np.asarray(disp))
    assert disp.dtype == np.float32 and (disp[..., 2] == 0).any()
    cams = rig(51, TSAI)
    check_a(vwb, disp, cams)
    check_b(vwb, disp, cams)
    filled = vwb.fill_holes_grass(torch.from_numpy(disp).cuda(), 10).cpu().numpy()
    check_a(vwb, filled, cams, (10, 20, 200, 150))
    check_b(vwb, filled, cams)


def test_universe_radius_cases(vwb):
    import torch
    rng = np.random.default_rng(61)
    p = rng.uniform(-10, 10, (37, 29, 3))
    p[0, 0] = (0.0, -0.0, 0.0)
    p[0, 1] = (-0.0, -0.0, -0.0)
    p[0, 2] = (np.nan, 1.0, 2.0)
    p[0, 3] = (np.inf, 0.0, 0.0)
    p[0, 4] = (1.0, 2.0, 2.0)                                    # dist exactly 3 from the origin
    for near, far in ((0.0, ot.DBL_MAX), (3.0, 3.0), (0.0, 0.0), (2.0, 9.0), (3.0, 0.0 + 1e300)):
        want, r, t = ot.universe_radius(p, (0, 0, 0), near, far)
        for dev in (False, True):
            x = torch.from_numpy(p.copy()).cuda() if dev else p.copy()
            got, gr, gt = vwb.universe_radius(x, (0, 0, 0), near, far)
            g = got.cpu().numpy() if dev else got
            assert same(g, want) and (gr, gt) == (r, t), (near, far, dev)
            got, gr, gt = vwb.universe_radius(x, (0, 0, 0), near, far, out=x)          # in place
            g = got.cpu().numpy() if dev else got
            assert got is x and same(g, want) and (gr, gt) == (r, t), (near, far, dev)
    for near, far in ((-1.0, 2.0), (3.0, 2.0), (np.nan, 2.0)):
        with pytest.raises(vwb.ArgumentErr):
            vwb.universe_radius(p, (0, 0, 0), near, far)


# ---- the C ABI: host and device rasters, padded pitches, NULL and side streams --------------------------------------------------
def padded(a, pad, fill):
    b = np.full(a.shape[:1] + (a.shape[1] + pad,) + a.shape[2:], fill, a.dtype)
    b[:, :a.shape[1]] = a
    return b


@pytest.mark.parametrize("dtype", [np.int32, np.float32], ids=["i32", "f32"])
def test_abi_places_pitches_streams(vwb, dtype):
    import torch
    L = vwb.lib()
    w, h = 41, 37
    cams = rig(71, TSAI, pitch=2.0, frame=True)
    c1, c2 = (vwb.api.Pinhole.from_buffer_copy(ot.pinhole(c)) for c in cams)
    d = disparity_field(w, h, 0.1, dtype, 72)
    side = torch.cuda.Stream()
    ptype = I32 if dtype == np.int32 else F32
    ptr = lambda a: a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data  # noqa: E731
    for dev in (0, 1):
        for ipad, opad in ((0, 0), (3, 0), (0, 5), (2, 1)):
            for stream in ((None, side) if dev else (None,)):
                sp = C.c_void_p(stream.cuda_stream) if stream is not None else None
                src = padded(d, ipad, -77)
                for win in ((0, 0, w, h), (5, 4, 30, 25)):
                    x0, y0, ow, oh = win
                    want = ot.stereo_triangulate(d, cams[0], cams[1], win)
                    dst = padded(np.zeros((oh, ow, 3)), opad, -77.0)
                    s, o = (torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda()) if dev else (src, dst)
                    torch.cuda.synchronize()
                    rc = L.vwb200_stereo_triangulate(ptype, ptr(s), w, h, w + ipad, x0, y0, ow, oh, C.byref(c1), C.byref(c2), 0.0, ptr(o),
                                                     ow + opad, dev, sp)
                    assert rc == 0, L.vwb200_last_error()
                    if stream is not None:
                        stream.synchronize()
                    out = o.cpu().numpy() if dev else o
                    assert same(np.ascontiguousarray(out[:, :ow]), want) and (out[:, ow:] == -77).all(), (win, dev, ipad, opad)
                if dtype != np.float32:
                    continue
                xyz, err, _ = ot.stereo_model(d, cams[0], cams[1])
                dx, de = padded(np.zeros((h, w, 3)), opad, -77.0), padded(np.zeros((h, w)), ipad, -77.0)
                s, ox, oe = (torch.from_numpy(src).cuda(), torch.from_numpy(dx).cuda(), torch.from_numpy(de).cuda()) if dev else (src, dx, de)
                torch.cuda.synchronize()
                rc = L.vwb200_stereo_model_points(ptr(s), w, h, w + ipad, C.byref(c1), C.byref(c2), 0.0, ptr(ox), w + opad, ptr(oe), w + ipad,
                                                  dev, sp)
                assert rc == 0, L.vwb200_last_error()
                if stream is not None:
                    stream.synchronize()
                gx, ge = (ox.cpu().numpy(), oe.cpu().numpy()) if dev else (ox, oe)
                assert same(np.ascontiguousarray(gx[:, :w]), xyz) and same(np.ascontiguousarray(ge[:, :w]), err), (dev, ipad, opad)
                assert (gx[:, w:] == -77).all() and (ge[:, w:] == -77).all()
                pts = padded(xyz, ipad, -77.0)
                want, r, t = ot.universe_radius(xyz, (0.5, 0.5, 10.0), 1.0, 30.0)
                p = torch.from_numpy(pts).cuda() if dev else pts
                rej, tot = C.c_longlong(), C.c_longlong()
                org = np.array([0.5, 0.5, 10.0])
                rc = L.vwb200_universe_radius(ptr(p), w, h, w + ipad, org.ctypes.data, 1.0, 30.0, ptr(p), w + ipad, C.byref(rej), C.byref(tot), dev, sp)
                assert rc == 0, L.vwb200_last_error()
                if stream is not None:
                    stream.synchronize()
                g = p.cpu().numpy() if dev else p
                assert same(np.ascontiguousarray(g[:, :w]), want) and (rej.value, tot.value) == (r, t) and (g[:, w:] == -77).all()


# Traced in a process of its own, so that its profiler sessions neither depend on nor add to the ones of the rest of the suite.
TRACE_SCRIPT = """
import numpy as np, torch
import visionworkbench_b200 as v
from kernel_trace import KernelTrace
from test_oracle_triangulate import TSAI, api_cam, disparity_field, rig


class K10Trace(KernelTrace):
    def hot(self):
        return {n for n in self.raw if "k10_" in n}


torch.cuda.init()
for lens in ("null", "tsai"):
    cams = rig(3, None if lens == "null" else TSAI)
    a, b = api_cam(v, cams[0]), api_cam(v, cams[1])
    for dt in (np.int32, np.float32):
        d = torch.from_numpy(disparity_field(64, 32, 0.1, dt, 4)).cuda()
        forms = [("a", lambda: v.stereo_triangulate(d, a, b))]
        if dt == np.float32:
            forms.append(("b", lambda: v.stereo_model_points(d, a, b)))
        for form, fn in forms:
            fn()
            tr = K10Trace()
            tr.run(fn)
            print("CASE", lens, np.dtype(dt).name, form, "|".join(sorted(set(tr.raw))))
pts = torch.zeros(16, 16, 3, dtype=torch.float64, device="cuda")
fn = lambda: v.universe_radius(pts, (0, 0, 0), 1.0, 2.0, out=pts)
fn()
tr = K10Trace()
tr.run(fn)
print("CASE", "-", "float64", "c", "|".join(sorted(set(tr.raw))))
"""


def test_kernel_trace_per_camera_type():
    """each form and lens runs its own k10_triangulate_kernel<TriCam, T, MODEL, TSAI> instantiation; universe radius its kernel"""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here]), PYTHONNOUSERSITE="1")
    r = subprocess.run([sys.executable, "-c", TRACE_SCRIPT], cwd=here, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    cases = [ln.split(" ", 4)[1:] for ln in r.stdout.splitlines() if ln.startswith("CASE ")]
    assert len(cases) == 7, r.stdout
    for lens, dt, form, names in cases:
        k10 = {n for n in names.split("|") if "k10_" in n}
        assert len(k10) == 1, (lens, dt, form, names)
        name = k10.pop()
        if form == "c":
            assert "k10_universe_radius_kernel" in name, name
            continue
        assert "k10_triangulate_kernel" in name, name
        args = name.split("<", 1)[1].split(">")[0].replace("(bool)1", "true").replace("(bool)0", "false").split(", ")
        assert args[0].endswith("TriCam") and args[1].endswith("vwb200_dispi" if dt == "int32" else "DispF"), name
        assert args[2:] == ["true" if form == "b" else "false", "true" if lens == "tsai" else "false"], name
