"""The triangulation oracle (oracle/vw_triangulate_oracle.c) against the reference's known-answer tests, the independent numpy
restatement in triangulate_reference.py, bit for bit (raw bits, NaN == NaN), and two sanity properties (the inverse camera
transform inverts the camera matrix; a triangulated point projects back onto both pixels)."""
import numpy as np
import pytest

from oracle import triangulate as ot
import triangulate_reference as ref

TSAI = (-0.12, 0.03, 1e-3, -2e-3, 0.0)
TSAI_K3 = (-0.12, 0.03, 1e-3, -2e-3, 0.01)
STRONG = (-1.0 / 3.0, 0.0, 0.0, 0.0, 0.0)       # J = 0 at normalised (1, 0); no inverse beyond r = 1


def bits(a):
    a = np.ascontiguousarray(a, np.float64)
    b = a.view(np.uint64).copy()
    b[np.isnan(a)] = 0x7ff8000000000000
    return b


def same(a, b):
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


def rotation(rng):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


def rig(seed, tsai, pitch=1.0, frame=False):
    """a rectified pair of seeded cameras, f in pixels about 500, the second one baseline 0.5 .. 2 to the right of the first
    along the image rows; frame=True: a non-identity signed-permutation u, v, w frame"""
    rng = np.random.default_rng(seed)
    R = rotation(rng)
    if frame:
        u, v, w = (0.0, 1.0, 0.0), (0.0, 0.0, -1.0), (-1.0, 0.0, 0.0)
    else:
        u, v, w = (1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0)
    f = float(rng.uniform(400, 700))
    c1 = rng.uniform(-5, 5, 3)
    axis = R @ np.array(u)                                        # the world direction of the image rows
    c2 = c1 + rng.uniform(0.5, 2.0) * axis
    cu, cv = float(rng.uniform(20, 40)) * pitch, float(rng.uniform(10, 30)) * pitch
    return [ot.camera(center=tuple(c), rotation=R, fu=f * pitch, fv=f * 1.01 * pitch, cu=cu, cv=cv, u=u, v=v, w=w, pixel_pitch=pitch, tsai=tsai)
            for c in (c1, c2)]


def disparity_field(w, h, density, dtype, seed, lo=-60, hi=-8):
    """a disparity with children in [lo, hi) (invalid pixels keep theirs) and the given fraction of invalid pixels"""
    rng = np.random.default_rng(seed)
    d = np.zeros((h, w, 3), dtype)
    if dtype == np.int32:
        d[..., 0] = rng.integers(lo, hi, (h, w))
        d[..., 1] = rng.integers(-2, 3, (h, w))
    else:
        d[..., 0] = rng.uniform(lo, hi, (h, w)).astype(np.float32)
        d[..., 1] = rng.uniform(-2, 2, (h, w)).astype(np.float32)
    d[..., 2] = (rng.random((h, w)) >= density).astype(dtype)
    return d


def api_cam(vwb, cam):
    """the engine's PinholeModel of an oracle camera dict"""
    t = cam.get("tsai")
    return vwb.PinholeModel(cam["center"], cam["rotation"], cam["fu"], cam["fv"], cam["cu"], cam["cv"], cam["u"], cam["v"], cam["w"],
                            None if t is None else vwb.TsaiLensDistortion(t), cam["pixel_pitch"])


# ---- the reference's known-answer tests ---------------------------------------------------------------------------------
def test_kat_pinhole_stereo():
    """TestStereoModel.cxx:35-58: the point (2, 0, 1) seen by unit cameras at the origin and at (1, 0, 0) projects to (2, 0)
    and (1, 0)"""
    pt, _ = ot.triangulate(ot.camera(), ot.camera(center=(1, 0, 0)), (2, 0), (1, 0))
    assert np.allclose(pt, (2, 0, 1), atol=1e-6)


@pytest.mark.parametrize("masked", [True, False], ids=["PixelMaskVec2", "Vec2"])
def test_kat_stereo_view(masked):
    """TestStereoModel.cxx:99-203, the four StereoView cases: Vec2 and Float fed as valid PixelMask<Vector2f> (same arithmetic)"""
    c1, c2 = ot.camera(cu=1), ot.camera(center=(1, 0, 0), cu=1)
    d = np.zeros((1, 3, 3), np.float32)
    d[0, :, 2] = 1
    d[0, :, 0] = (-1.5, -1, -1.3)
    if masked:
        d[0, 0, 2] = 0
    pc = ot.stereo_triangulate(d, c1, c2)
    first = (0, 0, 0) if masked else (-0.666, 0, 0.666)
    assert np.allclose(pc[0, 0], first, atol=1e-2) and (pc[0, 0] == 0).all() == masked
    assert np.allclose(pc[0, 1], (0, 0, 1), atol=1e-2)
    assert np.allclose(pc[0, 2], (0.769, 0, 0.769), atol=1e-2)


# ---- bit for bit against the numpy restatement ----------------------------------------------------------------------------
def test_lu_inverse():
    rng = np.random.default_rng(1)
    mats = [rng.normal(size=(3, 3)) for _ in range(20)] + [np.diag([2.0, 3.0, 5.0]), np.array([[0, 1, 0], [0, 0, 1], [1, 0, 0.0]]),
                                                            np.array([[1e-300, 2, 3], [4, 5, 6], [7, 8, 10.0]]), -np.eye(3)]
    for m in mats:
        assert same(ot.inverse3(m), np.array(ref.inverse(m))), m
    with pytest.raises(ot.OracleError):
        ot.inverse3(np.array([[1, 2, 3], [2, 4, 6], [1, 1, 1.0]]))
    with pytest.raises(ZeroDivisionError):
        ref.inverse([[1, 2, 3], [2, 4, 6], [1, 1, 1.0]])


def test_camera_inverse_and_frames():
    for seed in range(6):
        for cam in rig(seed, None, pitch=(1.0, 0.02)[seed % 2], frame=seed % 3 == 0):
            assert same(ot.camera_inverse(cam), np.array(ref.camera_inverse(cam)))
    bad = ot.camera(u=(1, 0, 0), v=(0, 1, 0), w=(0, 0, 1.01))
    with pytest.raises(ot.OracleError) as e:
        ot.camera_inverse(bad)
    assert e.value.rc == -3
    ok = ot.camera(u=(1, 0, 0), v=(0, 1, 0), w=(0, 0, 1.0009))                 # within 0.001 of a unit norm
    ot.camera_inverse(ok)
    with pytest.raises(ot.OracleError) as e:
        ot.camera_inverse(ot.camera(fu=0.0))                                      # singular K
    assert e.value.rc == -2


def test_tsai_exits():
    """each exit of the Newton-Raphson loop: converged, |det| < 1e-6, NaN |F|, 19 iterations, fu < 1e-300"""
    strong = ot.camera(fu=300, fv=300, cu=320, cv=240, tsai=STRONG)
    rng = np.random.default_rng(2)
    pts = [tuple(p) for p in rng.uniform(-400, 1100, (300, 2))] + [(620.0, 240.0), (np.inf, 3.0), (-np.inf, np.inf), (1e300, 240.0)]
    seen = set()
    for cam in (strong, ot.camera(fu=300, fv=300, cu=320, cv=240, tsai=TSAI_K3)):
        for p in pts:
            got, ex, _ = ot.tsai_undistort(cam, p)
            want = ref.tsai_undistort(cam, np.float64(p[0]), np.float64(p[1]))
            assert same(got, np.array(want[:2])) and ex == want[2], (p, ex, want)
            seen.add(ex)
    tiny = ot.camera(fu=1e-301, fv=300, cu=320, cv=240, tsai=TSAI)
    got, ex, _ = ot.tsai_undistort(tiny, (5.0, 6.0))
    assert ex == 4 and (got == np.inf).all()
    assert seen >= {0, 1, 2, 3}, seen
    assert ot.tsai_undistort(strong, (620.0, 240.0))[1] == 1


def _cases():
    """(disparity, cameras) pairs covering both lenses, pitches, frames, and the special disparities"""
    out = []
    for k, lens in enumerate((None, TSAI, TSAI_K3, STRONG)):
        cams = rig(10 + k, lens, pitch=(1.0, 0.05, 3.0, 1.0)[k], frame=k % 2 == 1)
        d = disparity_field(9, 7, 0.2, np.float32, 20 + k)
        d[0, 0, :2] = (-1e8, -1e8)                               # invalid_pixel() on the right
        d[0, 1, :2] = (np.nan, 1)
        d[0, 2, :2] = (np.inf, 0)
        d[0, 3, :2] = (-np.inf, 2)
        d[0, 4, :2] = (-0.0, -0.0)
        d[0, 5, :2] = (3e38, -3e38)
        d[1, 0, :2] = (0.1, 0.0)                                 # in front / behind: reflection
        d[1, 1, :2] = (5.0, 0.0)
        d[1, 2:5, 2] = 1
        out.append((d, cams))
    return out


@pytest.mark.parametrize("k", range(4))
def test_forms_match_restatement(k):
    d, cams = _cases()[k]
    for tol in (0.0, 0.02):
        assert same(ot.stereo_triangulate(d, cams[0], cams[1], None, tol), ref.stereo_triangulate(d, cams, None, tol))
        assert same(ot.stereo_triangulate(d, cams[0], cams[1], (2, 1, 5, 4), tol), ref.stereo_triangulate(d, cams, (2, 1, 5, 4), tol))
        xyz, err, st = ot.stereo_model(d, cams[0], cams[1], tol)
        rx, re, rst = ref.stereo_model(d, cams, tol)
        assert same(xyz, rx) and same(err, re) and st == rst, (st, rst)
    di = d.copy()
    di[..., :2] = np.clip(np.nan_to_num(di[..., :2], nan=0.0), -2e9, 2e9)
    di = di.astype(np.int32)
    assert same(ot.stereo_triangulate(di, cams[0], cams[1]), ref.stereo_triangulate(di, cams))


def test_float_versus_double_right_pixel():
    """StereoModel's image form sums x + d in float, StereoView in double: at x = 1001 they differ in the last bits"""
    cams = [dict(c, cu=1000.0) for c in rig(30, None)]
    d = disparity_field(1003, 1, 0.0, np.float32, 31)
    d[..., 0] = np.float32(-20.1)
    a = ot.stereo_triangulate(d, cams[0], cams[1], (1000, 0, 3, 1))
    b = ot.stereo_model(d, cams[0], cams[1])[0][:, 1000:]
    assert not same(a, b)
    assert same(a, ref.stereo_triangulate(d, cams, (1000, 0, 3, 1)))


def test_parallel_tolerance():
    """1 - dot(d0, d1) >= tol at and around tol, identical cameras, and NaN directions counting as parallel"""
    cams = rig(40, None)
    inv = [ref.camera_inverse(c) for c in cams]
    d0 = ref.pixel_to_vector(cams[0], inv[0], 5.0, 5.0)
    d1 = ref.pixel_to_vector(cams[1], inv[1], 0.0, 5.0)
    tol = float(np.float64(1) - ref.dot(d0, d1))
    for t in (tol, np.nextafter(tol, 0), np.nextafter(tol, 1)):
        got, _ = ot.triangulate(cams[0], cams[1], (5, 5), (0, 5), t)
        want, _ = ref.triangulate(cams, inv, ((5, 5), (0, 5)), t)
        assert same(got, np.array(want)) and ((got == 0).all() == (t > tol)), t
    got, err = ot.triangulate(cams[0], cams[0], (5, 5), (5, 5))
    assert (got == 0).all() and (err == 0).all()


def test_universe_radius_cases():
    rng = np.random.default_rng(50)
    p = rng.uniform(-10, 10, (9, 11, 3))
    p[0, 0] = (0.0, -0.0, 0.0)
    p[0, 1] = (-0.0, -0.0, -0.0)
    p[0, 2] = (np.nan, 1, 2)
    p[0, 3] = (1.0, 2.0, 2.0)
    p[0, 4] = (np.inf, 0, 0)
    for near, far in ((0.0, ot.DBL_MAX), (3.0, 3.0), (0.0, 0.0), (2.0, 9.0)):
        got = ot.universe_radius(p, (0, 0, 0), near, far)
        want = ref.universe_radius(p, (0, 0, 0), near, far)
        assert same(got[0], want[0]) and got[1:] == want[1:], (near, far)
        assert same(got[0][0, 2], p[0, 2]) and not np.signbit(got[0][0, 1]).any()
    assert ot.universe_radius(p, (0, 0, 0), 3.0, 3.0)[0][0, 3].tolist() == [1.0, 2.0, 2.0]
    for near, far in ((-1.0, 2.0), (3.0, 2.0), (np.nan, 1.0)):
        with pytest.raises(ot.OracleError):
            ot.universe_radius(p, (0, 0, 0), near, far)


# ---- sanity properties ----------------------------------------------------------------------------------------------------
def test_inverse_inverts_camera_matrix():
    for seed in range(5):
        for cam in rig(60 + seed, None, pitch=(1.0, 0.1)[seed % 2], frame=seed % 2 == 0):
            uvw = np.array([cam["u"], cam["v"], cam["w"]])
            K = np.array([[cam["fu"], 0, cam["cu"]], [0, cam["fv"], cam["cv"]], [0, 0, 1]])
            assert np.allclose(ot.camera_inverse(cam) @ (K @ uvw @ np.asarray(cam["rotation"]).T), np.eye(3), atol=1e-12, rtol=0)


def _project(cam, pt):
    """pixel of a world point: q = uvw * R^T * (X - C), normalised, distorted (Tsai), through K, over the pixel pitch"""
    uvw = np.array([cam["u"], cam["v"], cam["w"]])
    q = uvw @ np.asarray(cam["rotation"]).T @ (np.asarray(pt) - np.array(cam["center"]))
    x, y = q[0] / q[2], q[1] / q[2]
    if cam["tsai"] is not None:
        x, y = (float(v) for v in ref.tsai_norm(np.float64(x), np.float64(y), cam["tsai"]))
    return np.array([x * cam["fu"] + cam["cu"], y * cam["fv"] + cam["cv"]]) / cam["pixel_pitch"]


def test_projection_round_trip():
    """a world point projected into both cameras triangulates to a point that projects back onto both pixels"""
    for lens in (None, TSAI, TSAI_K3):
        cams = rig(70, lens, pitch=0.5, frame=True)
        for px, depth in (((10.0, 12.0), 8.0), ((30.0, 5.0), 20.0), ((-40.0, 50.0), 5.0)):
            world = np.array(cams[0]["center"]) + depth * ot.pixel_to_vector(dict(cams[0], tsai=None), px)
            pix = [_project(c, world) for c in cams]
            pt, _ = ot.triangulate(cams[0], cams[1], pix[0], pix[1])
            for cam, want in zip(cams, pix):
                assert np.allclose(_project(cam, pt), want, atol=1e-6, rtol=0), (lens, px)
