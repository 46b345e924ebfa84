"""The epipolar-rectification oracle (oracle/vw_epipolar_oracle.c): pinned by
the known answers of Camera/tests/TestPinholeModel.cxx, checked bit for bit against the numpy restatement in
epipolar_reference.py (every quaternion branch, the check's sum retry and its failure, HUGE_VAL, BBox2f's NaN skip and float
rounding, size truncation), and by two sanity checks: epipolar cameras put a 3-D point on one row, and forward inverts
reverse."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import epipolar_reference as ref
from oracle import epipolar as oe
from oracle import triangulate as ot
from oracle import warp as ow
from test_oracle_triangulate import STRONG, TSAI, TSAI_K3, rotation, same


def tilted_rig(seed, lens0, lens1=None, pitch=1.0, frame=False):
    """two cameras about 1 apart, looking roughly along +z with seeded small tilts, f about 500 px over a 640 x 480 image;
    frame=True gives the first a non-identity u, v, w frame"""
    rng = np.random.default_rng(seed)
    cams = []
    for k, lens in enumerate((lens0, lens1)):
        R = Rotation.from_rotvec(rng.normal(0, 0.05, 3)).as_matrix()
        f = rng.uniform(480, 520) * pitch
        c = ot.camera(center=(k * rng.uniform(0.8, 1.2), rng.normal(0, 0.05), rng.normal(0, 0.05)), rotation=R, fu=f, fv=f * rng.uniform(0.98, 1.02),
                      cu=(320 + rng.normal(0, 5)) * pitch, cv=(240 + rng.normal(0, 5)) * pitch, pixel_pitch=pitch, tsai=lens)
        if frame and k == 0:
            c.update(u=(0.0, 1.0, 0.0), v=(1.0, 0.0, 0.0), w=(0.0, 0.0, -1.0), rotation=R @ np.diag([1.0, 1.0, -1.0]) @ np.array([[0, 1, 0], [1, 0, 0], [0, 0, 1.0]]))
        cams.append(c)
    return cams


def cam_bits(a, b):
    keys = ("center", "rotation", "fu", "fv", "cu", "cv", "u", "v", "w", "pixel_pitch")
    return all(same(np.asarray(a[k], np.float64), np.asarray(b[k], np.float64)) for k in keys) and a["tsai"] is None and b["tsai"] is None


# ---- known answers (TestPinholeModel.cxx) -------------------------------------------------------------------------------

def test_kat_standard_construct():
    cam = ot.camera(fu=500, fv=500, cu=500, cv=500)
    for pt, px in (((0, 0, 10), (500, 500)), ((-10, 0, 10), (0, 500)), ((10, 0, 10), (1000, 500)), ((0, -10, 10), (500, 0)),
                   ((0, 10, 10), (500, 1000))):
        assert np.allclose(oe.point_to_pixel(cam, pt), px, atol=1e-6)


def test_kat_coordinate_frame():
    cam = ot.camera(fu=500, fv=500, cu=500, cv=500, u=(0, 1, 0), v=(1, 0, 0), w=(0, 0, -1))
    for pt, px in (((0, 0, -10), (500, 500)), ((-10, 0, -10), (500, 0)), ((10, 0, -10), (500, 1000)), ((0, -10, -10), (0, 500)),
                   ((0, 10, -10), (1000, 500))):
        assert np.allclose(oe.point_to_pixel(cam, pt), px, atol=1e-5)


def test_kat_tsai_distortion():
    """distorted_coordinates(200, 200) of the test's lens (k3 = 0) is about (244.865, 244.395): the point whose undistorted
    pixel is (200, 200) projects there, and the check's undistortion takes it back"""
    cam = ot.camera(fu=500, fv=500, cu=500, cv=500, tsai=(-0.2805362343788147, 0.1062035113573074, -0.0001422458299202845, 0.00116333004552871, 0.0))
    px = oe.point_to_pixel(cam, (-0.6, -0.6, 1.0))
    assert np.allclose(px, (244.865, 244.395), atol=1e-3)
    und, _, _ = ot.tsai_undistort(cam, px)
    assert np.allclose(und, (200, 200), atol=1e-6)


def test_kat_projection_round_trip():
    """PinholeTest::projection_test: pixel_to_vector then point_to_pixel returns the pixel within 1e-6 over the image grid
    (the test's camera, its rotation euler (1.15, 0, -1.57) built here with scipy)"""
    R = Rotation.from_euler("xyz", (1.15, 0.0, -1.57)).as_matrix()
    cam = ot.camera(center=(-0.329, 0.065, -0.82), rotation=R, fu=605.320556640625, fv=606.3638305664062, cu=518.89208984375,
                    cv=387.5555114746094)
    for lens in (None, TSAI):
        c = dict(cam, tsai=lens)
        for x in range(10, 1037, 80):
            for y in range(10, 775, 80):
                d = ot.pixel_to_vector(c, (x, y))
                assert np.allclose(oe.point_to_pixel(c, d + np.array(c["center"])), (x, y), atol=1e-6)


# ---- the oracle against the numpy restatement, bit for bit ----------------------------------------------------------------

def test_quaternion_every_branch():
    rng = np.random.default_rng(3)
    mats = [rotation(rng) for _ in range(40)] + [np.eye(3), np.diag([1.0, -1, -1]), np.diag([-1.0, 1, -1]), np.diag([-1.0, -1, 1]),
                                                 Rotation.from_rotvec((0, 0, np.pi)).as_matrix(), Rotation.from_rotvec((np.pi, 0, 0)).as_matrix()]
    seen = set()
    for R in mats:
        got, b, _ = oe.quaternion_round_trip(R)
        want, wb = ref.quaternion_round_trip(R)
        assert b == wb and same(got, np.array(want)), R
        assert np.allclose(got, R, atol=1e-12)
        seen.add(b)
    assert seen == {0, 1, 2, 3}


@pytest.mark.parametrize("seed", range(8))
def test_epipolar_and_camera_matrix(seed):
    lenses = (None, TSAI, TSAI_K3, STRONG)
    cams = tilted_rig(seed, lenses[seed % 4], lenses[(seed + 1) % 4], pitch=(1.0, 0.01)[seed % 2], frame=seed % 3 == 0)
    e0, e1 = oe.epipolar(*cams)
    r0, r1 = ref.epipolar(*cams)
    assert cam_bits(e0, r0) and cam_bits(e1, r1)
    for c in cams + [e0, e1]:
        assert same(oe.camera_matrix(c), np.array(ref.camera_matrix(c)))


def test_epipolar_coincident_centers_give_nan():
    c = tilted_rig(1, None)
    e0, e1 = oe.epipolar(c[0], dict(c[1], center=c[0]["center"]))
    r0, _ = ref.epipolar(c[0], dict(c[1], center=c[0]["center"]))
    assert np.isnan(e0["rotation"]).all() and cam_bits(e0, r0)


def test_epipolar_rows_and_round_trip():
    """a 3-D point projects to the same row in both epipolar cameras (within 1e-9 px), and forward(reverse(p)) = p"""
    rng = np.random.default_rng(5)
    for seed in range(4):
        cams = tilted_rig(seed, TSAI, TSAI_K3)
        e0, e1 = oe.epipolar(*cams)
        for _ in range(30):
            X = np.array([rng.uniform(-3, 4), rng.uniform(-2, 2), rng.uniform(5, 30)])
            assert abs(oe.point_to_pixel(e0, X)[1] - oe.point_to_pixel(e1, X)[1]) < 1e-9
        for _ in range(30):
            p = rng.uniform((0, 0), (640, 480))
            q = oe.camera_reverse(cams[0], e0, p)
            assert np.allclose(oe.camera_forward(cams[0], e0, q), p, atol=1e-6)


def point_cases():
    """(camera, point) pairs: in front, behind (the check's sum retry), far off-axis through a strong lens (failure), fu below
    1e-300 (HUGE_VAL), NaN and infinite points"""
    rng = np.random.default_rng(7)
    out = []
    for lens in (None, TSAI, TSAI_K3, STRONG):
        cam = ot.camera(center=(0.1, -0.2, 0.3), rotation=rotation(rng), fu=300, fv=310, cu=320, cv=240, tsai=lens, pixel_pitch=1.0)
        for _ in range(25):
            out.append((cam, rng.normal(0, 1, 3) * (1, 1, 1) + rng.normal(0, 3, 3)))
        out += [(cam, (np.nan, 1.0, 2.0)), (cam, (np.inf, 0.0, 1.0)), (cam, cam["center"])]
    out.append((ot.camera(fu=1e-301, fv=5, tsai=TSAI), (0.1, 0.2, 1.0)))
    out.append((ot.camera(fu=300, fv=300, cu=320, cv=240, tsai=STRONG), (5.0, 0.0, 1.0)))
    return out


def test_point_to_pixel_matches_restatement():
    outcomes = {True: 0, False: 0}
    retried = 0
    for cam, X in point_cases():
        want, ok = ref.point_to_pixel(ref.Cam(cam), X)
        try:
            got = oe.point_to_pixel(cam, X)
            assert ok
        except oe.PointToPixelErr as e:
            assert not ok, (cam, X)
            got = e.where
        assert same(np.asarray(got), np.array(want)), (cam, X)
        outcomes[ok] += 1
        d = np.asarray(X, float) - np.asarray(cam["center"], float)
        retried += ok and np.dot(np.asarray(cam["rotation"]).T[2], d) < 0     # behind the camera: only the sum passes
    assert outcomes[True] > 20 and outcomes[False] > 5 and retried > 5, (outcomes, retried)
    with pytest.raises(oe.PointToPixelErr) as e:                    # fu < 1e-300: distorted_coordinates is HUGE_VAL
        oe.point_to_pixel(ot.camera(fu=1e-301, fv=5, tsai=TSAI), (0.1, 0.2, 1.0))
    assert np.isinf(e.value.where).all()


def test_bbox_fast_and_resize_match_restatement():
    for seed, lenses in enumerate(((None, None), (TSAI, TSAI_K3), (TSAI_K3, None))):
        cams = tilted_rig(20 + seed, *lenses, pitch=(1.0, 0.02, 1.0)[seed])
        epis = oe.epipolar(*cams)
        for roi in ((0, 0, 64, 48), (0, 0, 1, 1), (5, 7, 6, 40), (0, 0, 97, 13)):
            for c, e in zip(cams, epis):
                assert same(oe.transformed_bbox_fast(c, e, roi), np.array(ref.bbox_fast(ref.Cam(c), ref.Cam(e), roi), np.float32))
        for rois in (((0, 0, 64, 48), (0, 0, 64, 48)), ((0, 0, 50, 30), (0, 0, 20, 60)), ((0, 0, 1, 1), (0, 0, 1, 1))):
            got = oe.resize_epipolar(*cams, *epis, *rois)
            want = ref.resize(*cams, *epis, *rois)
            assert cam_bits(got[0], want[0]) and cam_bits(got[1], want[1]) and got[2:] == want[2:], rois


def test_bbox_float_rounding_nan_and_truncation():
    """BBox2f keeps float(point): the bounds are float32 roundings of the doubles; NaN coordinates are skipped; the sizes
    truncate toward zero"""
    cams = tilted_rig(31, TSAI, None)
    e0, _ = oe.epipolar(*cams)
    roi = (0, 0, 30, 20)
    bb = oe.transformed_bbox_fast(cams[0], e0, roi)
    pts = [oe.camera_forward(cams[0], e0, p) for p in [(x, 0) for x in range(30)] + [(x, 19) for x in range(30)] + [(0, y) for y in range(20)]
           + [(29, y) for y in range(20)]]
    pts = np.array(pts)
    assert np.array_equal(bb, np.array([pts[:, 0].min(), pts[:, 1].min(), pts[:, 0].max(), pts[:, 1].max()]).astype(np.float32))
    # NaN intrinsics: every projection is NaN, and the check fails on the first point
    nan_epi = dict(e0, cu=np.nan, cv=np.nan)
    with pytest.raises(oe.PointToPixelErr):
        oe.transformed_bbox_fast(cams[0], nan_epi, roi)
    _, _, s1, _ = oe.resize_epipolar(*cams, *oe.epipolar(*cams), (0, 0, 30, 20), (0, 0, 30, 20))
    _, _, r1, _ = ref.resize(*cams, *oe.epipolar(*cams), (0, 0, 30, 20), (0, 0, 30, 20))
    assert s1 == r1


def test_failure_reports_first_pixel():
    """a Tsai camera with strong distortion and a window far outside its image: the first failing pixel in row-major order"""
    src = ot.camera(fu=300, fv=300, cu=320, cv=240, tsai=STRONG)
    dst = ot.camera(fu=300, fv=300, cu=320, cv=240)
    _, fail = oe.camera_reverse_window(src, dst, (100, 200, 900, 60))
    assert fail is not None
    x, y = fail
    for j in range(200, y + 1):
        for i in range(100, 1000 if j < y else x):
            assert ref.reverse(ref.Cam(src), ref.Cam(dst), (i, j))[1], (i, j)
    assert not ref.reverse(ref.Cam(src), ref.Cam(dst), fail)[1]


def test_masked_bilinear_cases():
    """the masked interpolation at integral and fractional points, with NaN values and valid words 0, 1, 0.5 and NaN, against
    a scalar restatement of the PixelMask arithmetic"""
    rng = np.random.default_rng(9)
    img = np.zeros((5, 6, 2), np.float32)
    img[..., 0] = rng.normal(0, 10, (5, 6))
    img[..., 1] = rng.choice(np.array([0.0, 1.0, 0.5, np.nan], np.float32), (5, 6))
    img[2, 3, 0] = np.nan
    coords = np.array([(x, y) for x in np.arange(-1.5, 7, 0.75) for y in np.arange(-1.25, 6, 0.5)] + [(2.0, 3.0), (0.0, 0.0), (3.0, 2.0)])
    for edge, ev in ((ow.ZERO, (0, 0)), (ow.CONSTANT, (0, 0)), (oe.VALUE, (7.5, 1.0)), (oe.VALUE, (-2.0, 0.0))):
        got = oe.sample(img, ow.BILINEAR, edge, coords, ev)
        for (x, y), g in zip(coords, got):
            w = restated_masked(img, edge, ev, x, y)
            assert same(g.astype(np.float64), np.array(w, np.float32).astype(np.float64)), (edge, x, y, g, w)


def restated_masked(img, edge, ev, x, y):
    h, w = img.shape[:2]

    def at(i, j):
        if edge == ow.CONSTANT:
            return img[min(max(j, 0), h - 1), min(max(i, 0), w - 1)]
        if 0 <= i < w and 0 <= j < h:
            return img[j, i]
        return np.array((0, 0) if edge == ow.ZERO else ev, np.float32)

    F32 = np.float32
    xi, yi = int(np.floor(x)), int(np.floor(y))
    if xi == x and yi == y:
        p = at(xi, yi)
        return (p[0], F32(p[1] != 0))
    nx, ny = F32(x) - F32(xi), F32(y) - F32(yi)
    ps = [at(xi, yi), at(xi + 1, yi), at(xi, yi + 1), at(xi + 1, yi + 1)]
    with np.errstate(all="ignore"):
        r = (ps[0][0] * (F32(1) - nx) + ps[1][0] * nx) * (F32(1) - ny)
        row = ps[2][0] * (F32(1) - nx) + ps[3][0] * nx
        v = r + row * ny
    return (v, F32(all(p[1] != 0 for p in ps)))
