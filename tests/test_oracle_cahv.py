"""The CAHV / CAHVOR oracle (oracle/vw_cahv_oracle.c) pinned by the reference's known answers (TestCAHVModel.cxx
PinholeConversion, FakeEpipolarConversion and ForwardReverse; TestCAHVORModel.cxx ForwardReverse and the pixel part of
PointDerivatives), and equal bit for bit to the numpy restatement in cahv_reference.py on seeded and edge-case cameras: both
handednesses, every Newton exit, NaN / inf / -0.0 inputs, odd and even linearize_camera sizes."""
import numpy as np
import pytest

import cahv_reference as cr
from oracle import cahv as oc
from oracle import triangulate as ot

pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")


def same(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return a.shape == b.shape and bool(np.all((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))))


def same_cam(a, b):
    return a["model"] == b["model"] and all(same(a[k], b[k]) for k in ("CAHV" if a["model"] == 1 else "CAHVOR"))


def test_forward_reverse_kats():
    for c in (cr.FR_CAHV, cr.FR_CAHVOR):
        for i in range(100, 901, 100):
            for j in range(100, 901, 100):
                d = oc.pixel_to_vector(c, (i, j))[0]
                p = oc.point_to_pixel(c, np.asarray(c["C"]) + 30 * d)
                assert np.allclose(p, (i, j), atol=1e-2)


def test_point_derivatives_pixel_kat():
    """PointDerivatives' pixel part: point_to_pixel of the origin through the cahvor.txt camera with exact vectors, and
    get_point_derivatives' u, v restated (within the test's 1e-5)"""
    c = dict(cr.CAHVOR_TXT, A=tuple(np.array([1, 2, 3.0]) / np.sqrt(14)), O=tuple(np.array([2, 3, 4.0]) / np.sqrt(29)))
    ref = oc.point_to_pixel(c, (0.0, 0.0, 0.0))
    P, C, O, A, H, V, R = (np.asarray(x, float) for x in ((0, 0, 0), c["C"], c["O"], c["A"], c["H"], c["V"], c["R"]))
    xi = (P - C) @ O
    lam = P - C - xi * O
    tau = lam @ lam / (xi * xi)
    mu = R[0] + tau * (R[1] + tau * R[2])
    PPC = P + mu * lam - C
    assert np.allclose(ref, (PPC @ H / (PPC @ A), PPC @ V / (PPC @ A)), atol=1e-5)


def test_pinhole_conversion_kat():
    pose = np.array([[0.0665748562545205, -0.997208917590965, 0.0337959049552638], [0.992575027692545, 0.0627338358137274, -0.104207870361314],
                     [0.101796870854825, 0.0404825952867597, 0.993981165094699]])
    pin = ot.camera(center=(-57.315, 13.2, -106.947), rotation=pose, fu=421.0, fv=421.0, cu=0.0, cv=0.0, pixel_pitch=0.1)
    from oracle import epipolar as oe
    c = oc.from_pinhole(ot.pinhole(pin))
    for x in range(0, 10, 2):
        for y in range(0, 20, 4):
            for z in range(-5, 5, 3):
                assert np.allclose(oe.point_to_pixel(pin, (x, y, z)), oc.point_to_pixel(c, (x, y, z)), atol=1e-4)


def fake_epipolar_cameras():
    def model(f, px, C, A, Hv, Vv):
        fH, fV = f / px, f / px
        return {"model": 1, "C": C, "A": tuple(A), "H": tuple(fH * np.asarray(Hv)), "V": tuple(fV * np.asarray(Vv))}
    a1 = np.array([-1, 0, -1.0]) / np.sqrt(2)
    a2 = np.array([1, 0, -1.0]) / np.sqrt(2)
    return (model(2, 0.1, (30.0, 0.0, 30.0), a1, (0, 1, 0), np.cross(a1, (0, 1, 0))),
            model(2, 0.1, (-30.0, 0.0, 30.0), a2, (0, -1, 0), np.cross(a2, (0, -1, 0))))


def test_fake_epipolar_conversion_kat():
    ma, mb = fake_epipolar_cameras()
    ea, eb = oc.epipolar(ma, mb)
    rng = np.random.default_rng(0)
    for _ in range(100):
        pt = (rng.uniform(-15, 15), rng.uniform(-15, 15), 0.0)
        ia, ib = oc.point_to_pixel(ma, pt), oc.point_to_pixel(mb, pt)
        fa = oc.point_to_pixel(ea, oc.pixel_to_vector(ma, ia)[0] + np.asarray(ma["C"]))
        fb = oc.point_to_pixel(eb, oc.pixel_to_vector(mb, ib)[0] + np.asarray(mb["C"]))
        assert abs((fa - fb)[0] + 40) < 0.1 and abs((fa - fb)[1]) < 0.1


def cameras():
    out = [cr.FR_CAHV, cr.FR_CAHVOR, cr.CAHVOR_TXT]
    for s in range(6):
        out += [cr.rover(s, 640, 480, model=1), cr.rover(s, 640, 480), cr.rover(s, 641, 479, left=True), cr.rover(s, 64, 48, r=(0.0, -3.0, -4.0)),
                cr.rover(s, 64, 48, r=(-0.9, 40.0, 900.0), left=True)]
    return out


PIXELS = [(0, 0), (320, 240), (-0.0, 17.5), (639, 479), (-1e3, 2e3), (np.nan, 3.0), (np.inf, 1.0), (1e300, -1e300), (5.25, -0.0)]


def test_pixel_to_vector_and_point_to_pixel_match_restatement():
    exits = set()
    for c in cameras():
        for p in PIXELS:
            d, code, it = oc.pixel_to_vector(c, p)
            r, code2, it2 = cr.pixel_to_vector(c, p)
            assert same(d, r) and (code, it) == (code2, it2), (c, p)
            exits.add(code)
            for pt in (np.asarray(c["C"]) + 7 * np.asarray(d), (1.0, -2.0, 30.0), (-0.0, 0.0, 0.0), (np.inf, 0, 1)):
                assert same(oc.point_to_pixel(c, pt), cr.point_to_pixel(c, pt)), (c, pt)
    assert exits == {-1, 0, 1, 2}


def test_left_handed_camera_flips_the_ray():
    """negating H flips the handedness of V x H and so the sign of the unnormalised ray"""
    for c in (cr.FR_CAHV, dict(cr.FR_CAHV, H=tuple(-np.asarray(cr.FR_CAHV["H"])))):
        A, H, V = (np.asarray(c[k]) for k in "AHV")
        raw = np.cross(V - 20 * A, H - 10 * A)
        sign = -1.0 if np.cross(V, H) @ A < 0 else 1.0
        d = oc.pixel_to_vector(c, (10, 20))[0]
        assert same(d, cr.pixel_to_vector(c, (10, 20))[0]) and np.allclose(d, sign * raw / np.linalg.norm(raw), atol=1e-15)


@pytest.mark.parametrize("size", [(1, 1), (2, 2), (640, 480), (641, 479), (1023, 1024), (7, 3)])
def test_linearize_matches_restatement(size):
    for c in cameras():
        if c["model"] == 2:
            for out_size in (size, (size[0] + 1, size[1])):
                assert same_cam(oc.linearize(c, size, out_size), cr.linearize(c, size, out_size)), (c, size)


def test_epipolar_matches_restatement():
    cams = [c for c in cameras() if c["model"] == 1] + list(fake_epipolar_cameras())
    for a in cams:
        for b in cams:
            e = oc.epipolar(a, b)
            r = cr.epipolar(a, b)
            assert same_cam(e[0], r[0]) and same_cam(e[1], r[1])


def test_linearized_camera_is_undistorted_close_to_source():
    """the linearized camera sees the image centre where the CAHVOR camera does, within a pixel"""
    c = cr.rover(3, 1024, 768)
    lin = oc.linearize(c, (1024, 768), (1024, 768))
    d = oc.pixel_to_vector(c, (511.5, 383.5))[0]
    assert np.allclose(oc.point_to_pixel(lin, np.asarray(c["C"]) + d), (511.5, 383.5), atol=1.0)
