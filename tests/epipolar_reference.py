"""An independent restatement of epipolar rectification in numpy float64 / float32 scalars, walking the reference's expressions
one operation at a time: Quaternion(R) and rotation_matrix() (Math/Quaternion.h:211-252, 314-335), epipolar()
(Camera/PinholeModel.cc:679-732), the camera matrix (:553-605), point_to_pixel with its check (:351-397,
Camera/LensDistortion.cc:345-369), CameraTransform (Camera/CameraTransform.h:52-74), compute_transformed_bbox_fast with
BBox2f (Image/Transform.h:271-315, Math/BBox.tcc:38-97) and resize_epipolar_cameras_to_fit (Camera/EpipolarUtils.cc:37-76).
The ray side (pixel_to_vector, the Tsai Newton-Raphson) is triangulate_reference's.  Slow: for small inputs only."""
import numpy as np

from triangulate_reference import camera_inverse, cross, dot, norm, pixel_to_vector, tsai_norm

F = np.float64
F32 = np.float32


class ProjectionError(ArithmeticError):
    """where the reference throws PointToPixelErr"""


def quaternion_round_trip(R):
    """(rotation_matrix() of Quaternion(R) as a 3 x 3 list, the branch: 0 ww, 1 xx, 2 yy, 3 zz)"""
    r = [[F(R[i][j]) for j in range(3)] for i in range(3)]
    d0, d1, d2 = r[0][0], r[1][1], r[2][2]
    one = F(1.0)
    ww, xx, yy, zz = one + d0 + d1 + d2, one + d0 - d1 - d2, one - d0 + d1 - d2, one - d0 - d1 + d2
    mx = ww
    for c in (xx, yy, zz):
        if c > mx:
            mx = c
    if ww == mx:
        s = np.sqrt(ww * F(4.0))
        q, b = (s / F(4), (r[2][1] - r[1][2]) / s, (r[0][2] - r[2][0]) / s, (r[1][0] - r[0][1]) / s), 0
    elif xx == mx:
        s = np.sqrt(xx * F(4.0))
        q, b = ((r[2][1] - r[1][2]) / s, s / F(4), (r[0][1] + r[1][0]) / s, (r[0][2] + r[2][0]) / s), 1
    elif yy == mx:
        s = np.sqrt(yy * F(4.0))
        q, b = ((r[0][2] - r[2][0]) / s, (r[0][1] + r[1][0]) / s, s / F(4), (r[1][2] + r[2][1]) / s), 2
    else:
        s = np.sqrt(zz * F(4.0))
        q, b = ((r[1][0] - r[0][1]) / s, (r[0][2] + r[2][0]) / s, (r[1][2] + r[2][1]) / s, s / F(4)), 3
    w, x, y, z = q
    w2, x2, y2, z2 = w * w, x * x, y * y, z * z
    wx, wy, wz, xy, yz, zx = w * x, w * y, w * z, x * y, y * z, z * x
    two = F(2)
    out = [[w2 + x2 - y2 - z2, two * (xy - wz), two * (zx + wy)],
           [two * (xy + wz), w2 - x2 + y2 - z2, two * (yz - wx)],
           [two * (zx - wy), two * (yz + wx), w2 - x2 - y2 + z2]]
    return out, b


def epipolar(cam0, cam1):
    camera_inverse(cam0)                                   # the sources are cameras the reference can construct
    camera_inverse(cam1)
    with np.errstate(all="ignore"):
        rot0, _ = quaternion_round_trip(cam0["rotation"])
        rot1, _ = quaternion_round_trip(cam1["rotation"])
        c0, c1 = [F(x) for x in cam0["center"]], [F(x) for x in cam1["center"]]
        look0, look1 = [F(-1) * rot0[i][2] for i in range(3)], [F(-1) * rot1[i][2] for i in range(3)]
        d = [c1[i] - c0[i] for i in range(3)]
        nd = norm(d)
        u = [x / nd for x in d]
        mean = [(look0[i] + look1[i]) / F(2.0) for i in range(3)]
        t = cross(u, cross(mean, u))
        nt = norm(t)
        w = [x / nt for x in t]
        v = cross(w, u)
    rot = np.array([[u[i], -v[i], -w[i]] for i in range(3)])
    half = F(2.0)
    base = dict(rotation=rot, fu=(F(cam0["fu"]) + F(cam1["fu"])) / half, fv=(F(cam0["fv"]) + F(cam1["fv"])) / half,
                cu=(F(cam0["cu"]) + F(cam1["cu"])) / half, cv=(F(cam0["cv"]) + F(cam1["cv"])) / half, u=(1.0, 0.0, 0.0),
                v=(0.0, 1.0, 0.0), w=(0.0, 0.0, 1.0), pixel_pitch=(F(cam0["pixel_pitch"]) + F(cam1["pixel_pitch"])) / half, tsai=None)
    return dict(base, center=tuple(c0)), dict(base, center=tuple(c1))


def camera_matrix(cam):
    camera_inverse(cam)                                    # the frame asserts
    uvw = [list(map(F, cam[k])) for k in ("u", "v", "w")]
    R = np.asarray(cam["rotation"], np.float64)
    rt = [[F(R[c][r]) for c in range(3)] for r in range(3)]
    nrt = [[-x for x in row] for row in rt]
    C = [F(x) for x in cam["center"]]
    extr = [[dot(uvw[r], [rt[q][c] for q in range(3)]) for c in range(3)] for r in range(3)]
    m2 = [[dot(uvw[r], [nrt[q][c] for q in range(3)]) for c in range(3)] for r in range(3)]
    for r in range(3):
        extr[r].append(dot(m2[r], C))
    K = [[F(cam["fu"]), F(0), F(cam["cu"])], [F(0), F(cam["fv"]), F(cam["cv"])], [F(0), F(0), F(1)]]
    return [[dot(K[r], [extr[q][c] for q in range(3)]) for c in range(4)] for r in range(3)]


class Cam:
    """a camera with the two matrices the reference keeps"""

    def __init__(self, cam):
        self.cam, self.P, self.inv = cam, camera_matrix(cam), camera_inverse(cam)


def point_to_pixel(c, point):
    """(pixel, ok): ok False where the reference throws"""
    P, cam = c.P, c.cam
    X = [F(x) for x in point]
    with np.errstate(all="ignore"):
        den = P[2][0] * X[0] + P[2][1] * X[1] + P[2][2] * X[2] + P[2][3]
        px = (P[0][0] * X[0] + P[0][1] * X[1] + P[0][2] * X[2] + P[0][3]) / den
        py = (P[1][0] * X[0] + P[1][1] * X[1] + P[1][2] * X[2] + P[1][3]) / den
        if cam.get("tsai") is not None:
            fu, fv, cu, cv = (F(cam[k]) for k in ("fu", "fv", "cu", "cv"))
            if fu < 1e-300 or fv < 1e-300:
                px = py = F(np.inf)
            else:
                dx, dy = tsai_norm((px - cu) / fu, (py - cv) / fv, cam["tsai"])
                px, py = dx * fu + cu, dy * fv + cv
        pitch = F(cam["pixel_pitch"])
        px, py = px / pitch, py / pitch
        pv = pixel_to_vector(cam, c.inv, px, py)
        d = [X[i] - F(cam["center"][i]) for i in range(3)]
        n = norm(d)
        phys = [x / n for x in d]
        diff = norm([pv[i] - phys[i] for i in range(3)])
        if diff >= 0.01:
            diff = norm([pv[i] + phys[i] for i in range(3)])
    return (px, py), not (diff >= 0.01 or diff != diff)


def _map(frm, to, p):
    r = pixel_to_vector(frm.cam, frm.inv, F(p[0]), F(p[1]))
    return point_to_pixel(to, [r[i] + F(frm.cam["center"][i]) for i in range(3)])


def forward(src, dst, p):
    return _map(src, dst, p)


def reverse(src, dst, p):
    return _map(dst, src, p)


def bbox_fast(src, dst, roi):
    """compute_transformed_bbox_fast(roi, CameraTransform(src, dst)) as float32 [min x, min y, max x, max y]; ProjectionError
    with the perimeter index"""
    x0, y0, x1, y1 = (int(v) for v in roi)
    big = F32(2147483647 - 1)
    mn, mx = [big, big], [-big, -big]
    pts = [(x, y0) for x in range(x0, x1)] + [(x, y1 - 1) for x in range(x0, x1)] + [(x0, y) for y in range(y0, y1)] + \
          [(x1 - 1, y) for y in range(y0, y1)]
    for k, p in enumerate(pts):
        q, ok = forward(src, dst, p)
        if not ok:
            raise ProjectionError(k)
        for i in range(2):
            if q[i] > F(mx[i]):
                mx[i] = F32(q[i])
            if q[i] < F(mn[i]):
                mn[i] = F32(q[i])
    return [mn[0], mn[1], mx[0], mx[1]]


def resize(cam1, cam2, epi1, epi2, roi1, roi2):
    c1, c2 = Cam(cam1), Cam(cam2)
    b1, b2 = bbox_fast(c1, Cam(epi1), roi1), bbox_fast(c2, Cam(epi2), roi2)
    min_col = F(b2[0] if b2[0] < b1[0] else b1[0])
    min_row = F(b2[1] if b2[1] < b1[1] else b1[1])
    pitch = F(epi1["pixel_pitch"])
    cu, cv = F(epi1["cu"]) - min_col * pitch, F(epi1["cv"]) - min_row * pitch
    e1, e2 = dict(epi1, cu=cu, cv=cv), dict(epi2, cu=cu, cv=cv)
    b1, b2 = bbox_fast(c1, Cam(e1), roi1), bbox_fast(c2, Cam(e2), roi2)
    return e1, e2, (int(b1[2]), int(b1[3])), (int(b2[2]), int(b2[3]))
