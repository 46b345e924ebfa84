"""An independent restatement of dense two-camera triangulation in numpy float64 scalars, walking the reference's expressions
one operation at a time (Camera/PinholeModel.cc:422-430, 553-605; Camera/LensDistortion.cc:258-400; Math/NewtonRaphson.cc:58-119;
Math/Matrix.h:2218-2281; Stereo/StereoModel.cc:35-147, 254-309; Stereo/StereoView.h:91-99, 172-186).  numpy float64 scalar
arithmetic is IEEE double with no contraction, so it rounds as the reference does.  Slow: for small inputs only."""
import numpy as np

F = np.float64
ZERO = F(0.0)


def dot(a, b):
    r = ZERO
    for x, y in zip(a, b):
        r = r + F(x) * F(y)
    return r


def norm(a):
    return np.sqrt(dot(a, a))


def inverse(m):
    """vw::math::inverse: LU with partial pivoting (first largest magnitude), then the two triangular solves"""
    buf = [[F(m[r][c]) for c in range(3)] for r in range(3)]
    pm = [0, 1, 2]
    for i in range(3):
        best, idx = F(-1), 0
        for k in range(3 - i):
            a = abs(buf[i + k][i])
            if a > best:
                best, idx = a, k
        p = i + idx
        if buf[p][i] == 0:
            raise ZeroDivisionError("Matrix is singular in inverse()")
        if p != i:
            pm[i], pm[p] = pm[p], pm[i]
            buf[i], buf[p] = buf[p], buf[i]
        if i != 2:
            for k in range(i + 1, 3):
                buf[k][i] = buf[k][i] / buf[i][i]
            for k in range(i + 1, 3):
                for c in range(i + 1, 3):
                    buf[k][c] = buf[k][c] - buf[k][i] * buf[i][c]
    inv = [[ZERO] * 3 for _ in range(3)]
    for i in range(3):
        inv[i][pm[i]] = F(1)
    for i in range(3):
        for j in range(3):
            t = inv[i][j]
            if t != 0:
                for k in range(i + 1, 3):
                    inv[k][j] = inv[k][j] - buf[k][i] * t
    for i in (2, 1, 0):
        for j in (2, 1, 0):
            inv[i][j] = inv[i][j] / buf[i][i]
            t = inv[i][j]
            if t != 0:
                for k in range(i - 1, -1, -1):
                    inv[k][j] = inv[k][j] - buf[k][i] * t
    return inv


def matmul(a, b):
    return [[dot(a[r], [b[q][c] for q in range(3)]) for c in range(3)] for r in range(3)]


def camera_inverse(cam):
    u, v, w = (list(map(F, cam[k])) for k in ("u", "v", "w"))
    for x, y in ((u, v), (u, w), (v, w)):
        if not dot(x, y) == 0:
            raise AssertionError("frame not orthonormal")
    for x in (u, v, w):
        if not abs(norm(x) - 1) < 0.001:
            raise AssertionError("frame not orthonormal")
    R = np.asarray(cam["rotation"], np.float64)
    rt = [[F(R[c][r]) for c in range(3)] for r in range(3)]
    K = [[F(cam["fu"]), ZERO, F(cam["cu"])], [ZERO, F(cam["fv"]), F(cam["cv"])], [ZERO, ZERO, F(1)]]
    a = inverse(matmul([u, v, w], rt))
    b = inverse(K)
    return matmul(a, b)


def tsai_norm(x, y, k):
    k1, k2, p1, p2, k3 = map(F, k)
    r2 = x * x + y * y
    rdist = F(1.0) + k1 * r2 + k2 * r2 * r2 + k3 * r2 * r2 * r2
    xo = x * rdist + (F(2.0) * p1 * x * y + p2 * (r2 + F(2.0) * x * x))
    yo = y * rdist + (p1 * (r2 + F(2.0) * y * y) + F(2.0) * p2 * x * y)
    return xo, yo


def tsai_jac(x, y, k):
    k1, k2, p1, p2, k3 = map(F, k)
    r2 = x * x + y * y
    dx, dy = F(2.0) * x, F(2.0) * y
    rdist = F(1.0) + k1 * r2 + k2 * r2 * r2 + k3 * r2 * r2 * r2
    ax = k1 * dx + k2 * dx * F(2.0) * r2 + k3 * dx * F(3.0) * r2 * r2
    ay = k1 * dy + k2 * dy * F(2.0) * r2 + k3 * dy * F(3.0) * r2 * r2
    return (rdist + x * ax + F(2.0) * p1 * y + p2 * (dx + F(4.0) * x),
            x * ay + F(2.0) * p1 * x + p2 * dy,
            y * ax + (p1 * dx + F(2.0) * p2 * y),
            rdist + y * ay + p1 * (dy + F(4.0) * y) + F(2.0) * p2 * x)


def tsai_undistort(cam, px, py):
    """(ux, uy, exit): exit 0 converged, 1 bad determinant, 2 NaN |F|, 3 out of iterations, 4 fu or fv < 1e-300"""
    fu, fv, cu, cv = (F(cam[k]) for k in ("fu", "fv", "cu", "cv"))
    if fu < 1e-300 or fv < 1e-300:
        return F(np.inf), F(np.inf), 4
    ox, oy = (px - cu) / fu, (py - cv) / fv
    X, best, best_err, ex = (ox, oy), (ox, oy), F(np.finfo(np.float64).max), 3
    with np.errstate(all="ignore"):
        for _ in range(1, 20):
            fx, fy = tsai_norm(X[0], X[1], cam["tsai"])
            Fv = (fx - ox, fy - oy)
            nf = np.sqrt(ZERO + Fv[0] * Fv[0] + Fv[1] * Fv[1])
            if np.isnan(nf):
                ex = 2
                break
            if nf < best_err:
                best_err, best = nf, X
            J = tsai_jac(X[0], X[1], cam["tsai"])
            det = J[0] * J[3] - J[1] * J[2]
            if abs(det) < 1e-6 or np.isnan(det):
                ex = 1
                break
            D = ((J[3] * Fv[0] - J[1] * Fv[1]) / det, (J[0] * Fv[1] - J[2] * Fv[0]) / det)
            X = (X[0] - D[0], X[1] - D[1])
            if np.sqrt(ZERO + D[0] * D[0] + D[1] * D[1]) < 1e-9:
                best, ex = X, 0
                break
        return best[0] * fu + cu, best[1] * fv + cv, ex


def pixel_to_vector(cam, inv, px, py):
    u, v = F(px) * F(cam["pixel_pitch"]), F(py) * F(cam["pixel_pitch"])
    with np.errstate(all="ignore"):
        if cam.get("tsai") is not None:
            u, v, _ = tsai_undistort(cam, u, v)
        r = [dot(inv[i], (u, v, F(1))) for i in range(3)]
        n = norm(r)
        return [x / n for x in r]


def cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def triangulate(cams, invs, pix, angle_tol=0.0):
    """StereoModel::operator()(pixVec, errorVec) for two cameras: (point, errorVec)"""
    zero = [ZERO] * 3
    dirs, ctrs = [], []
    for cam, inv, (px, py) in zip(cams, invs, pix):
        px, py = F(px), F(py)
        if px != px or py != py or (px == -1e8 and py == -1e8):
            continue
        dirs.append(pixel_to_vector(cam, inv, px, py))
        ctrs.append([F(c) for c in cam["center"]])
    if len(dirs) < 2:
        return zero, zero
    tol = F(angle_tol) if angle_tol > 0 else F(1e-4)
    with np.errstate(all="ignore"):
        if not (F(1) - dot(dirs[0], dirs[1]) >= tol):
            return zero, zero
        (d0, d1), (c0, c1) = dirs, ctrs
        v12 = cross(d0, d1)
        v1, v2 = cross(v12, d0), cross(v12, d1)
        s1 = dot(v2, [b - a for a, b in zip(c0, c1)]) / dot(v2, d0)
        s2 = dot(v1, [a - b for a, b in zip(c0, c1)]) / dot(v1, d1)
        p1 = [c + s1 * d for c, d in zip(c0, d0)]
        p2 = [c + s2 * d for c, d in zip(c1, d1)]
        err = [a - b for a, b in zip(p1, p2)]
        r = [F(0.5) * (a + b) for a, b in zip(p1, p2)]
        if any(dot([a - b for a, b in zip(r, c)], d) < 0 for c, d in zip(ctrs, dirs)):
            r = [-a + F(2) * c for a, c in zip(r, c0)]
    return r, err


def stereo_triangulate(d, cams, window=None, angle_tol=0.0):
    h, w = d.shape[:2]
    x0, y0, ow, oh = (0, 0, w, h) if window is None else window
    invs = [camera_inverse(c) for c in cams]
    out = np.zeros((oh, ow, 3))
    for j in range(y0, y0 + oh):
        for i in range(x0, x0 + ow):
            if d[j, i, 2] != 0:
                out[j - y0, i - x0] = triangulate(cams, invs, ((F(i), F(j)), (F(i) + F(d[j, i, 0]), F(j) + F(d[j, i, 1]))), angle_tol)[0]
    return out


def stereo_model(d, cams, angle_tol=0.0):
    h, w = d.shape[:2]
    invs = [camera_inverse(c) for c in cams]
    xyz, err = np.zeros((h, w, 3)), np.zeros((h, w))
    total, mx, pts, div = ZERO, ZERO, 0, 0
    for y in range(h):
        for x in range(w):
            if d[y, x, 2] == 0:
                continue
            right = (F(np.float32(x) + d[y, x, 0]), F(np.float32(y) + d[y, x, 1]))     # int32 + float, in float
            p, e = triangulate(cams, invs, ((F(x), F(y)), right), angle_tol)
            err[y, x] = norm(e)
            if err[y, x] >= 0:
                xyz[y, x] = p
                mx = max(mx, err[y, x])
                total = total + err[y, x]
                pts += 1
            else:
                div += 1
    return xyz, err, dict(points=pts, divergent=div, max_error=float(mx), error_sum=float(total))


def universe_radius(points, origin, near, far):
    out = np.zeros_like(points)
    rej = 0
    for idx in np.ndindex(points.shape[:2]):
        p = [F(v) for v in points[idx]]
        if p[0] == 0 and p[1] == 0 and p[2] == 0:
            continue
        with np.errstate(all="ignore"):
            dist = norm([a - F(b) for a, b in zip(p, origin)])
        if (near != 0 and dist < near) or (far != 0 and dist > far):
            rej += 1
        else:
            out[idx] = p
    return out, rej, points.shape[0] * points.shape[1]
