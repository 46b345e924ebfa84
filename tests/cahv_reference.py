"""An independent numpy scalar restatement of the CAHV / CAHVOR camera math (Camera/CAHVModel.cc, CAHVORModel.cc), one float64
operation per reference operation, to check oracle/vw_cahv_oracle.c against; and the seeded test cameras the CAHV tests share."""
import numpy as np

f64 = np.float64


def dot(a, b):
    r = f64(0.0)
    for i in range(3):
        r = f64(r + f64(a[i]) * f64(b[i]))
    return r


def cross(a, b):
    a, b = [f64(x) for x in a], [f64(x) for x in b]
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def normalize(a):
    n = np.sqrt(dot(a, a))
    return [f64(x) / n for x in a]


def pixel_to_vector(c, pix):
    """(direction, exit code: -1 CAHV, 0 converged, 1 deriv <= 0, 2 20 passes, Newton passes)"""
    x, y = f64(pix[0]), f64(pix[1])
    A, H, V = [[f64(v) for v in c[k]] for k in "AHV"]
    rr = normalize(cross([V[i] - y * A[i] for i in range(3)], [H[i] - x * A[i] for i in range(3)]))
    if dot(cross(V, H), A) < 0:
        rr = [v * f64(-1.0) for v in rr]
    if c["model"] == 1:
        return rr, -1, 0
    O, R = [f64(v) for v in c["O"]], [f64(v) for v in c["R"]]
    omega = dot(rr, O)
    lam = [rr[i] - omega * O[i] for i in range(3)]
    tau = dot(lam, lam) / (omega * omega)
    k1, k3, k5 = f64(1) + R[0], R[1] * tau, R[2] * tau * tau
    u = f64(1.0) - (R[0] + k3 + k5)
    code, n = 2, 0
    with np.errstate(all="ignore"):
        for _ in range(20):
            n += 1
            u2 = u * u
            poly = ((k5 * u2 + k3) * u2 + k1) * u - f64(1)
            deriv = (f64(5) * k5 * u2 + f64(3) * k3) * u2 + k1
            if deriv <= 0:
                code = 1
                break
            du = poly / deriv
            u = u - du
            if abs(du) < 1e-6:
                code = 0
                break
        return normalize([rr[i] - (f64(1) - u) * lam[i] for i in range(3)]), code, n


def point_to_pixel(c, point):
    v = [f64(point[i]) - f64(c["C"][i]) for i in range(3)]
    if c["model"] == 2:
        O, R = [f64(x) for x in c["O"]], [f64(x) for x in c["R"]]
        omega = dot(v, O)
        lam = [v[i] - omega * O[i] for i in range(3)]
        tau = dot(lam, lam) / (omega * omega)
        mu = R[0] + (R[1] * tau) + (R[2] * tau * tau)
        v = [v[i] + mu * lam[i] for i in range(3)]
    alpha = dot(v, c["A"])
    return [dot(v, c["H"]) / alpha, dot(v, c["V"]) / alpha]


def epipolar(s0, s1):
    hc = dot(s0["H"], s0["A"]) / f64(2.0) + dot(s1["H"], s1["A"]) / f64(2.0)
    vc = dot(s0["V"], s0["A"]) / f64(2.0) + dot(s1["V"], s1["A"]) / f64(2.0)
    nrm = lambda a: np.sqrt(dot(a, a))
    hs = nrm(cross(s0["A"], s0["H"])) / f64(2.0) + nrm(cross(s1["A"], s1["H"])) / f64(2.0)
    vs = nrm(cross(s0["A"], s0["V"])) / f64(2.0) + nrm(cross(s1["A"], s1["V"])) / f64(2.0)
    app = [f64(s0["A"][i]) + f64(s1["A"][i]) for i in range(3)]
    f = cross(cross(app, [f64(s1["C"][i]) - f64(s0["C"][i]) for i in range(3)]), app)
    nf = nrm(f)
    hp = [f[i] * hs / nf for i in range(3)] if dot(f, s0["H"]) > 0 else [-f[i] * hs / nf for i in range(3)]
    app = [v * f64(0.5) for v in app]
    d = dot(app, hp)
    a = normalize([app[i] - hp[i] * d / (hs * hs) for i in range(3)])
    vp = [v * vs / hs for v in cross(a, hp)]
    e = {"model": 1, "A": tuple(a), "H": tuple(hp[i] + hc * a[i] for i in range(3)), "V": tuple(vp[i] + vc * a[i] for i in range(3))}
    return dict(e, C=tuple(f64(x) for x in s0["C"])), dict(e, C=tuple(f64(x) for x in s1["C"]))


def linearize(c, in_size, out_size):
    ix, iy = int(in_size[0]), int(in_size[1])
    half = lambda n: int(n / 2) if n >= 0 else -int(-n / 2)          # C's truncating int division of n by 2
    hpts = [(0, 0), (0, (iy - 1) / 2.0), (0, iy - 1), (ix - 1, 0), (ix - 1, (iy - 1) / 2.0), (ix - 1.0, iy - 1.0)]
    vpts = [(0, 0), ((ix - 1) / 2.0, 0), (ix - 1, 0), (0, iy - 1), (half(ix - 1), iy - 1), (ix - 1.0, iy - 1.0)]
    A = [f64(0.0)] * 3
    for p in vpts + hpts:
        r = pixel_to_vector(c, p)[0]
        A = [A[i] + r[i] for i in range(3)]
    A = normalize(A)
    dn = cross(c["A"], c["H"])
    rt = normalize(cross(dn, c["A"]))
    dn = normalize(dn)
    rt = cross(dn, A)
    dn = normalize(cross(A, rt))
    rt = normalize(rt)
    mins = []
    for pts, axis in ((hpts, dn), (vpts, rt)):
        lo = f64(1)
        for p in pts:
            u3 = pixel_to_vector(c, p)[0]
            d = dot(axis, u3)
            t = cross(A, normalize([u3[i] - d * axis[i] for i in range(3)]))
            sn = np.sqrt(dot(t, t))
            if lo > sn:
                lo = sn
        mins.append(lo)
    ic = [(f64(out_size[0]) - f64(1)) / f64(2.0), (f64(out_size[1]) - f64(1)) / f64(2.0)]
    ic2 = [ic[0] * ic[0], ic[1] * ic[1]]
    with np.errstate(all="ignore"):
        sf = [np.sqrt(ic2[k] / (mins[k] * mins[k]) - ic2[k]) for k in range(2)]
    return {"model": 1, "C": tuple(f64(x) for x in c["C"]), "A": tuple(A), "H": tuple(sf[0] * rt[i] + ic[0] * A[i] for i in range(3)),
            "V": tuple(sf[1] * dn[i] + ic[1] * A[i] for i in range(3))}


# ---- seeded cameras ------------------------------------------------------------------------------------------------------------

def rover(seed, w, h, center=(0.0, 0.0, 0.0), model=2, r=(1e-3, -2e-3, 1.8e-2), left=False, tilt=0.03):
    """a Navcam-like CAHV / CAHVOR camera over a w x h image looking roughly along +x (f about 0.9 w), O near A"""
    rng = np.random.default_rng(seed)
    A = np.array([1.0, rng.normal(0, tilt), rng.normal(0, tilt)])
    A /= np.linalg.norm(A)
    hv = np.cross(A, [0, 0, 1.0]) * -1
    hv /= np.linalg.norm(hv)
    vv = np.cross(A, hv)
    if left:
        hv = -hv
    f = 0.9 * max(w, 4) * rng.uniform(0.97, 1.03)
    H = f * hv + (w / 2 + rng.normal(0, 1)) * A
    V = f * vv + (h / 2 + rng.normal(0, 1)) * A
    c = {"model": model, "C": tuple(center), "A": tuple(A), "H": tuple(H), "V": tuple(V)}
    if model == 2:
        O = A + rng.normal(0, 0.01, 3)
        c["O"], c["R"] = tuple(O / np.linalg.norm(O)), tuple(r)
    return c


# the reference's cahvor.txt camera (TestCAHVORModel.cxx) and the ForwardReverse cameras
CAHVOR_TXT = {"model": 2, "C": (76.0, -34.0, 20.0), "A": (0.267261, 0.534522, 0.801784), "H": (1300.0, 123.0, 456.0), "V": (345.0, 900.0, 157.0),
              "O": (0.371391, 0.557086, 0.742781), "R": (1.0, -1.0, 1.0)}
FR_CAHV = {"model": 1, "C": (0.606583, -0.036214, -0.234717), "A": (0.708256, -0.0113108, 0.705866), "H": (365.881, 275.126, 361.931),
           "V": (173.589, -3.95587, 550.402)}
FR_CAHVOR = {"model": 2, "C": (0.491222, -0.0717236, -1.24143), "A": (0.921657, -0.230518, 0.312107), "H": (757.076, 1071.6, 160.227),
             "V": (91.7479, -27.7504, 1319.48), "O": (0.920759, -0.206185, 0.331197), "R": (0.00096, -0.002183, 0.018547)}
