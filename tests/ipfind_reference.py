"""A numpy restatement of ipfind's iagd + sgrad path that walks the reference's loops literally (float32 scalars for the
reference's float operations, Python floats for its doubles), independent of the C oracle: normalize, the integral image,
the OBALoG box filters, is_extrema, the auto-gain threshold, the Harris test, the stable cull, the tile loop,
remove_ip_near_nodata and describe_interest_points with SGradDescriptorGenerator (libstdc++'s partition, the crop boxes, the
AffineTransform support, bilinear sampling, IntegralBlock).  Slow: for small images.  Citations are under src/vw/."""
import math

import numpy as np

F = np.float32
SIGMA = [1.2, 1.5, 1.875, 2.34375, 2.9296875, 3.662109, 4.577636, 5.722046]          # IntegralInterestOperator.cc:28
BW = [[11, 7, 5, 3, 3, 1], [13, 9, 7, 5, 3, 1], [17, 11, 9, 5, 5, 3], [21, 13, 11, 7, 7, 3],
      [27, 17, 13, 9, 9, 5], [33, 21, 17, 11, 11, 5], [41, 27, 21, 13, 13, 7], [51, 33, 27, 17, 17, 7]]
BH = [[11, 5, 7, 3, 1, 3], [13, 7, 9, 1, 3, 5], [17, 9, 11, 5, 3, 5], [21, 11, 13, 3, 7, 7],
      [27, 13, 17, 5, 9, 9], [33, 17, 21, 5, 11, 11], [41, 21, 27, 7, 13, 13], [51, 27, 33, 7, 17, 17]]
WT = [[0.0006179999909, 0.008283999749, 0.008283999749, -0.03556599841, -0.05576400086, -0.05576400086],
      [0.0002659999882, 0.004889999982, 0.004889999982, -0.0221420005, -0.0488499999, -0.0221420005],
      [0.0002659424644, 0.003207367443, 0.003207367443, -0.001847865087, -0.022190776, -0.022190776],
      [0.000218920823, 0.002005755751, 0.002005755751, -0.01499466244, -0.0008247125278, -0.01499466244],
      [0.0001030362087, 0.00137811946, 0.00137811946, -0.009606413672, 0.002226325845, -0.009606413672],
      [7.198028372e-05, 0.0008259398524, 0.0008259398524, -0.006072390568, -1.177469443e-06, -0.006072390568],
      [3.803569417e-05, 0.0005251058097, 0.0005251058097, -0.003885340628, 0.0002823550512, -0.003885340628],
      [2.892054582e-05, 0.0003287680581, 0.0003287680581, -0.002447736656, -0.0002717150913, -0.002447736656]]
STRT, BSZ, BHF = [17, 15, 9, 6, 0], [2, 4, 8, 10, 14], [1, 2, 4, 5, 7]                   # Descriptor.cc:27-29


def normalize(raw, nodata=None):
    """AutoNormalize.h:76-86 over create_mask when nodata is given; MinMaxAccumulator keeps the first of equal values"""
    nd = None if nodata is None else F(nodata)
    mn = mx = None
    for v in raw.ravel():
        if nd is not None and v == nd:
            continue
        if mn is None:
            mn = mx = v
        else:
            if v < mn:
                mn = v
            if mx < v:
                mx = v
    ratio = 0.0 if mx == mn else float(F(1)) / float(F(mx - mn))
    out = np.empty_like(raw)
    for (r, c), v in np.ndenumerate(raw):
        out[r, c] = F(0) if (nd is not None and v == nd) else F(float(F(v - mn)) * ratio + 0.0)
    return out


def integral(img):
    """IntegralImage.h:41-91"""
    h, w = img.shape
    I = np.zeros((h + 1, w + 1), F)
    for y in range(h):
        for x in range(w):
            I[y + 1, x + 1] = F(F(F(img[y, x] + I[y + 1, x]) + I[y, x + 1]) - I[y, x])
    return I


def interest(I, s):
    """abs(box_filter(I, scale s)) (BoxFilter.h:48-114), each pixel's boxes in order"""
    h, w = I.shape[0] - 1, I.shape[1] - 1
    pb = BW[s][0] >> 1
    out = np.zeros((h, w), F)
    for y in range(pb, h - pb):
        for x in range(pb, w - pb):
            res = F(0)
            for b in range(6):
                bw, bh = BW[s][b], BH[s][b]
                x0, y0 = x - (bw >> 1), y - (bh >> 1)
                box = F(F(F(F(0) + I[y0, x0]) - I[y0, x0 + bw]) - I[y0 + bh, x0])
                box = F(box + I[y0 + bh, x0 + bw])
                res = F(res + F(F(WT[s][b]) * box))
            out[y, x] = abs(res)
    return out


def gaussian_taps():
    """generate_gaussian_kernel(k, 2, 9) (Filter.tcc:37-80) with the C library's erf"""
    z = 1 / (math.sqrt(2.0) * 2.0)
    k = [0.0] * 9
    total = 0.0
    for i in range(1, 5):
        tap = math.erf((i + 0.5) * z) - math.erf((i - 0.5) * z)
        total += tap
        k[4 + i] = k[4 - i] = tap
    total *= 2.0
    tap = math.erf(0.5 * z) - math.erf(-0.5 * z)
    total += tap
    k[4] = tap
    norm = 1.0 / total
    return [t * norm for t in k]


def is_extrema(lo, mid, hi, x, y):
    v = mid[y, x]
    if v <= lo[y, x] or v <= hi[y, x]:
        return False
    for dy, dx in ((-1, -1), (-1, 0), (-1, 1), (0, 1), (1, 1), (1, 0), (1, -1), (0, -1)):
        if v <= lo[y + dy, x + dx] or v <= mid[y + dy, x + dx] or v <= hi[y + dy, x + dx]:
            return False
    return True


def harris(mid, ix, iy, m, k):
    step = int(F(SIGMA[m]))
    offset = 4 * step
    sxx = syy = sxy = F(0)
    for jy, y in enumerate(range(iy - offset, iy + offset + 1, step)):
        for jx, x in enumerate(range(ix - offset, ix + offset + 1, step)):
            Lx = F(mid[y, x - 1] - mid[y, x + 1])
            Ly = F(mid[y - 1, x] - mid[y + 1, x])
            wgt = F(k[jx] * k[jy])
            sxx = F(sxx + F(F(Lx * Lx) * wgt))
            syy = F(syy + F(F(Ly * Ly) * wgt))
            sxy = F(sxy + F(F(Lx * Ly) * wgt))
    trace = F(sxx + syy)
    det = F(F(sxx * syy) - F(sxy * sxy))
    with np.errstate(divide="ignore", invalid="ignore"):
        return bool(F(F(trace * trace) / det) < 12)


def process_tile(tile, num_ip, k):
    """IntegralAutoGainDetector::process_image (IntegralDetector.cc:264-370): [(x, y, scale, interest)]"""
    h, w = tile.shape
    I = integral(tile)
    data = [interest(I, s) for s in range(8)]
    pts = []
    for m in range(1, 7):
        lo, mid, hi = data[m - 1], data[m], data[m + 1]
        found = []
        for r in range(1, h - 1):
            for c in range(1, w - 1):
                if is_extrema(lo, mid, hi, c, r):
                    found.append((c, r, F(SIGMA[m]), mid[r, c]))
        imin = imax = mid.ravel()[0]
        for v in mid.ravel()[1:]:
            if v < imin:
                imin = v
            if imax < v:
                imax = v
        thr = F(float(imin) + 0.001 * float(F(imax - imin)))
        pts += [p for p in found if not p[3] < thr and harris(mid, p[0], p[1], m, k)]
    if 0 < num_ip < len(pts):
        pts = sorted(pts, key=lambda p: -float(p[3]))[:num_ip]   # Python's sort is stable, as std::list::sort
    return pts


def detect(img, ip_per_tile, tile_size=1024):
    """detect_interest_points (DetectorBase.h:250-328): structured rows (x, y, ix, iy, scale, interest, orientation)"""
    ts = max(1024, tile_size)
    k = gaussian_taps()
    h, w = img.shape
    out = []
    for y0 in range(0, h, ts):
        for x0 in range(0, w, ts):
            tw, th = min(ts, w - x0), min(ts, h - y0)
            num_ip = 0
            if ip_per_tile > 0:
                num_ip = min(max(int(math.ceil(tw * th / float(ts * ts) * ip_per_tile)), 1), ip_per_tile)
            for (x, y, s, v) in process_tile(img[y0:y0 + th, x0:x0 + tw], num_ip, k):
                out.append((F(F(x) + F(x0)), F(F(y) + F(y0)), x + x0, y + y0, s, v, F(0)))
    return out


def remove_near_nodata(raw, pts, nodata, radius):
    """InterestPointUtils.h:45-82"""
    h, w = raw.shape
    keep = []
    for p in pts:
        ix, iy = p[2], p[3]
        if not (radius <= ix < w - radius and radius <= iy < h - radius):
            continue
        if any(float(raw[y, x]) == nodata for y in range(iy - radius, iy + radius + 1) for x in range(ix - radius, ix + radius + 1)):
            continue
        keep.append(p)
    return keep


def _affine(x, y, scale, ori):
    """get_support's AffineTransform (Descriptor.h:242-254) with its 2 x 2 inverse (Matrix.h:2209-2216): (ai, bi, ci, di, ox, oy)"""
    scaling = float(F(F(1) / F(scale)))
    c, s = math.cos(float(-F(ori))), math.sin(float(-F(ori)))
    a, b, cc, d = scaling * c, -scaling * s, scaling * s, scaling * c
    ox = scaling * (s * float(y) - c * float(x)) + 20.5
    oy = -scaling * (s * float(x) + c * float(y)) + 20.5
    det = a * d - b * cc
    return d / det, -b / det, -cc / det, a / det, ox, oy


def _reverse(t, px, py):
    qx, qy = px - t[4], py - t[5]
    return t[0] * qx + t[1] * qy, t[2] * qx + t[3] * qy


def sgrad(support):
    I = integral(support)
    out = []
    sqr = F(0)
    for s in range(5):
        inv = F(F(1) / F(BHF[s] * BHF[s]))
        b = BHF[s]
        for i in range(3):
            for j in range(3):
                tx, ty = STRT[s] + i * BSZ[s], STRT[s] + j * BSZ[s]
                q = []
                for (x0, y0) in ((tx, ty), (tx + b, ty), (tx, ty + b), (tx + b, ty + b)):   # IntegralBlock, IntegralImage.cc:27-53
                    x1, y1 = x0 + b, y0 + b
                    q.append(F(F(F(I[y0, x0] + I[y1, x1]) - I[y1, x0]) - I[y0, x1]))
                for v in (F(q[0] - q[2]), F(q[1] - q[3]), F(q[0] - q[1]), F(q[2] - q[3])):
                    g = F(v * inv)
                    out.append(g)
                    sqr = F(sqr + F(g * g))
    inv = F(1.0 / math.sqrt(float(sqr)))          # ::sqrt(double): a double quotient
    if not (np.isfinite(inv) and abs(inv) >= np.finfo(F).tiny):
        inv = F(0)
    return [F(g * inv) for g in out]


def describe(img, pts, tile_size=1024):
    """describe_interest_points with SGradDescriptorGenerator (Descriptor.h:202-355, 414-471): (points, descriptors)"""
    ts = max(1024, tile_size)
    h, w = img.shape
    pts = [list(p) for p in pts]
    desc = [None] * len(pts)
    first = 0
    for ty in range(0, h, ts):
        for tx in range(0, w, ts):
            x1, y1 = tx + min(ts, w - tx), ty + min(ts, h - ty)
            inside = lambda p: tx <= int(p[0]) < x1 and ty <= int(p[1]) < y1      # IsInBBox: Vector2i(ip.x, ip.y)
            f, l = first, len(pts)
            while True:                                   # libstdc++'s std::partition for bidirectional iterators
                while f != l and inside(pts[f]):
                    f += 1
                if f == l:
                    break
                l -= 1
                while f != l and not inside(pts[l]):
                    l -= 1
                if f == l:
                    break
                pts[f], pts[l] = pts[l], pts[f]
                f += 1
            sec = range(first, f)
            first = f
            if not sec:
                continue
            box = None
            for q in sec:
                t = _affine(pts[q][0], pts[q][1], pts[q][4], pts[q][6])
                cs = [_reverse(t, px, py) for px, py in ((0, 0), (41, 0), (0, 41), (41, 41))]
                mnx, mxx = min(c[0] for c in cs), max(c[0] for c in cs)
                mny, mxy = min(c[1] for c in cs), max(c[1] for c in cs)
                b = (math.floor(mnx), math.floor(mny), math.floor(mxx) + 1, math.floor(mxy) + 1)
                box = b if box is None else (min(box[0], b[0]), min(box[1], b[1]), max(box[2], b[2]), max(box[3], b[3]))
            bx0, by0, bx1, by1 = box[0] - 1, box[1] - 1, box[2] + 1, box[3] + 1
            crop = np.zeros((by1 - by0, bx1 - bx0), F)
            for j in range(by1 - by0):
                for i in range(bx1 - bx0):
                    if 0 <= bx0 + i < w and 0 <= by0 + j < h:
                        crop[j, i] = img[by0 + j, bx0 + i]
            for q in sec:
                pts[q][0] = F(pts[q][0] - F(bx0))
                pts[q][1] = F(pts[q][1] - F(by0))
                t = _affine(pts[q][0], pts[q][1], pts[q][4], pts[q][6])
                sup = np.zeros((42, 42), F)
                for j in range(42):
                    for i in range(42):
                        sup[j, i] = _bilinear(crop, *_reverse(t, float(i), float(j)))
                desc[q] = sgrad(sup)
                pts[q][0] = F(pts[q][0] + F(bx0))
                pts[q][1] = F(pts[q][1] + F(by0))
    assert first == len(pts)
    return [tuple(p) for p in pts], desc


def _px(crop, i, j):
    return crop[j, i] if 0 <= i < crop.shape[1] and 0 <= j < crop.shape[0] else F(0)


def _bilinear(crop, i, j):
    """BilinearInterpolation (Interpolation.h:76-110) with real_type float, zero edge"""
    x, y = math.floor(i), math.floor(j)
    if x == i and y == j:
        return _px(crop, x, y)
    nx, ny = F(F(i) - F(x)), F(F(j) - F(y))
    n1mx, n1my = F(F(1) - nx), F(F(1) - ny)
    r = F(_px(crop, x, y) * n1mx)
    r = F(r + F(_px(crop, x + 1, y) * nx))
    r = F(r * n1my)
    row = F(_px(crop, x, y + 1) * n1mx)
    row = F(row + F(_px(crop, x + 1, y + 1) * nx))
    return F(r + F(row * ny))
