"""Independent Python restatement of the neighbourhood outlier filters of Stereo/DisparityMap.h, used to check the C
oracle (oracle/vw_outlier_oracle.c).  It walks the window with an accessor that behaves like the reference's
PixelAccessor (advance / next_col / next_row over edge_extend(in, ConstantEdgeExtension())), so that
RmOutliersUsingMeanFunc's `if (val > cutoff) continue;` -- which skips col_acc.next_col() -- is taken literally: the
following iterations of that window row read the same pixel again.

Pixel values keep their type: numpy int32 or float32 scalars.  The steps the reference takes in the pixel type are taken
in it here (the difference of two disparities, |dx| + |dy|); everything else is a Python float (IEEE double, no FMA).
Slow: meant for small rasters."""
import math

import numpy as np

THRESH, MEAN, STDDEV = 0, 1, 2


class Accessor:
    """a PixelAccessor over the constant edge extension of d (rows, cols, 3)"""

    def __init__(self, d, x, y):
        self.d, self.x, self.y = d, x, y

    def copy(self):
        return Accessor(self.d, self.x, self.y)

    def advance(self, dx, dy):
        self.x += dx
        self.y += dy

    def next_col(self):
        self.x += 1

    def next_row(self):
        self.y += 1

    def get(self):
        h, w = self.d.shape[:2]
        return self.d[min(max(self.y, 0), h - 1), min(max(self.x, 0), w - 1)]


def is_valid(p):
    return p[2] != 0


def _is_float(p):
    return p.dtype == np.float32


def absdiff(a, b):
    """fabs((*acc)[i] - (*col_acc)[i]): the difference in the pixel type, then a double"""
    if isinstance(a, np.float32):
        return abs(float(np.float32(a) - np.float32(b)))
    return float(abs(int(a) - int(b)))


def length(p):
    """std::abs(v[0]) + std::abs(v[1]) in the pixel type, then a double"""
    if _is_float(p):
        return float(np.abs(p[0]) + np.abs(p[1]))
    return float(abs(int(p[0])) + abs(int(p[1])))


def _invalid(p):
    return np.zeros(3, p.dtype)


def thresh_func(acc, hx, hy, pt, rt):
    """RmOutliersUsingThreshFunc::operator() (DisparityMap.h:359-386)"""
    c = acc.get()
    if is_valid(c):
        matched = total = 0
        row = acc.copy()
        row.advance(-hx, -hy)
        for _ in range(-hy, hy + 1):
            col = row.copy()
            for _ in range(-hx, hx + 1):
                n = col.get()
                if is_valid(n) and absdiff(c[0], n[0]) <= pt and absdiff(c[1], n[1]) <= pt:
                    matched += 1
                col.next_col()
                total += 1
            row.next_row()
        if matched / total < rt:
            return _invalid(c)
    return c.copy()


def mean_func(acc, hx, hy, max_mean_diff, literal=True):
    """RmOutliersUsingMeanFunc::operator() (:485-553).  literal=False advances col_acc on the `continue` (skips just the
    one pixel): a contrast that the hand cases must tell apart from the reference."""
    c = acc.get()
    if not is_valid(c):
        return c.copy()
    mdsq = max_mean_diff * max_mean_diff
    lens = []
    row = acc.copy()
    row.advance(-hx, -hy)
    for _ in range(-hy, hy + 1):
        col = row.copy()
        for _ in range(-hx, hx + 1):
            if is_valid(col.get()):
                lens.append(length(col.get()))
            col.next_col()
        row.next_row()
    lens.sort()
    cutoff = 2.0 * lens[int(0.75 * len(lens))] if lens else 0.0
    matched = 0
    mx = my = 0.0
    row = acc.copy()
    row.advance(-hx, -hy)
    for _ in range(-hy, hy + 1):
        col = row.copy()
        for _ in range(-hx, hx + 1):
            q = col.get()
            if is_valid(q):
                if length(q) > cutoff:
                    if not literal:
                        col.next_col()
                    continue
                mx += float(q[0])
                my += float(q[1])
                matched += 1
            col.next_col()
        row.next_row()
    err = mdsq + 1.0
    if matched > 0:
        mx /= matched
        my /= matched
        tx, ty = float(c[0]), float(c[1])
        err = (tx - mx) * (tx - mx) + (ty - my) * (ty - my)
    return _invalid(c) if err > mdsq else c.copy()


def stddev_func(acc, hx, hy, pt, rt):
    """RmOutliersUsingStdDev::operator() (:647-723) over every valid window pixel"""
    c = acc.get()
    if not is_valid(c):
        return c.copy()
    xs, ys = [], []
    mx = my = 0.0
    row = acc.copy()
    row.advance(-hx, -hy)
    for _ in range(-hy, hy + 1):
        col = row.copy()
        for _ in range(-hx, hx + 1):
            q = col.get()
            if is_valid(q):
                xs.append(float(q[0]))
                ys.append(float(q[1]))
                mx += float(q[0])
                my += float(q[1])
            col.next_col()
        row.next_row()
    n = len(xs)
    if n == 0:
        return _invalid(c)
    mx /= n
    my /= n
    sx = sy = 0.0
    for x, y in zip(xs, ys):
        sx += (x - mx) * (x - mx)
        sy += (y - my) * (y - my)
    sdx = math.sqrt(sx / n)
    sdy = math.sqrt(sy / n)
    if sdx < rt:
        sdx = rt
    if sdy < rt:
        sdy = rt
    ex, ey = abs(float(c[0]) - mx), abs(float(c[1]) - my)
    return _invalid(c) if (ex > pt * sdx or ey > pt * sdy) else c.copy()


def valid_count(d, x, y, hx, hy):
    """valid pixels in the window of (x, y) of the edge-extended d"""
    return sum(bool(is_valid(Accessor(d, x + i, y + j).get())) for j in range(-hy, hy + 1) for i in range(-hx, hx + 1))


def _pass1(method, acc, hx, hy, pt, rt, mmd, literal):
    if method == THRESH:
        return thresh_func(acc, hx, hy, pt, rt)
    if method == MEAN:
        return mean_func(acc, hx, hy, mmd, literal)
    return stddev_func(acc, hx, hy, pt, rt)


def outlier_filter(method, cleanup, d, hx, hy, pt=0.0, rt=0.0, mmd=0.0, literal=True, pass2_edge_extended=False):
    """rm_outliers_using_* (cleanup False) or disparity_cleanup_using_* (cleanup True) of d (rows, cols, 3), int32 or
    float32.  The composite's outer functor reads the inner view without an edge extension of its own, so at the border it
    reads pass 1 evaluated at out-of-image centres.  pass2_edge_extended=True instead clamps pass 2's reads to the image:
    a contrast the border hand cases must tell apart from the reference."""
    h, w = d.shape[:2]
    p1 = np.zeros((h + 2, w + 2, 3), d.dtype)
    for y in range(-1, h + 1):
        for x in range(-1, w + 1):
            inside = 0 <= x < w and 0 <= y < h
            if cleanup or inside:
                p1[y + 1, x + 1] = _pass1(method, Accessor(d, x, y), hx, hy, pt, rt, mmd, literal)
    if not cleanup:
        return p1[1:-1, 1:-1].copy()
    src = p1[1:-1, 1:-1].copy() if pass2_edge_extended else p1
    off = 0 if pass2_edge_extended else 1
    out = np.zeros_like(d)
    for y in range(h):
        for x in range(w):
            out[y, x] = thresh_func(Accessor(src, x + off, y + off), 1, 1, 3.0, 0.20)
    return out


def random_disparity(seed, shape, invalid, dtype, scale=6.0, outliers=0.05):
    """a smooth field with noise, outliers and holes; invalid pixels carry non-zero children"""
    rng = np.random.default_rng(seed)
    h, w = shape
    yy, xx = np.mgrid[0:h, 0:w]
    dx = 0.3 * xx - 0.2 * yy + scale * rng.standard_normal((h, w)) * 0.3
    dy = 0.1 * yy + rng.standard_normal((h, w))
    wild = rng.random((h, w)) < outliers
    dx[wild] += rng.uniform(-40, 40, wild.sum())
    dy[wild] += rng.uniform(-40, 40, wild.sum())
    v = (rng.random((h, w)) >= invalid).astype(np.float64)
    if dtype == np.int32:
        d = np.stack([np.rint(dx), np.rint(dy), v], -1).astype(np.int32)
    else:
        d = np.stack([dx, dy, v], -1).astype(np.float32)
    return d
