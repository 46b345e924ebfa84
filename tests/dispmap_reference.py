"""An independent numpy restatement of the disparity resampling, range and transform operations of
src/vw/Stereo/DisparityMap.h, walking the reference's accessors literally: ConstantEdgeExtension reads, each subsample term
cast (or not) to AccumulatorType before its multiply, a sequential accumulator, PixelAccumulator<EWMinMaxAccumulator> in
raster order, and HomographyTransform's operation order.  Scalars are numpy float32 / float64 / int32 / int64 so that every
step rounds as the reference's does.  Used to check the C oracle (oracle/vw_dispmap_oracle.c) pixel for pixel.

Pixels are (rows, cols, 3) {dx, dy, valid} int32 or float32 arrays.  Created pixels get valid = 1, invalid ones {0, 0, 0};
passed-through pixels are copied."""
import math

import numpy as np

F32, F64, I32, I64 = np.float32, np.float64, np.int32, np.int64


def _types(d):
    """(channel type, AccumulatorType) of Core/FundamentalTypes.h:111-122"""
    return (I32, I64) if d.dtype == np.int32 else (F32, F64)


def _mul_px(k, v, ch):
    """k * child in the channel type: an int32 product wraps, a float32 one rounds"""
    if ch is I32:
        return I32(((int(k) * int(v) + 2 ** 31) % 2 ** 32) - 2 ** 31)
    return F32(F32(k) * v)


def disparity_subsample(d):
    ch, acc = _types(d)
    h, w = d.shape[:2]
    ow, oh = 1 + (w - 1) // 2, 1 + (h - 1) // 2
    out = np.zeros((oh, ow, 3), d.dtype)

    def child(i, j):                                      # EdgeExtensionView<ViewT, ConstantEdgeExtension>
        return d[min(max(j, 0), h - 1), min(max(i, 0), w - 1)]

    cast_terms = ((0, 0, 10), (1, 0, 5), (0, 1, 5))
    px_terms = ((-1, 0, 5), (0, -1, 5), (1, 1, 2), (-1, -1, 2), (-1, 1, 2), (1, -1, 2))
    for j in range(oh):
        for i in range(ow):
            ci, cj = i << 1, j << 1
            bx, by, count = acc(0), acc(0), acc(0)
            for di, dj, k in cast_terms:                  # k * bff_type(child)
                p = child(ci + di, cj + dj)
                if p[2] != 0:
                    count = acc(count + acc(k))
                    bx = acc(bx + acc(acc(k) * acc(p[0])))
                    by = acc(by + acc(acc(k) * acc(p[1])))
            for di, dj, k in px_terms:                    # k * child, then widened
                p = child(ci + di, cj + dj)
                if p[2] != 0:
                    count = acc(count + acc(k))
                    bx = acc(bx + acc(_mul_px(k, p[0], ch)))
                    by = acc(by + acc(_mul_px(k, p[1], ch)))
            if count > 0:
                n = acc(count * acc(2))
                if acc is I64:                            # C++ integer division truncates toward zero
                    qx = int(bx) // int(n) if (int(bx) >= 0) == (int(n) > 0) else -((-int(bx)) // int(n))
                    qy = int(by) // int(n) if (int(by) >= 0) == (int(n) > 0) else -((-int(by)) // int(n))
                    out[j, i] = (qx, qy, 1)
                else:
                    out[j, i] = (F32(bx / n), F32(by / n), 1)
    return out


def disparity_upsample(d):
    ch, _ = _types(d)
    h, w = d.shape[:2]
    out = np.zeros((2 * h, 2 * w, 3), d.dtype)
    for j in range(2 * h):
        for i in range(2 * w):
            p = d[j >> 1, i >> 1]
            out[j, i] = (_mul_px(2, p[0], ch), _mul_px(2, p[1], ch), 1 if p[2] != 0 else 0)
    return out


def get_disparity_range(d):
    """(min dx, min dy, max dx, max dy) as float32: the first valid pixel sets both, then `<` / else `>` per channel"""
    mn = mx = None
    for j in range(d.shape[0]):
        for i in range(d.shape[1]):
            p = d[j, i]
            if p[2] == 0:
                continue
            if mn is None:
                mn, mx = [p[0], p[1]], [p[0], p[1]]
                continue
            for c in range(2):
                if p[c] < mn[c]:
                    mn[c] = p[c]
                elif p[c] > mx[c]:
                    mx[c] = p[c]
    if mn is None:
        return np.zeros(4, np.float32)
    return np.array([F32(mn[0]), F32(mn[1]), F32(mx[0]), F32(mx[1])], np.float32)


def disparity_range_mask(d, mn, mx):
    ch, _ = _types(d)
    mn, mx = np.asarray(mn, d.dtype), np.asarray(mx, d.dtype)
    m0 = ch(I32(int(mx[0]) - 1) if ch is I32 else F32(mx[0] - F32(1)))
    m1 = ch(I32(int(mx[1]) - 1) if ch is I32 else F32(mx[1] - F32(1)))
    out = d.copy()
    for j in range(d.shape[0]):
        for i in range(d.shape[1]):
            p = d[j, i]
            if p[2] == 0:
                continue
            ax, ay = F64(i) + F64(p[0]), F64(j) + F64(p[1])
            if ax < F64(mn[0]) or ax >= F64(m0) or ay < F64(mn[0]) or ay >= F64(m1):   # :278-279, m_min[0] for y
                out[j, i] = 0
    return out


def _apply(m, px, py):
    """HomographyTransform::forward / reverse with matrix m (Math/Transform.h:377-387)"""
    w = F64(F64(F64(m[2, 0] * px) + F64(m[2, 1] * py)) + m[2, 2])
    return (F64(F64(F64(m[0, 0] * px) + F64(m[0, 1] * py)) + m[0, 2]) / w,
            F64(F64(F64(m[1, 0] * px) + F64(m[1, 1] * py)) + m[1, 2]) / w)


def _to(ch, v):
    """the double -> channel conversion of C++: round to nearest float, or truncate toward zero (a NaN or out-of-range
    value gives INT32_MIN, as x86-64's cvttsd2si does)"""
    if ch is F32:
        return F32(v)
    return I32(math.trunc(float(v))) if -2147483649.0 < v < 2147483648.0 else I32(-2 ** 31)


def transform_lazy(m_inverse, d):
    """TransformDisparitiesFunc with the matrix reverse() applies"""
    ch, _ = _types(d)
    m = np.asarray(m_inverse, np.float64).reshape(3, 3)
    out = np.zeros_like(d)
    for j in range(d.shape[0]):
        for i in range(d.shape[1]):
            p = d[j, i]
            lx, ly = F64(i), F64(j)
            nx, ny = _apply(m, F64(lx + F64(p[0])), F64(ly + F64(p[1])))
            out[j, i] = (_to(ch, F64(nx - lx)), _to(ch, F64(ny - ly)), 1 if p[2] != 0 else 0)
    return out


def _round(v):
    """std::round: halves away from zero (the fraction of a double is exact)"""
    if not math.isfinite(v):
        return v
    a = math.floor(abs(v))
    return F64(math.copysign(a + 1 if abs(v) - a >= 0.5 else a, v))


def transform_explicit(do_round, origin, T, d):
    ch, _ = _types(d)
    m = np.asarray(T, np.float64).reshape(3, 3)
    out = np.zeros_like(d)
    for j in range(d.shape[0]):
        for i in range(d.shape[1]):
            p = d[j, i]
            if p[2] == 0:
                continue
            bx, by = F64(F64(origin[0]) + F64(i)), F64(F64(origin[1]) + F64(j))
            tx, ty = _apply(m, F64(bx + F64(p[0])), F64(by + F64(p[1])))
            dx, dy = F64(tx - bx), F64(ty - by)
            if do_round:
                dx, dy = _round(dx), _round(dy)
            out[j, i] = (_to(ch, dx), _to(ch, dy), 1)
    return out


def random_disparity(seed, shape, invalid, dtype, scale=40.0):
    """a random (rows, cols, 3) disparity with the given fraction of invalid pixels (keeping their values, and some with
    a valid word other than 1)"""
    rng = np.random.default_rng(seed)
    h, w = shape
    dx = rng.uniform(-scale, scale, (h, w))
    dy = rng.uniform(-scale / 4, scale / 4, (h, w))
    v = (rng.random((h, w)) >= invalid).astype(np.float64)
    v[(v != 0) & (rng.random((h, w)) < 0.1)] = 7
    if dtype == np.int32:
        return np.stack([np.rint(dx), np.rint(dy), v], -1).astype(np.int32)
    return np.stack([dx, dy, v], -1).astype(np.float32)
