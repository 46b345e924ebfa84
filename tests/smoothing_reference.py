"""Restatement of the reference's disparity smoothing filters (Stereo/Algorithms.cc:26-67, Algorithms.h:144-281), written
straight from the C++ loops for small images: Python floats are the reference's doubles, numpy float32 scalars its floats.

Both disparity filters start with `disparity_out = disparity_in;`.  ImageView has no non-template copy assignment of its
own (Image/ImageView.h:95-148), so the implicitly-declared one runs and `out` shares `in`'s buffer: the filters work in
place, in raster order, and every window reads the already-filtered pixels above and to the left.  `jacobi=True` reads all
windows from the unfiltered input instead; it is not what the reference computes and exists only as a contrast for tests.

Disparities are float32 (h, w, 3) {dx, dy, valid} arrays; valid means valid != 0."""
import math

import numpy as np

F = np.float32


def destructive_median(values):
    """math::destructive_median (Math/Functors.h:393-398): sort, the middle value, or the mean of the middle two"""
    v = sorted(float(x) for x in values)
    n = len(v)
    assert n, "median: no valid samples."
    return v[n // 2] if n % 2 else (v[n // 2 - 1] + v[n // 2]) / 2.0


def disparity_median_filter(disparity, kernel_size, jacobi=False):
    """disparity_median_filter (Algorithms.cc:26-67) on a copy; returns the copy"""
    out = np.array(disparity, F, copy=True)
    src = np.array(disparity, F, copy=True) if jacobi else out
    if kernel_size < 3:
        return out
    half = (kernel_size - 1) // 2
    h, w = out.shape[:2]
    for row in range(half, h - half):
        for col in range(half, w - half):
            if src[row, col, 2] == 0:
                continue
            dx, dy = [], []
            for r in range(row - half, row + half + 1):
                for c in range(col - half, col + half + 1):
                    if src[r, c, 2] != 0:
                        dx.append(float(src[r, c, 0]))
                        dy.append(float(src[r, c, 1]))
            if not dx:
                continue
            out[row, col] = (F(destructive_median(dx)), F(destructive_median(dy)), F(1))
    return out


def derivative(img, axis):
    """derivative_filter(img, 1, 0) (axis=1) or (img, 0, 1) (axis=0) of a float image (Image/Filter.h:304-308,
    Filter.tcc:91-118, Convolution.h:53-65,275-297): kernel {0.5, 0, -0.5} applied reversed to the clamped neighbours,
    accumulated in float from 0"""
    a = np.asarray(img, F)
    n = a.shape[axis]
    idx = np.arange(n)
    lo = np.take(a, np.clip(idx - 1, 0, n - 1), axis=axis)
    mid = a
    hi = np.take(a, np.clip(idx + 1, 0, n - 1), axis=axis)
    r = F(0) + F(-0.5) * lo
    r = r + F(0) * mid
    return (r + F(0.5) * hi).astype(F)


def texture_measure(image, kernel_size=9, gradient_weight=0.5, stddev_weight=0.5):
    """texture_measure (Algorithms.h:144-209) of a plain float image (every pixel valid)"""
    img = np.asarray(image, F)
    h, w = img.shape
    half = (kernel_size - 1) // 2
    gx, gy = derivative(img, 1), derivative(img, 0)
    g = (np.abs(gx) + np.abs(gy)).astype(F)              # std::abs(dx) + std::abs(dy): a float add, widened after
    out = np.empty((h, w), F)
    for row in range(h):
        for col in range(w):
            win = [(min(max(r, 0), h - 1), min(max(c, 0), w - 1))
                   for r in range(row - half, row + half + 1) for c in range(col - half, col + half + 1)]
            mean, count = 0.0, 0.0
            for r, c in win:
                mean += float(img[r, c])
                count += 1.0
            mean /= count
            grad, sd = 0.0, 0.0
            for r, c in win:
                grad += float(g[r, c])
                e = float(img[r, c]) - mean
                sd += e * e
            grad = grad / (2.0 * count)
            sd = math.sqrt(sd / count)
            out[row, col] = F(grad * gradient_weight + sd * stddev_weight)
    return out


def texture_kernel_size(t, texture_max, max_kernel_size):
    """the per-pixel kernel of Algorithms.h:222,243-257 in float arithmetic, or None where the pixel is skipped"""
    t, texture_max = F(t), F(texture_max)
    if t < 0:
        return None
    with np.errstate(all="ignore"):
        scale = F(F(max_kernel_size) / texture_max)
        adj = F(texture_max - t)
        if adj < 0:
            adj = F(0)
        f = np.floor(F(adj * scale))
    k = int(f) if np.isfinite(f) and -2.0 ** 31 <= f < 2.0 ** 31 else -2 ** 31     # x86-64 cvttss2si: INT_MIN
    if k % 2 == 0:
        k += 1
    if k < 3 or k > max_kernel_size:
        return None
    return k


def texture_preserving_disparity_filter(disparity, texture_image, texture_max=0.15, max_kernel_size=11, jacobi=False):
    """texture_preserving_disparity_filter<float> (Algorithms.h:213-281) on a copy; returns the copy"""
    out = np.array(disparity, F, copy=True)
    src = np.array(disparity, F, copy=True) if jacobi else out
    tex = np.asarray(texture_image, F)
    if max_kernel_size < 3 or F(texture_max) <= 0:
        return out
    h, w = out.shape[:2]
    for row in range(h):
        for col in range(w):
            if src[row, col, 2] == 0:
                continue
            k = texture_kernel_size(tex[row, col], texture_max, max_kernel_size)
            if k is None:
                continue
            half = (k - 1) // 2
            sx, sy, count = 0.0, 0.0, 0.0
            for r in range(row - half, row + half + 1):
                for c in range(col - half, col + half + 1):
                    q = src[min(max(r, 0), h - 1), min(max(c, 0), w - 1)]
                    if q[2] != 0:
                        sx += float(q[0])
                        sy += float(q[1])
                        count += 1.0
            if count < 1.0:
                continue
            out[row, col] = (F(sx / count), F(sy / count), F(1))
    return out


def random_disparity(seed, shape, invalid=0.1, spread=8.0, integer=False):
    """float32 (h, w, 3) {dx, dy, valid}: a smooth ramp plus noise, a fraction `invalid` of the pixels invalid (their
    dx / dy hold junk, which the filters must leave alone)"""
    rng = np.random.default_rng(seed)
    h, w = shape
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    d = np.empty((h, w, 3), F)
    d[..., 0] = 0.05 * xx - 3.0 + rng.normal(0, spread / 4, shape)
    d[..., 1] = -0.03 * yy + 1.5 + rng.normal(0, spread / 8, shape)
    if integer:
        d[..., :2] = np.rint(d[..., :2])
    d[..., 2] = (rng.random(shape) >= invalid).astype(F)
    bad = d[..., 2] == 0
    d[..., 0][bad] = rng.normal(0, 100, int(bad.sum()))
    d[..., 1][bad] = -7.25
    return d
