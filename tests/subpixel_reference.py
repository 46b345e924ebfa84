"""A plain restatement of vw::stereo::ParabolaSubpixelView with PREFILTER_NONE in numpy, written from the reference
(Stereo/ParabolaSubpixelView.cc:31-330, .h:76-89, Math/Vector.h, Math/Matrix.h), independently of oracle/vw_oracle.c.

Per pixel of the bbox with a valid integer disparity d: the nine AbsoluteCost window sums at d + (-1..1, -1..1), each a
float |a - b| summed in double and stored in a Vector<float,9> (the zone loop of :74-218 only decides the order in which
they are computed); the 6x9 float pseudo-inverse times those nine floats; the peak of the fitted paraboloid, in float;
the offset kept when its norm is below 5.  Every float operation is done in numpy float32, which rounds each operation
correctly and never contracts a multiply and an add -- as the reference's scalar float code does on x86-64 -- so the
result is bit-exact.  The images are read through ConstantEdgeExtension (PreFilter.h:41-47: the nearest pixel), and the
window sums are only exact, hence independent of the reference's sliding order, for integer imagery or a 1x1 kernel
(asserted)."""
import numpy as np

from sgm_reference import PINV                 # the same literals, stored as Matrix<float,6,9> (.h:76-89)

F = np.float32
MAX_SUBPIXEL_SHIFT = F(5.0)                    # :253

BRANCHES = ("invalid", "all_equal", "kept", "too_far", "denom_zero")


def disparity_range(idisp, valid):
    """get_disparity_range (DisparityMap.h:52-66) over the valid pixels, then max += 1 and expand(1) (:287-289):
    (min_x, min_y, max_x, max_y) half-open.  No valid pixel: the empty range (0, 0, 0, 0) expanded."""
    if valid.any():
        dx, dy = idisp[..., 0][valid], idisp[..., 1][valid]
        lo, hi = (int(dx.min()), int(dy.min())), (int(dx.max()), int(dy.max()))
    else:
        lo = hi = (0, 0)
    return lo[0] - 1, lo[1] - 1, hi[0] + 2, hi[1] + 2


def fit(patch):
    """the fit of :242-254 on (N, 9) float32 cost patches: Matrix<float,6,9> * Vector<float,9> is dot_prod of each row
    (Math/Matrix.h:1977-1980, Math/Vector.h:1719-1726): a float product per entry, summed from 0.0f in index order.  Then
    denom = 4ab - c^2 and the offset (ce - 2bd, cd - 2ae) / denom, each operation in float, left to right.
    Returns (ox, oy, nn, denom) with nn = norm_2_sqr(offset) (Math/Vector.h:1593-1598): float squares summed in double, cast to
    float."""
    p = np.asarray(patch, F)
    x = []
    for r in range(6):
        acc = np.zeros(p.shape[0], F)
        for k in range(9):
            acc = acc + PINV[r, k] * p[:, k]
        x.append(acc)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        denom = F(4) * x[0] * x[1] - x[2] * x[2]
        ox = (x[2] * x[4] - F(2) * x[1] * x[3]) / denom
        oy = (x[2] * x[3] - F(2) * x[0] * x[4]) / denom
        nn = ((ox * ox).astype(np.float64) + (oy * oy).astype(np.float64)).astype(F)
    return ox, oy, nn, denom


def accepted(nn):
    """norm_2(offset) < MAX_SUBPIXEL_SHIFT: sqrt of the float squared norm in double, against 5.0f (NaN: not accepted)"""
    with np.errstate(invalid="ignore"):
        return np.sqrt(nn.astype(np.float64)) < np.float64(MAX_SUBPIXEL_SHIFT)


def refine(idisp, valid, patch, counts=None):
    """the output loop of :221-271 on (N,) integer disparities / validity and (N, 9) patches: (N, 3) float32"""
    idisp, valid, patch = np.asarray(idisp), np.asarray(valid, bool), np.asarray(patch, F)
    out = np.zeros((len(valid), 3), F)
    out[valid, :2] = idisp[valid].astype(F)
    out[valid, 2] = 1
    eq = (patch[:, 1:] == patch[:, :1]).all(1)                  # std::equal(begin + 1, end, begin)
    ox, oy, nn, denom = fit(patch)
    take = valid & ~eq & accepted(nn)
    out[take, 0] = idisp[take, 0].astype(F) + ox[take]           # Vector2i + Vector2f: float(d) + offset, in float
    out[take, 1] = idisp[take, 1].astype(F) + oy[take]
    if counts is not None:
        counts["invalid"] += int((~valid).sum())
        counts["all_equal"] += int((valid & eq).sum())
        counts["kept"] += int(take.sum())
        counts["too_far"] += int((valid & ~eq & ~take).sum())          # NaN offsets (0 / 0) included
        counts["denom_zero"] += int((valid & ~eq & (denom == 0)).sum())
    return out


def parabola_subpixel(disp, left, right, kernel, bbox=None, counts=None):
    """ParabolaSubpixelView(disp, left, right, PREFILTER_NONE, 0, kernel).prerasterize(bbox): disp (rows, cols, 3) float32
    {dx, dy, valid} the size of the left image (cropped into PixelMask<Vector2i>: the floats truncated), kernel (kx, ky),
    bbox (x0, y0, x1, y1) half-open.  Returns (bh, bw, 3) float32."""
    left, right = np.asarray(left, F), np.asarray(right, F)
    rows, cols = left.shape
    x0, y0, x1, y1 = bbox if bbox is not None else (0, 0, cols, rows)
    kx, ky = kernel
    assert kx * ky == 1 or (np.array_equal(left, np.floor(left)) and np.array_equal(right, np.floor(right))), \
        "a window of more than one pixel needs integer imagery"
    hx, hy = kx // 2, ky // 2
    d = np.asarray(disp, F)[y0:y1, x0:x1]
    idisp = d[..., :2].astype(np.int64)
    valid = d[..., 2] != 0
    bh, bw = y1 - y0, x1 - x0
    ys, xs = np.nonzero(valid)
    patch = np.zeros((bh * bw, 9), F)
    flat = (ys * bw + xs)
    wy, wx = np.mgrid[-hy:hy + 1, -hx:hx + 1]
    ly = np.clip(y0 + ys[:, None, None] + wy, 0, rows - 1)       # ConstantEdgeExtension of the left image
    lx = np.clip(x0 + xs[:, None, None] + wx, 0, cols - 1)
    lwin = left[ly, lx]
    for k in range(9):
        ex, ey = k % 3 - 1, k // 3 - 1                            # patch index = (ey + 1) * 3 + (ex + 1) (:187-205)
        ry = y0 + ys[:, None, None] + wy + idisp[ys, xs, 1][:, None, None] + ey
        rx = x0 + xs[:, None, None] + wx + idisp[ys, xs, 0][:, None, None] + ex
        # the windows of valid pixels stay inside the right image, where the crop of the edge-extended view (:297-298,
        # over disparity_range()) is the image itself
        assert (ry >= 0).all() and (rx >= 0).all() and (ry < right.shape[0]).all() and (rx < right.shape[1]).all(), \
            "a window leaves the right image"
        cost = np.abs(lwin - right[ry, rx]).astype(np.float64)   # float |a - b|, widened
        patch[flat, k] = cost.sum(axis=(1, 2)).astype(F)         # exact for integer imagery, stored as float
    out = refine(idisp.reshape(-1, 2), valid.ravel(), patch, counts)
    return out.reshape(bh, bw, 3)


# ---- test imagery -----------------------------------------------------------------------------------------------------------
VERTEX = np.array([1, 10, 21, 0, 9, 20, 1, 10, 21], F)      # z = x^2 + y^2 + 10 x + 9: the vertex at exactly (-5, 0)


def norm_edge_patches():
    """three perturbations of VERTEX whose float squared offset norm is one ulp below 25, exactly 25 and one ulp above
    (so the norm is just below 5, exactly 5 and just above).  Found by a fixed search with fit(): VERTEX alone gives
    (-5.0000005, 1.2e-7), and its x offset moves in steps of 2.5 ulps of 25 when the middle row moves by float ulps; the
    bottom row lifted by t (0 .. 0.02) adds a y offset of about -t / 4, whose square fills in the ulps between."""
    rng = np.random.default_rng(7)
    n = 20000
    cand = np.repeat(VERTEX[None], n, 0)
    cand[:, 6:] += np.linspace(0, 0.02, n, dtype=F)[:, None]
    cand[:, 3:6] = (cand[:, 3:6].view(np.int32) + rng.integers(-2, 3, (n, 3)).astype(np.int32)).view(F)
    _, _, nn, _ = fit(cand)
    out = []
    for target in (np.nextafter(F(25), F(0)), F(25), np.nextafter(F(25), F(100))):
        hit = np.nonzero(nn == target)[0]
        assert len(hit), f"no patch with squared norm {target!r}"
        out.append(cand[hit[0]])
    return np.stack(out)


def patch_set():
    """name -> (N, 9) float32 cost patches that reach every branch of the output loop"""
    rng = np.random.default_rng(8)
    eight = np.full((9, 9), 40, F)
    eight[np.arange(9), np.arange(9)] = 13                    # eight equal, the odd one at each of the nine places
    ridge = np.array([[3, 1, 3] * 3, [5, 2, 9] * 3, [0, 7, 7] * 3], F)   # three equal rows: b = c = 0
    bowls = rng.integers(0, 200, (64, 9)).astype(F)
    bowls[:, 4] = 0                                           # a minimum at the centre: offsets of either sign
    shifted = (rng.integers(0, 60, (64, 9)) + np.array([0, 5, 30, 5, 10, 35, 30, 35, 60])).astype(F)   # low corner at -1, -1
    return {"all_equal": np.full((2, 9), 17, F), "eight_equal": eight, "ridge": ridge, "bowls": bowls,
            "negative": shifted, "norm_edge": norm_edge_patches(), "vertex": VERTEX[None]}


def patch_raster(patches, disparity, step=4):
    """(disp, left, right) for a 1x1 kernel: left = 0, so the cost of disparity d at p is |right(p + d)|; each patch goes
    into right around p + disparity of its own valid pixel, on a grid of `step` pixels so that no two overlap.  Pixels
    off the grid are invalid."""
    n = len(patches)
    per_row = 8
    rows_, cols_ = (n + per_row - 1) // per_row * step + 6, per_row * step + 6
    dx, dy = disparity
    disp = np.zeros((rows_, cols_, 3), F)
    left = np.zeros((rows_, cols_), F)
    right = np.zeros((rows_ + max(dy, 0) + 6, cols_ + max(dx, 0) + 6), F)
    for i, p in enumerate(patches):
        y, x = 3 + (i // per_row) * step, 3 + (i % per_row) * step
        disp[y, x] = (dx, dy, 1)
        right[y + dy - 1:y + dy + 2, x + dx - 1:x + dx + 2] = np.asarray(p, F).reshape(3, 3)
    return disp, left, right


def integer_scene(seed, shape, base, spread, kernel, valid=0.9):
    """(disp, left, right) of integer imagery: right = left moved by base plus noise, on a canvas large enough that every
    window of a disparity base + (-spread - 1 .. spread + 1) stays inside it; integer disparities base + (-spread ..
    spread) per pixel, a fraction `valid` of them valid."""
    rng = np.random.default_rng(seed)
    rows_, cols_ = shape
    m = spread + 1 + max(kernel) // 2
    bx, by = base
    left = rng.integers(0, 256, (rows_, cols_)).astype(F)
    right = rng.integers(0, 256, (rows_ + abs(by) + 2 * m, cols_ + abs(bx) + 2 * m)).astype(F)
    oy, ox = max(by, 0), max(bx, 0)                           # right(p + base) = left(p) + noise where both exist
    ys, xs = np.mgrid[0:rows_, 0:cols_]
    ty, tx = ys + by, xs + bx
    ok = (ty >= 0) & (tx >= 0)
    right[ty[ok], tx[ok]] = np.clip(left[ok] + rng.integers(-6, 7, int(ok.sum())), 0, 255)
    disp = np.zeros((rows_, cols_, 3), F)
    disp[..., 0] = bx + rng.integers(-spread, spread + 1, shape)
    disp[..., 1] = by + rng.integers(-spread, spread + 1, shape)
    disp[..., 2] = rng.random(shape) < valid
    del oy, ox
    return disp, left, right
