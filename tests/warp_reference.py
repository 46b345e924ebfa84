"""An independent numpy restatement of transform(image, tx, edge, interp) (Image/Transform.h:485-601) on a float image: it walks
TransformView::operator() -> tx.reverse -> InterpolationView -> the interpolator -> EdgeExtensionView pixel by pixel, with
numpy float32 scalars where the reference computes in float and Python floats (IEEE double, no contraction) where it
computes in double.  Used to check the C oracle (oracle/vw_warp_oracle.c) on the cases of test_oracle_warp.py; it covers the
domain of the exactness contract only (finite reversed coordinates with |c| < 2^30)."""
import numpy as np

F = np.float32
HOMOGRAPHY, DISPARITY = 0, 1
BILINEAR, BICUBIC, NEAREST = 0, 1, 2
ZERO, CONSTANT = 0, 1
DOMAIN = 2.0 ** 30


def _floor(val):
    """math::impl::_floor(double) -> int32 (Math/Functions.h:74-81); int() truncates toward zero like int32(val)"""
    if val < 0:
        ival = int(val)
        return ival if float(ival) == val else ival - 1
    return int(val)


def _round(val):
    """math::impl::_round(double) (Math/Functions.h:48-51)"""
    return int(val - 0.5) if val < 0 else int(val + 0.5)


class EdgeView:
    """EdgeExtensionView<ImageView<PixelGray<float>>, EdgeT>"""

    def __init__(self, image, edge):
        self.im, self.edge = image, edge
        self.rows, self.cols = image.shape

    def __call__(self, i, j):
        if self.edge == ZERO:                                        # EdgeExtension.tcc:47-61
            if i >= 0 and j >= 0 and i < self.cols and j < self.rows:
                return F(self.im[j, i])
            return F(0.0)                                            # PixelGray<float>()
        ci = 0 if i < 0 else (self.cols - 1 if i >= self.cols else i)   # :89-94
        cj = 0 if j < 0 else (self.rows - 1 if j >= self.rows else j)
        return F(self.im[cj, ci])


class Accessor:
    """the ProceduralPixelAccessor of the edge-extended view: origin().advance(x, y), next_col(), advance(dc, dr)"""

    def __init__(self, view, c, r):
        self.v, self.c, self.r = view, c, r

    def next_col(self):
        self.c += 1

    def advance(self, dc, dr):
        self.c += dc
        self.r += dr

    def get(self):
        return self.v(self.c, self.r)


def bilinear(view, i, j):
    """BilinearInterpolationImpl (Image/Interpolation.h:76-110), real_type float"""
    x, y = _floor(i), _floor(j)
    if x == i and y == j:
        return view(x, y)
    normx, normy = F(F(i) - F(x)), F(F(j) - F(y))
    norm1mx, norm1my = F(F(1) - normx), F(F(1) - normy)
    acc = Accessor(view, x, y)
    result = F(acc.get() * norm1mx)
    acc.next_col()
    result = F(result + F(acc.get() * normx))
    result = F(result * norm1my)
    acc.advance(-1, 1)
    row = F(acc.get() * norm1mx)
    acc.next_col()
    row = F(row + F(acc.get() * normx))
    return F(result + F(row * normy))


def bicubic(view, i, j):
    """BicubicInterpolationImpl (Image/Interpolation.h:138-186), result_type double"""
    x, y = _floor(i), _floor(j)
    if x == i and y == j:
        return view(x, y)
    normx, normy = i - x, j - y
    s = (((2 - normx) * normx - 1) * normx, (3 * normx - 5) * normx * normx + 2, ((4 - 3 * normx) * normx + 1) * normx, (normx - 1) * normx * normx)
    t = (((2 - normy) * normy - 1) * normy, (3 * normy - 5) * normy * normy + 2, ((4 - 3 * normy) * normy + 1) * normy, (normy - 1) * normy * normy)
    acc = Accessor(view, x - 1, y - 1)
    result = None
    for k in range(4):
        if k:
            acc.advance(-3, 1)
        row = s[0] * float(acc.get())
        for c in range(1, 4):
            acc.next_col()
            row += s[c] * float(acc.get())
        result = t[k] * row if result is None else result + t[k] * row
    result *= 0.25
    return F(result)


def nearest(view, i, j):
    """NearestPixelInterpolation (Image/Interpolation.h:209-225)"""
    return view(_round(i), _round(j))


INTERP = {BILINEAR: bilinear, BICUBIC: bicubic, NEAREST: nearest}


def homography_reverse(m):
    """HomographyTransform::reverse (Math/Transform.h:377-381); m = m_H_inverse"""
    m = [[float(m[r][c]) for c in range(3)] for r in range(3)]

    def rev(px, py):
        w = np.float64(m[2][0] * px + m[2][1] * py + m[2][2])                # numpy: w == 0 gives inf / NaN, not an exception
        return float((m[0][0] * px + m[0][1] * py + m[0][2]) / w), float((m[1][0] * px + m[1][1] * py + m[1][2]) / w)
    return rev


def disparity_reverse(disparity):
    """DisparityTransform::reverse (Stereo/DisparityMap.h:1177-1182): the offset image is read with NearestPixelInterpolation
    over ZeroEdgeExtension, whose outside pixel is an invalid PixelMask"""
    d = np.asarray(disparity, np.float32)
    rows, cols = d.shape[:2]

    def rev(px, py):
        x, y = _round(px), _round(py)
        if not (x >= 0 and y >= 0 and x < cols and y < rows) or d[y, x, 2] == 0:
            return -1.0, py
        return px + float(d[y, x, 0]), py + float(d[y, x, 1])
    return rev


def transform(image, kind, interp, edge, window, matrix=None, disparity=None):
    """the TransformView pixels of window (x0, y0, ow, oh), float32 (oh, ow), and a boolean mask of the pixels inside the
    contract's domain (the others are left 0 here)"""
    view = EdgeView(np.asarray(image, np.float32), edge)
    rev = homography_reverse(matrix) if kind == HOMOGRAPHY else disparity_reverse(disparity)
    x0, y0, ow, oh = window
    out = np.zeros((oh, ow), np.float32)
    inside = np.zeros((oh, ow), bool)
    with np.errstate(all="ignore"):
        for jj in range(oh):
            for ii in range(ow):
                rx, ry = rev(float(x0 + ii), float(y0 + jj))
                if abs(rx) < DOMAIN and abs(ry) < DOMAIN:
                    out[jj, ii] = INTERP[interp](view, rx, ry)
                    inside[jj, ii] = True
    return out, inside
