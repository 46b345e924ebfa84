"""Numpy restatement of fill_holes_grass (src/vw/Image/InpaintView.h:239-311), written apart from oracle/vw_inpaint_oracle.c
so the two can be checked against each other bit for bit.  Small images only: the sweeps are scalar Python loops.

The holes are labelled by scipy.ndimage.label with a 3 x 3 structure (8-connected components, what BlobIndex yields), the
grassfire is the literal two passes of Grassfire.h:79-150, and each stencil product is an np.float64 added to an np.float32
accumulator through np.float64, as `AccumulatorType sum; sum += .176765 * pixel` does (ProductType<double, channel> is
double, and `float += double` rounds the double sum to float)."""
import numpy as np
from scipy import ndimage

CORNER, EDGE = np.float64(.176765), np.float64(.073235)
# the accessor walk of InpaintView.h:119-135: (dx, dy, weight)
STENCIL = [(-1, -1, CORNER), (0, -1, EDGE), (1, -1, CORNER), (-1, 0, EDGE), (1, 0, EDGE), (-1, 1, CORNER), (0, 1, EDGE),
           (1, 1, CORNER)]


def grassfire(mask):
    """grassfire(mask) without ignore_borders: int32 city-block distance of each non-zero pixel to a zero one."""
    rows, cols = mask.shape
    d = np.zeros((rows, cols), np.int64)
    if cols <= 1 or rows <= 1:
        return d
    for c in range(cols):
        d[0, c] = 1 if mask[0, c] else 0
        d[rows - 1, c] = 1 if mask[rows - 1, c] else 0
    for r in range(1, rows - 1):
        d[r, 0] = 1 if mask[r, 0] else 0
        for c in range(1, cols - 1):
            d[r, c] = 0 if not mask[r, c] else 1 + min(d[r, c - 1], d[r - 1, c])
        d[r, cols - 1] = 1 if mask[r, cols - 1] else 0
    for r in range(rows - 2, 0, -1):
        for c in range(cols - 2, 0, -1):
            if d[r, c] != 0:
                m = min(d[r, c + 1], d[r + 1, c])
                if m < d[r, c]:
                    d[r, c] = m + 1
    return d


def holes(tile_valid, length):
    """the holes BlobIndexThreaded(invert_mask(tile), len*len).wipe_big_blobs(len) keeps: a list of (pixel mask, (x0, y0, x1, y1))"""
    lbl, n = ndimage.label(~tile_valid, structure=np.ones((3, 3), int))
    out = []
    for k in range(1, n + 1):
        m = lbl == k
        ys, xs = np.nonzero(m)
        box = (xs.min(), ys.min(), xs.max() + 1, ys.max() + 1)
        if length * length > 0 and m.sum() > length * length:
            continue
        if box[2] - box[0] > length or box[3] - box[1] > length:
            continue
        out.append((m, box))
    return out


def inpaint(tile, m, box):
    """InpaintTask on one hole: returns (crop origin, filled crop, crop mask), or None for a skipped hole"""
    rows, cols = tile.shape[:2]
    x0, y0, x1, y1 = box[0] - 1, box[1] - 1, box[2] + 1, box[3] + 1
    if x0 < 0 or y0 < 0 or x1 >= cols or y1 >= rows:
        return None
    crop = tile[y0:y1, x0:x1, :2].copy()
    mask = m[y0:y1, x0:x1]
    dist = grassfire(mask)
    dmax = int(dist.max())
    order = [(i, j) for d in range(1, dmax + 1) for i in range(crop.shape[1]) for j in range(crop.shape[0]) if dist[j, i] == d]
    for _ in range(10 * dmax * dmax):
        for i, j in order:
            for c in range(2):
                s = np.float32(0)
                for dx, dy, wt in STENCIL:
                    s = np.float32(np.float64(s) + wt * np.float64(crop[j + dy, i + dx, c]))
                if crop.dtype == np.int32:
                    crop[j, i, c] = np.int32(np.trunc(np.float64(s)))
                else:
                    crop[j, i, c] = s
    return (x0, y0), crop, mask


def fill_holes_grass(disp, length, window=None):
    """FillHolesGrass(disp, len) over window (x0, y0, ow, oh); disp is (rows, cols, 3) int32 or float32"""
    rows, cols = disp.shape[:2]
    x0, y0, ow, oh = (0, 0, cols, rows) if window is None else window
    tx0, ty0 = max(x0 - length, 0), max(y0 - length, 0)
    tx1, ty1 = min(x0 + ow + length, cols), min(y0 + oh + length, rows)
    tile = disp[ty0:ty1, tx0:tx1].copy()
    res = tile.copy()
    with np.errstate(invalid="ignore", over="ignore"):
        for m, box in holes(tile[..., 2] != 0, length):
            r = inpaint(tile, m, box)
            if r is None:
                continue
            (cx, cy), crop, mask = r
            sub = res[cy:cy + crop.shape[0], cx:cx + crop.shape[1]]
            sub[mask, :2] = crop[mask]
            sub[mask, 2] = 1
    return res[y0 - ty0:y0 - ty0 + oh, x0 - tx0:x0 - tx0 + ow].copy()
