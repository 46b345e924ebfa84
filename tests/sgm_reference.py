"""A plain restatement of the SemiGlobalMatcher core in numpy and Python integers, written from the reference
(Stereo/SGM.cc, Stereo/SGMAssist.h, Image/CensusTransform.h), independently of oracle/vw_sgm_oracle.c.

It exists to check the oracle, and through it the device kernels, where the penalties are large enough for the uint16
accumulation to wrap.  It is slow by design -- a full search volume per pixel, one Python step per scan line -- so it is
meant for rasters of a few thousand output pixels and search boxes of a few hundred disparities.

Covered: binary census 3/5/7/9 with Hamming costs, 8-bit imagery whose u8 stretch is the identity, the SSE flavour of
evaluate_path along all 8 directions, the uint16 accumulation kept both wrapped and unwrapped, and select_best_disparity
with its tie smoothing.  Not covered: ternary census, MGM, masks, the previous-level boxes and the sub-pixel stage."""
import math
from typing import NamedTuple

import numpy as np

U16 = 0xFFFF

# SemiGlobalMatcher::set_parameters, CENSUS_TRANSFORM rows (SGM.cc:106-160): p1 / p2 <= 0 select these
DEFAULT_P1 = {3: 3, 5: 15, 7: 30, 9: 20}
DEFAULT_P2 = {3: 70, 5: 750, 7: 1500, 9: 1000}

# get_census_value_9x9 (CensusTransform.h:112-160): the 32 positions of the 9x9 pattern, bit i = position i
C9_COLS = (0, 4, 8, 1, 3, 5, 7, 2, 4, 6, 1, 4, 7, 0, 2, 3, 5, 6, 8, 1, 4, 7, 2, 4, 6, 1, 3, 5, 7, 0, 4, 8)
C9_ROWS = (0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4, 4, 4, 4, 5, 5, 5, 6, 6, 6, 7, 7, 7, 7, 8, 8, 8)

# the eight scan directions of accum_sgm_multithread (SGM.cc:2488-2610) as (column step, row step)
DIRECTIONS = ((0, 1), (0, -1), (1, 0), (-1, 0), (1, 1), (-1, 1), (1, -1), (-1, -1))


def penalties(kernel, p1=0, p2=0):
    """(P1, P2) after the defaults of set_parameters (SGM.cc:106-160)."""
    return (p1 if p1 > 0 else DEFAULT_P1[kernel], p2 if p2 > 0 else DEFAULT_P2[kernel])


def as_u8(img):
    """The u8 stretch of calc_disparity_sgm (SGM.cc:211-212, ImageThresh.h u8_convert) maps [min, max] onto [0, 255].
    This restatement only takes imagery on which that is the identity: integer values in 0..255 with both 0 and 255
    present.  Asserted, so that a caller cannot hand it imagery the stretch would change."""
    a = np.asarray(img)
    assert np.array_equal(a, np.floor(a)) and a.min() == 0 and a.max() == 255, "the u8 stretch is not the identity on this image"
    return a.astype(np.int64)


def census_offsets(k):
    """(row, column) offsets of the census neighbours, bit 0 first: 3x3 / 5x5 / 7x7 take every neighbour in reverse raster
    order, starting at (+hk, +hk) (CensusTransform.h:64-110); 9x9 takes the 32-position pattern."""
    if k == 9:
        return [(r - 4, c - 4) for c, r in zip(C9_COLS, C9_ROWS)]
    hk = k // 2
    return [(dr, dc) for dr in range(hk, -hk - 1, -1) for dc in range(hk, -hk - 1, -1) if (dr, dc) != (0, 0)]


def census_bits(img8, k):
    """(h - 2 hk, w - 2 hk, bits) bools: neighbour strictly greater than the centre.  Element (r, c) belongs to image pixel
    (c + hk, r + hk), as in fill_costs_census* (SGM.cc:1740-1871)."""
    hk = k // 2
    h, w = img8.shape
    ctr = img8[hk:h - hk, hk:w - hk]
    return np.stack([img8[hk + dr:h - hk + dr, hk + dc:w - hk + dc] > ctr for dr, dc in census_offsets(k)], -1)


def census_value(img8, col, row, k):
    """The census signature of one pixel as the reference's integer (bit i = offset i of census_offsets)."""
    ctr = img8[row, col]
    return sum(1 << i for i, (dr, dc) in enumerate(census_offsets(k)) if img8[row + dr, col + dc] > ctr)


def output_shape(lshape, rshape, search, k):
    """(rows, cols) of the output raster (SGM.cc:2404-2420, minimum disparity 0)."""
    hk = k // 2
    return (min(lshape[0] - 1 - hk, rshape[0] - 1 - (hk + search[1])) - hk + 1,
            min(lshape[1] - 1 - hk, rshape[1] - 1 - (hk + search[0])) - hk + 1)


def cost_volume(l8, r8, search, k):
    """Hamming distance of the census signatures (get_hamming_distance_costs, SGM.cc:40-75) for every disparity of the
    search box [0, sx] x [0, sy]: (oh, ow, sy + 1, sx + 1) int64."""
    oh, ow = output_shape(l8.shape, r8.shape, search, k)
    lb, rb = census_bits(l8, k)[:oh, :ow], census_bits(r8, k)
    cost = np.empty((oh, ow, search[1] + 1, search[0] + 1), np.int64)
    for dy in range(search[1] + 1):
        for dx in range(search[0] + 1):
            cost[:, :, dy, dx] = np.count_nonzero(lb != rb[dy:dy + oh, dx:dx + ow], axis=-1)
    return cost


def box_mask(bounds, search):
    """(oh, ow, sy + 1, sx + 1) bools: the disparity lies in the pixel's box {min_x, min_y, max_x, max_y} (inclusive)."""
    dx = np.arange(search[0] + 1)[None, None, None, :]
    dy = np.arange(search[1] + 1)[None, None, :, None]
    b = bounds[:, :, None, None, :]
    return (dx >= b[..., 0]) & (dx <= b[..., 2]) & (dy >= b[..., 1]) & (dy <= b[..., 3])


def evaluate_path(prior, prior_in_box, local, gradient, p1, p2):
    """evaluate_path, SSE flavour (SGM.cc:1014-1149, compute_path_internals_sse :937-983), for N pixels at once.

    prior: (N, ndy, ndx) path costs of the previous pixel of each line, valid where prior_in_box; local: (N, ndy, ndx) costs
    of the current pixel; gradient: (N,) |intensity change| along the path.  Returns (N, ndy, ndx) path costs; only the
    entries inside the current pixel's box mean anything."""
    bad = (255 + p2) & U16                                          # get_bad_accum_val (SGM.h:240)
    full = np.where(prior_in_box, prior, bad)                       # full_prior_buffer: BAD outside the previous box
    min_prior = np.minimum(full.min(axis=(1, 2)), bad)[:, None, None]
    p2_mod = np.where(gradient > 0, p2 // np.maximum(gradient, 1), p2)
    p2_mod = np.maximum(p2_mod, p1)[:, None, None]
    dJ = (min_prior + p2_mod) & U16                                 # min_prev_disparity_cost, a uint16
    # the 8 adjacent disparities; the lookup table clamps at the edges of the search box to the entry itself (:760-799)
    pad = np.pad(full, ((0, 0), (1, 1), (1, 1)), mode="edge")
    ny, nx = full.shape[1:]
    adj = None
    for oy, ox in ((0, 1), (1, 0), (1, 2), (2, 1), (0, 0), (0, 2), (2, 0), (2, 2)):
        v = pad[:, oy:oy + ny, ox:ox + nx]
        adj = v if adj is None else np.minimum(adj, v)
    res = np.minimum(adj + p1, U16)                                 # _mm_adds_epu16(minAdj, dp1)
    res = np.minimum(res, np.minimum(full, dJ))                     # min(.., d0, dJ)
    res = np.minimum(res + local, U16)                              # _mm_adds_epu16(.., dL)
    return np.maximum(res - min_prior, 0)                           # _mm_subs_epu16(.., dP)


def path_costs(cost, inbox, val, p1, p2, direction):
    """One direction of accum_sgm_multithread: every pixel lies on one line; the first pixel of a line takes its local cost
    (SGMAssist.h:752-759), every later one evaluate_path with the intensity change from its predecessor (:749-755)."""
    dc, dr = direction
    if dr == 0:                              # along rows: process columns in order, each as a vector over the rows
        cost, inbox, val = cost.transpose(1, 0, 2, 3), inbox.transpose(1, 0, 2, 3), val.T
        step, shift = dc, 0
    else:                                    # process rows in order; item i follows item i - dc of the previous row
        step, shift = dr, dc
    n0, n1 = cost.shape[:2]
    out = np.empty_like(cost)
    order = range(n0) if step > 0 else range(n0 - 1, -1, -1)
    items = np.arange(n1)
    for i, s in enumerate(order):
        res = cost[s].copy()                 # line starts
        if i:
            j = items - shift
            has = (j >= 0) & (j < n1)
            pj = j[has]
            q = s - step
            res[has] = evaluate_path(out[q][pj], inbox[q][pj], cost[s][has], np.abs(val[s][has] - val[q][pj]), p1, p2)
        out[s] = res
    return out.transpose(1, 0, 2, 3) if dr == 0 else out


def _c_round(x):
    f = math.floor(x)
    return f + 1 if x - f >= 0.5 else f      # C round() of a non-negative double: halves away from zero


def select_best_disparity(vals, wrap=True):
    """select_best_disparity (SGM.cc:1159-1284) on one pixel's box of accumulated costs, (h, w) row-major.
    Returns (min_index, smoothed, lowest cost before smoothing).  When the minimum is tied, 3-tap box filters (horizontal
    five times, then vertical) run until one minimum is left, at most six times."""
    h, w = vals.shape
    cur = [int(v) for v in vals.ravel()]
    lo = min(cur)
    if cur.count(lo) == 1:
        return cur.index(lo), False, lo
    third = 1.0 / 3.0
    min_count, it, min_index = 2, 0, 0
    while min_count > 1:
        nxt = []
        for idx in range(h * w):
            row, col = divmod(idx, w)
            pos, length, stride = (col, w, 1) if it < 5 else (row, h, w)
            kmin = 0 if pos - 1 < 0 else -1
            kmax = 0 if pos + 1 >= length else 1
            result = weight = 0.0
            for k in range(kmin, kmax + 1):
                result += float(cur[idx + k * stride]) * third
                weight += third
            v = _c_round(result / weight)
            nxt.append(v & U16 if wrap else v)
        cur = nxt
        m = min(cur)
        min_count, min_index = cur.count(m), cur.index(m)
        it += 1
        if it >= 6:
            break
    return min_index, True, lo


class SgmResult(NamedTuple):
    disparity: np.ndarray   # (oh, ow, 3) int32 {dx, dy, valid} from the uint16 (wrapping) accumulation, as the reference
    unwrapped: np.ndarray   # the same from an int64 accumulation that never wraps
    smoothed: np.ndarray    # (oh, ow) bool: the wrapped winner went through the tie smoothing
    lowest: np.ndarray      # (oh, ow) int64: lowest wrapped accumulated cost of the box (-1 where the box is empty)
    max_sum: int            # largest unwrapped 8-path sum over every (pixel, disparity) inside a box


def sgm(left, right, search, kernel, bounds=None, p1=0, p2=0):
    """calc_disparity_sgm (SGM.cc:167-230 -> semi_global_matching_func :2387-2448) with CENSUS_TRANSFORM, plain SGM and
    integer disparities.  left / right: the left_region / right_region rasters; bounds: (oh, ow, 4) boxes, or None for the
    whole search box [0, search] at every pixel."""
    assert kernel in (3, 5, 7, 9)
    p1, p2 = penalties(kernel, p1, p2)
    l8, r8 = as_u8(left), as_u8(right)
    cost = cost_volume(l8, r8, search, kernel)
    oh, ow = cost.shape[:2]
    if bounds is None:
        bounds = np.tile(np.array([0, 0, search[0], search[1]], np.int64), (oh, ow, 1))
    bounds = np.asarray(bounds, np.int64)
    assert bounds.shape == (oh, ow, 4)
    inbox = box_mask(bounds, search)
    hk = kernel // 2
    val = l8[hk:hk + oh, hk:hk + ow]         # the intensity of the left u8 image under each output pixel
    wrapped = np.zeros(cost.shape, np.int64)
    total = np.zeros(cost.shape, np.int64)
    for d in DIRECTIONS:
        p = path_costs(cost, inbox, val, p1, p2, d)
        wrapped = (wrapped + p) & U16        # update_accum_buffer (SGMAssist.h:792-819): uint16 +=
        total += p
    disp = np.zeros((oh, ow, 3), np.int32)
    disp_u = np.zeros((oh, ow, 3), np.int32)
    smoothed = np.zeros((oh, ow), bool)
    lowest = np.full((oh, ow), -1, np.int64)
    for r in range(oh):
        for c in range(ow):
            x0, y0, x1, y1 = (int(v) for v in bounds[r, c])
            if x1 < x0 or y1 < y0:           # no search area: invalid (create_disparity_view, :1317-1336)
                continue
            w = x1 - x0 + 1
            i, smoothed[r, c], lowest[r, c] = select_best_disparity(wrapped[r, c, y0:y1 + 1, x0:x1 + 1])
            disp[r, c] = (x0 + i % w, y0 + i // w, 1)
            i, _, _ = select_best_disparity(total[r, c, y0:y1 + 1, x0:x1 + 1], wrap=False)
            disp_u[r, c] = (x0 + i % w, y0 + i // w, 1)
    return SgmResult(disp, disp_u, smoothed, lowest, int(np.where(inbox, total, 0).max()))


def assert_wrap_decides(res):
    """The uint16 accumulation wraps on these inputs, and the wrap changes the winner at >= 1 % of the pixels -- so a
    kernel that carried into the neighbouring halfword, or saturated, would not go unnoticed."""
    assert res.max_sum > U16, f"largest 8-path sum {res.max_sum}: nothing wraps"
    frac = float((res.disparity != res.unwrapped).any(-1).mean())
    assert frac >= 0.01, f"the wrap changes only {frac:.4f} of the winners"


# ---- imagery on which the penalties, not the costs, dominate ---------------------------------------------------------------
def flat_pair(seed, oh, ow, search, kernel, off=(3, 2), levels=4):
    """left_region / right_region rasters for an (oh, ow) output: a random texture of `levels` grey values around 100, so
    neighbouring pixels differ by less than `levels` and p2_mod stays close to P2 along every path; left(c, r) =
    right(c + off_x, r + off_y), the offset clipped to the search box.  One 0 and one 255 in a corner of each (outside every census window's centre) make the
    u8 stretch the identity."""
    rng = np.random.default_rng(seed)
    hk = kernel // 2
    lh, lw = oh + 2 * hk, ow + 2 * hk
    off = (min(off[0], search[0]), min(off[1], search[1]))
    right = (100 + rng.integers(0, levels, (lh + search[1], lw + search[0]))).astype(np.float32)
    left = right[off[1]:off[1] + lh, off[0]:off[0] + lw].copy()
    for im in (left, right):
        im[0, 0] = 0
        im[-1, -1] = 255
    return np.ascontiguousarray(left), np.ascontiguousarray(right)


def moving_boxes(seed, oh, ow, search, maxw, maxh, empty=0.03):
    """A box of 1..maxw x 1..maxh disparities at a random place of the search box for every pixel, so that neighbouring
    boxes rarely overlap: entries new to a path start from BAD = 255 + P2, which drives the path costs towards P2.  A few
    pixels have no box."""
    rng = np.random.default_rng(seed)
    b = np.zeros((oh, ow, 4), np.int32)
    b[..., 0] = rng.integers(0, search[0] + 1, (oh, ow))
    b[..., 1] = rng.integers(0, search[1] + 1, (oh, ow))
    b[..., 2] = np.minimum(b[..., 0] + rng.integers(0, maxw, (oh, ow)), search[0])
    b[..., 3] = np.minimum(b[..., 1] + rng.integers(0, maxh, (oh, ow)), search[1])
    b[rng.random((oh, ow)) < empty] = (0, 0, -1, -1)
    return b
