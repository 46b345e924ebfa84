"""A plain restatement of the SemiGlobalMatcher core in numpy and Python integers, written from the reference
(Stereo/SGM.cc, Stereo/SGMAssist.h, Image/CensusTransform.h), independently of oracle/vw_sgm_oracle.c.

It exists to check the oracle, and through it the device kernels, where the penalties are large enough for the uint16
accumulation to wrap.  It is slow by design -- a full search volume per pixel, one Python step per scan line -- so it is
meant for rasters of a few thousand output pixels and search boxes of a few hundred disparities.

Covered: binary census 3/5/7/9 with Hamming costs, 8-bit imagery whose u8 stretch is the identity, the SSE flavour of
evaluate_path along all 8 directions, the uint16 accumulation kept both wrapped and unwrapped, select_best_disparity
with its tie smoothing (and the smoothed box it leaves behind), and the sub-pixel stage create_disparity_view_subpixel:
the four 1-D models with the two-value rule at a bound, and ParabolaFit2d::find_peak, every branch counted (BRANCHES).
Not covered: ternary census, MGM, masks and the previous-level boxes."""
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


def select_best_disparity(vals, wrap=True, return_box=False):
    """select_best_disparity (SGM.cc:1159-1284) on one pixel's box of accumulated costs, (h, w) row-major.
    Returns (min_index, smoothed, lowest cost before smoothing), and with return_box the box as the reference leaves it in
    accum_vec (a flat list): the input when the minimum is unique, else the last smoothing pass -- odd passes write into
    accum_vec itself, even ones into the buffer, which is then copied back (:1277-1281).  When the minimum is tied, 3-tap
    box filters (horizontal five times, then vertical) run until one minimum is left, at most six times."""
    h, w = vals.shape
    cur = [int(v) for v in vals.ravel()]
    lo = min(cur)
    if cur.count(lo) == 1:
        return (cur.index(lo), False, lo, cur) if return_box else (cur.index(lo), False, lo)
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
    return (min_index, True, lo, cur) if return_box else (min_index, True, lo)


# ---- the sub-pixel stage: create_disparity_view_subpixel (SGM.cc:1497-1614) -----------------------------------------------
PI = 3.14159265359                            # the literal of sinFit / cosFit / lcBlendFit (:1421-1432), not math.pi

# the branches of the sub-pixel stage, counted per call of compute_subpixel_offset (1-D models, once per axis) or per
# pixel (the 2-D fit, and winners that went through the tie smoothing)
BRANCHES = ("both_bounds", "two_value_left", "two_value_right", "ld_lt_rd", "ld_gt_rd", "ld_eq_rd",
            "fit_rejected", "fit_rescaled", "fit_kept", "smoothed_winner")


def _fit(x, mode):
    """linearFit / poly4Fit / cosFit / lcBlendFit (:1411-1436), in double, in the reference's operation order"""
    if mode == 3:
        return (x * x * x * x + x) / 4.0
    if mode == 4:
        return 1 - math.cos(x * PI / 3.0)
    if mode == 5:
        factor = 1.195 - math.cos(x * (PI / 2.3))
        return (1 - math.cos(x * PI / 3.0)) * factor + (x / 2.0) * (1.0 - factor)
    return x / 2.0                            # SUBPIXEL_LINEAR, and the default of the switch


def compute_subpixel_offset(prev, center, nxt, left_bound, right_bound, mode, counts=None):
    """compute_subpixel_offset (:1445-1479): prev / center / next are uint16 accumulated costs; the differences are taken
    in int and converted to double.  At a bound only two values are available (two_value_subpixel, :1440-1442); inside,
    the model is applied to the ratio of the smaller difference to the larger one, towards the lower neighbour."""
    def count(k):
        if counts is not None:
            counts[k] += 1
    ld, rd = float(int(prev) - int(center)), float(int(nxt) - int(center))
    if rd == 0 and ld == 0:                   # all values equal, or both bounds (prev = center = next)
        count("both_bounds")
        return 0.0
    if left_bound:
        count("two_value_left")
        return 0.5 * (float(center) / float(nxt))
    if right_bound:
        count("two_value_right")
        return -1.0 * (0.5 * (float(center) / float(prev)))
    x, mult = rd / ld, -1.0
    if ld < rd:
        x, mult = ld / rd, 1.0
    count("ld_lt_rd" if ld < rd else "ld_gt_rd" if ld > rd else "ld_eq_rd")
    return (_fit(x, mode) - 0.5) * mult


# Matrix<float,6,9> m_fit_params of ParabolaFit2d (SGMAssist.h:86-94, :139): the double literals stored as float
PINV = np.array([[1 / 6, -1 / 3, 1 / 6, 1 / 6, -1 / 3, 1 / 6, 1 / 6, -1 / 3, 1 / 6],
                 [1 / 6, 1 / 6, 1 / 6, -1 / 3, -1 / 3, -1 / 3, 1 / 6, 1 / 6, 1 / 6],
                 [1 / 4, 0, -1 / 4, 0, 0, 0, -1 / 4, 0, 1 / 4],
                 [-1 / 6, 0, 1 / 6, -1 / 6, 0, 1 / 6, -1 / 6, 0, 1 / 6],
                 [-1 / 6, -1 / 6, -1 / 6, 0, 0, 0, 1 / 6, 1 / 6, 1 / 6],
                 [-1 / 9, 2 / 9, -1 / 9, 2 / 9, 5 / 9, 2 / 9, -1 / 9, 2 / 9, -1 / 9]], np.float64).astype(np.float32)


def find_peak(z, counts=None):
    """ParabolaFit2d::find_peak (SGMAssist.h:99-135) on the 9 accumulated costs around the winner, row-major.
    Matrix<float,6,9> * Vector<double,9> is a double product (ProductType<float, double>): every float entry times a double,
    summed from 0 in index order (dot_prod, Math/Vector.h:1719-1726).  Returns (dx, dy), or None when |4ab - c^2| < 0.01
    rejects the fit."""
    z = [float(v) for v in z]
    vals = []
    for i in range(6):
        s = 0.0
        for j in range(9):
            s += float(PINV[i, j]) * z[j]
        vals.append(s)
    denom = 4.0 * vals[0] * vals[1] - (vals[2] * vals[2])
    if abs(denom) < 0.01:
        if counts is not None:
            counts["fit_rejected"] += 1
        return None
    # Vector2f offset: the double quotients are stored as float, then read back into double
    dx = float(np.float32((vals[2] * vals[4] - 2.0 * vals[1] * vals[3]) / denom))
    dy = float(np.float32((vals[2] * vals[3] - 2.0 * vals[0] * vals[4]) / denom))
    sX, sY = 0.34574, 0.38944
    dx = math.erf(dx / (sX * math.sqrt(2.0))) / 2.0
    dy = math.erf(dy / (sY * math.sqrt(2.0))) / 2.0
    nrm = math.sqrt(dx * dx + dy * dy)        # norm_2 of a Vector2 (double): squares summed in double
    if nrm >= 0.5:
        scale = nrm / 0.5
        dx /= scale
        dy /= scale
        if counts is not None:
            counts["fit_rescaled"] += 1
    elif counts is not None:
        counts["fit_kept"] += 1
    return dx, dy


def subpixel_pixel(box, width, bounds, dx, dy, mode, counts=None):
    """one pixel of the loop of create_disparity_view_subpixel (:1517-1598): box = the pixel's accumulated costs as the
    integer stage left them (flat, row-major), bounds = {min_x, min_y, max_x, max_y}, (dx, dy) = its valid integer
    disparity.  Returns the float32 pair."""
    if mode == 0:
        return np.float32(dx), np.float32(dy)
    x0, y0, x1, y1 = bounds
    min_index = (dy - y0) * width + (dx - x0)
    x_left, x_right, y_up, y_down = -1, 1, -width, width
    lb = rb = tb = bb = False
    if dx == x0:
        x_left, lb = 0, True
    if dx == x1:
        x_right, rb = 0, True
    if dy == y0:
        y_up, tb = 0, True
    if dy == y1:
        y_down, bb = 0, True
    if mode == 1:
        m = min_index
        peak = find_peak([box[m + x_left + y_up], box[m + y_up], box[m + x_right + y_up],
                          box[m + x_left], box[m], box[m + x_right],
                          box[m + x_left + y_down], box[m + y_down], box[m + x_right + y_down]], counts)
        if peak is None:
            return np.float32(dx), np.float32(dy)
        delta_x, delta_y = peak
    else:
        delta_x = compute_subpixel_offset(box[min_index + x_left], box[min_index], box[min_index + x_right], lb, rb, mode, counts)
        delta_y = compute_subpixel_offset(box[min_index + y_up], box[min_index], box[min_index + y_down], tb, bb, mode, counts)
    return np.float32(dx + delta_x), np.float32(dy + delta_y)   # p_type(dx + delta_x, ...): a double sum stored as float


def new_counts():
    return dict.fromkeys(BRANCHES, 0)


def subpixel_stage(res, mode, counts=None):
    """create_disparity_view_subpixel (:1497-1614) on the boxes an sgm() call left: (oh, ow, 3) float32 {dx, dy, valid}.
    Invalid pixels are all zeros.  counts (a new_counts() dict, or None) receives the branches taken."""
    oh, ow = res.disparity.shape[:2]
    out = np.zeros((oh, ow, 3), np.float32)
    for r in range(oh):
        for c in range(ow):
            dx, dy, valid = (int(v) for v in res.disparity[r, c])
            if not valid:
                continue
            b = [int(v) for v in res.bounds[r, c]]
            if counts is not None and res.smoothed[r, c] and mode:
                counts["smoothed_winner"] += 1
            out[r, c, :2] = subpixel_pixel(res.boxes[r][c], b[2] - b[0] + 1, b, dx, dy, mode, counts)
            out[r, c, 2] = 1
    return out


class SgmResult(NamedTuple):
    disparity: np.ndarray   # (oh, ow, 3) int32 {dx, dy, valid} from the uint16 (wrapping) accumulation, as the reference
    unwrapped: np.ndarray   # the same from an int64 accumulation that never wraps
    smoothed: np.ndarray    # (oh, ow) bool: the wrapped winner went through the tie smoothing
    lowest: np.ndarray      # (oh, ow) int64: lowest wrapped accumulated cost of the box (-1 where the box is empty)
    max_sum: int            # largest unwrapped 8-path sum over every (pixel, disparity) inside a box
    bounds: np.ndarray      # (oh, ow, 4) int64 boxes {min_x, min_y, max_x, max_y}
    boxes: list             # [oh][ow] the wrapped box as select_best_disparity left it (flat list), None if empty
    subpixel: np.ndarray    # (oh, ow, 3) float32 of create_disparity_view_subpixel in the requested mode, or None
    counts: dict            # the sub-pixel branches that mode took (new_counts()), or None


def sgm(left, right, search, kernel, bounds=None, p1=0, p2=0, subpixel_mode=None):
    """calc_disparity_sgm (SGM.cc:167-230 -> semi_global_matching_func :2387-2448) with CENSUS_TRANSFORM and plain SGM.
    left / right: the left_region / right_region rasters; bounds: (oh, ow, 4) boxes, or None for the whole search box
    [0, search] at every pixel.  subpixel_mode (SgmSubpixelMode 0-5): also run create_disparity_view_subpixel on the
    wrapped boxes; subpixel_stage(result, mode) gives the other modes of the same accumulation."""
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
    boxes = [[None] * ow for _ in range(oh)]
    for r in range(oh):
        for c in range(ow):
            x0, y0, x1, y1 = (int(v) for v in bounds[r, c])
            if x1 < x0 or y1 < y0:           # no search area: invalid (create_disparity_view, :1317-1336)
                continue
            w = x1 - x0 + 1
            i, smoothed[r, c], lowest[r, c], boxes[r][c] = select_best_disparity(wrapped[r, c, y0:y1 + 1, x0:x1 + 1], return_box=True)
            disp[r, c] = (x0 + i % w, y0 + i // w, 1)
            i, _, _ = select_best_disparity(total[r, c, y0:y1 + 1, x0:x1 + 1], wrap=False)
            disp_u[r, c] = (x0 + i % w, y0 + i // w, 1)
    res = SgmResult(disp, disp_u, smoothed, lowest, int(np.where(inbox, total, 0).max()), bounds, boxes, None, None)
    if subpixel_mode is None:
        return res
    counts = new_counts()
    return res._replace(subpixel=subpixel_stage(res, subpixel_mode, counts), counts=counts)


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


# ---- the sub-pixel cases: search boxes that put the winner on every branch of create_disparity_view_subpixel ---------------
SUB_OH, SUB_OW = 40, 56
# name: (search, boxes, imagery, offset, where the device keeps the totals).  boxes: None = the constant box; (w, h) =
# moving boxes of 1..w x 1..h; "w1" / "h1" / "1x1" / "w2" / "h2" = moving boxes of exactly that width or height (the other
# side 1..6); (w, h, "full") = moving boxes plus full-search pixels.  imagery: "flat" = flat_pair's 4 grey levels, whose
# ties drive the smoothing; "textured" = 48 levels.  totals: "shared" = summed in sgm_wta_kernel's shared memory (every box
# <= 32 entries), "sum4" = by sgm_sum4_kernel in global memory, "serial" = one volume (VWB200_SGM_SERIAL), "mgm".
SUBPIXEL_CASES = {
    "const-flat": ((5, 3), None, "flat", (3, 2), "shared"),
    "const-textured": ((8, 5), None, "textured", (3, 2), "sum4"),
    "w1": ((15, 11), "w1", "textured", (3, 2), "shared"),
    "h1": ((15, 11), "h1", "flat", (3, 2), "shared"),
    "1x1": ((15, 11), "1x1", "textured", (3, 2), "shared"),
    "w2": ((15, 11), "w2", "textured", (3, 2), "shared"),
    "h2": ((15, 11), "h2", "flat", (3, 2), "shared"),
    "moving-32": ((15, 11), (6, 5), "flat", (3, 2), "shared"),
    "moving-48": ((15, 11), (6, 8), "textured", (3, 2), "sum4"),
    "full": ((15, 11), (6, 8, "full"), "flat", (3, 2), "sum4"),
    "serial": ((15, 11), (6, 8, "full"), "textured", (3, 2), "serial"),
    "wide-x": ((140, 1), None, "textured", (133, 1), "sum4"),
}


def subpixel_case(name):
    """(left, right, bounds (oh, ow, 4) int32, search) of a SUBPIXEL_CASES entry"""
    search, boxes, imagery, off, _ = SUBPIXEL_CASES[name]
    seed = 70 + sorted(SUBPIXEL_CASES).index(name)
    left, right = flat_pair(seed, SUB_OH, SUB_OW, search, 5, off=off, levels=4 if imagery == "flat" else 48)
    if boxes is None:
        return left, right, np.tile(np.array([0, 0, search[0], search[1]], np.int32), (SUB_OH, SUB_OW, 1)), search
    fixed = {"w1": (1, 0), "h1": (0, 1), "1x1": (1, 1), "w2": (2, 0), "h2": (0, 2)}
    if boxes in fixed:
        fw, fh = fixed[boxes]
        b = moving_boxes(seed + 1, SUB_OH, SUB_OW, search, 6, 6, empty=0.0)
        rng = np.random.default_rng(seed + 2)
        if fw:
            b[..., 0] = rng.integers(0, search[0] + 2 - fw, (SUB_OH, SUB_OW))
            b[..., 2] = b[..., 0] + fw - 1
        if fh:
            b[..., 1] = rng.integers(0, search[1] + 2 - fh, (SUB_OH, SUB_OW))
            b[..., 3] = b[..., 1] + fh - 1
        return left, right, b, search
    b = moving_boxes(seed + 1, SUB_OH, SUB_OW, search, boxes[0], boxes[1])
    if len(boxes) > 2:
        full = np.random.default_rng(seed + 2).random((SUB_OH, SUB_OW)) < 0.05
        full[10:16, 20:36] = True
        b[full] = (0, 0, search[0], search[1])
    return left, right, b, search
