"""CPU references for the block-matching kernels of calc_disparity.

brute_calc_disparity is the reference's best_of_search_convolution (Stereo/Correlation.cc:33-137) in numpy.  The rest of
the module restates, in Python, the dispatch and geometry predicates of the CUDA sources, each citing the lines it
restates: from them `expected_kernels` derives which hot kernel instantiation a calc_disparity call runs, and whether a
merge or a seeding pass follows.  CASES is the case matrix built on them: every block-matching instantiation the library
compiles and calc_disparity can reach, at the shapes and value ranges where each one is most likely to go wrong.
tests/test_gpu_kernel_matrix.py runs it on the device, tests/test_oracle_kernel_matrix.py through the oracle."""
import math
import os
import re
from dataclasses import dataclass, field

import numpy as np

ABS, SQ, NCC = 0, 1, 2
COST_NAMES = {ABS: "abs", SQ: "sq", NCC: "ncc"}
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "visionworkbench_b200", "csrc")


# ---- brute force ---------------------------------------------------------------------------------------------------------
def _box(a, kx, ky):
    """kx x ky window sums by a summed-area table: exact while every prefix sum is an exact double (integer imagery, or
    multiples of 2^-8 below 256)"""
    c = np.zeros((a.shape[0] + 1, a.shape[1] + 1))
    c[1:, 1:] = a.cumsum(0).cumsum(1)
    return c[ky:, kx:] - c[:-ky, kx:] - c[ky:, :-kx] + c[:-ky, :-kx]


def brute_calc_disparity(cost, left, right, search, kernel):
    """best_of_search_convolution (Stereo/Correlation.cc:33-137): float32 per-pixel cost, float64 box sums, NCC as
    S_lr * sqrt((1 / box(l^2)) * (1 / box(r^2))), strict '<' ('>' for NCC) over dy-major / dx-minor disparities,
    best == worst -> invalid.  A NaN cost (zero-energy NCC window) follows the same comparisons: it never becomes the best
    and always becomes the worst, and a NaN best at (0, 0) is never replaced."""
    l, r = np.asarray(left, np.float32), np.asarray(right, np.float32)
    (sx, sy), (kx, ky) = search, kernel
    H, W = l.shape[0] - ky + 1, l.shape[1] - kx + 1
    r = r[:l.shape[0] + sy - 1, :l.shape[1] + sx - 1]
    if cost == NCC:
        with np.errstate(divide="ignore"):
            lp = 1.0 / _box((l * l).astype(np.float64), kx, ky)
            rp = 1.0 / _box((r * r).astype(np.float64), kx, ky)
    out = np.zeros((H, W, 3), np.int32)
    out[..., 2] = 1
    better = np.greater if cost == NCC else np.less
    with np.errstate(invalid="ignore"):
        for dy in range(sy):
            for dx in range(sx):
                rs = r[dy:dy + l.shape[0], dx:dx + l.shape[1]]
                if cost == ABS:
                    c = np.abs(l - rs)
                elif cost == SQ:
                    d = l - rs
                    c = d * d
                else:
                    c = l * rs
                m = _box(c.astype(np.float64), kx, ky)
                if cost == NCC:
                    m = m * np.sqrt(lp * rp[dy:dy + H, dx:dx + W])
                if dx == 0 and dy == 0:
                    best, worst = m.copy(), m.copy()
                    continue
                up = better(m, best)
                best[up] = m[up]
                out[up, 0], out[up, 1] = dx, dy
                down = ~up & ~better(m, worst)
                worst[down] = m[down]
        out[best == worst, 2] = 0
    return out


# ---- dispatch and geometry, restated ----------------------------------------------------------------------------------------
NUM_SMS = 132                     # kNumSMs, common.cuh:15
F_TH, F_COLS, F_B = 32, 256, 8    # k1_fast_common.cuh:8-12
FK_TH_MAX, FK_SMEM = 96, 227 * 1024   # k1_fast.cu:82-83
SMEM_MAX = 227 * 1024
K1G_DCHUNK = 256                  # common.cuh:96
ZR_MAX = 12288                    # k1_generic.cu:69
ZI_TH, ZI_MAX_U16 = 16, 28672     # k1_zone_int.cu:25-27
ZI_CLS = (3072, 12288)            # engine.cu:128
SD_MAX = 3                        # k1_screen.cu:39


@dataclass
class Geom:
    th: int
    NS: int
    NB: int
    J: int
    dy_per: int
    rw: int
    ltile_rows: int
    ring_slots: int
    sd: int = 1


def make_geom(W, H, sx, sy, kx, ky, th=F_TH):
    """make_geom, k1_fast_common.cuh:30-63"""
    out_cols = F_COLS - (kx - 1)
    NS = (W + out_cols - 1) // out_cols
    NB = (H + th - 1) // th
    rw = ((F_COLS + sx + 7) // 8) * 8 + 8
    J = 1
    items = NS * NB
    jmax = 1 if sy // 8 < 1 else min(sy // 8, 8)
    if items < 64 * NUM_SMS:
        best = -1.0
        for j in range(1, jmax + 1):
            w = items * j / NUM_SMS
            full = (items * j + NUM_SMS - 1) // NUM_SMS
            eff = w / full * (1.0 - 0.004 * (j - 1))
            if w < 6.0:
                eff *= 0.5 + w / 12.0
            if eff > best + 1e-9:
                best, J = eff, j
    dy_per = (sy + J - 1) // J
    J = (sy + dy_per - 1) // dy_per
    return Geom(th, NS, NB, J, dy_per, rw, th + ky - 1, th + ky)


def fast_smem_bytes(g):
    """k1_fast.cu:87-89"""
    return g.th * F_COLS * 4 + g.ltile_rows * F_COLS * 2 + g.ring_slots * g.rw * 2 + 64


def fast_geom(W, H, sx, sy, kx, ky):
    """fast_geom, k1_fast.cu:95-106: the band height with the least estimated time"""
    best, tbest = make_geom(W, H, sx, sy, kx, ky, F_TH), -1.0
    for th in range(F_TH, FK_TH_MAX + 1):
        g = make_geom(W, H, sx, sy, kx, ky, th)
        if fast_smem_bytes(g) > FK_SMEM:
            break
        waves = (g.NS * g.NB * g.J + NUM_SMS - 1) // NUM_SMS
        t = waves * g.dy_per * (min(th, H) + 0.15 * ky) * (1.0 + 0.004 * (g.J - 1))
        if tbest < 0.0 or t < tbest:
            tbest, best = t, g
    return best


def _f32(v):
    return float(np.float32(v))


def k1_fast_supported(cost, kx, ky, sx, sy, vmin, vmax, integer):
    """k1_fast.cu:108-124"""
    if cost not in (ABS, SQ) or not integer:
        return False
    vmin, vmax = _f32(vmin), _f32(vmax)
    if cost == SQ:
        r = vmax - vmin
        if not (r <= 4095.0) or not (r * r * kx * ky < 4294967295.0):
            return False
    elif not (_f32(vmax - vmin) <= 8191.0):
        return False
    if not (abs(vmin) < 1.0e6) or not (abs(vmax) < 1.0e6):
        return False
    if kx < 3 or kx > 31 or ky < 1 or ky > 41:
        return False
    if sx < F_B or sx > 512 or sy < 1 or sx * sy > 65536 or sx * sy < 64:
        return False
    return fast_smem_bytes(make_geom(256, F_TH, sx, sy, kx, ky, F_TH)) <= FK_SMEM


def screen_params(mode, kx, ky, vmin, vmax):
    """screen_params, k1_screen.cu:62-71: (c, maxc), or None outside the supported range"""
    vmin, vmax = _f32(vmin), _f32(vmax)
    if mode == NCC and (not (vmin >= 0.0) or not (vmax <= 4095.0)):
        return None
    if mode == SQ and not (vmax - vmin <= 4095.0):
        return None
    if not (abs(vmin) < 1.0e6) or not (abs(vmax) < 1.0e6):
        return None
    c = math.floor((vmin + vmax) * 0.5 + 0.5)
    maxc = max(vmax - c, c - vmin)
    if maxc > 32767.0 or maxc * maxc * kx * ky >= 2147483647.0:
        return None
    return c, maxc


def screen_smem_bytes(g, mode):
    """k1_screen.cu:40-50"""
    nq = F_TH + 2 * g.sd - 1
    return F_TH * F_COLS * 4 + g.ltile_rows * F_COLS * 2 + g.ring_slots * g.rw * 2 + (2 if mode == NCC else 1) * nq * g.rw * 4 + 128


def screen_geom(W, H, sx, sy, kx, ky, mode):
    """make_geom + screen_geom, k1_screen.cu:53-60: the deepest ring (sd dy rows per period) that fits; None if none does"""
    g = make_geom(W, H, sx, sy, kx, ky)
    for sd in range(SD_MAX, 0, -1):
        g.sd, g.ring_slots = sd, g.ltile_rows + 2 * sd - 1
        if screen_smem_bytes(g, mode) <= SMEM_MAX:
            return g
    return None


def k1_screen_supported(cost, kx, ky, sx, sy, vmin, vmax, integer):
    """k1_screen.cu:73-84"""
    if cost not in (NCC, SQ) or not integer:
        return False
    if screen_params(cost, kx, ky, vmin, vmax) is None:
        return False
    if kx < 3 or kx > 31 or ky < 1 or ky > 41:
        return False
    if sx < F_B or sx > 512 or sy < 1 or sx * sy < 64 or sx * sy > 65536:
        return False
    return screen_geom(256, 32, sx, sy, kx, ky, cost) is not None


def screen_seed(W, H, sx, sy, kx, ky, vmin, vmax):
    """the seeding stage's half-resolution k1_fast problem (k1_screen.cu:128-130) and whether it runs (:742-743):
    (kx2, ky2, sx2, sy2, W2, H2) or None"""
    W2, H2 = (W + 1) // 2, (H + 1) // 2
    kx2, ky2 = max(3, (kx // 2) | 1), max(1, (ky // 2) | 1)
    sx2, sy2 = (((sx + 1) // 2 + 7) // 8) * 8, (sy + 1) // 2
    if W >= 64 and H >= 64 and k1_fast_supported(ABS, kx2, ky2, sx2, sy2, vmin, vmax, True):
        return kx2, ky2, sx2, sy2, W2, H2
    return None


def k1_zone_int_mode(cost, kx, ky, rng):
    """k1_zone_int.cu:230-241: 0 unsupported, 1 narrow, 2 wide (the disparity chunk is always 2^8)"""
    if cost not in (ABS, SQ):
        return 0
    if kx != ky or kx < 3 or kx > 25 or not (kx & 1) or rng < 0 or rng > 65535:
        return 0
    if cost == SQ and rng > 4095:
        return 0
    per_pixel = rng * rng if cost == SQ else rng
    maxh = per_pixel * kx * ky
    if per_pixel <= 65535 and maxh < (1 << 24):
        return 1
    if cost == SQ and maxh < 0xffffffff:
        return 2
    return 0


def zone_int_stage_u16(k, sx, sy, nchunks, ib=8):
    """k1_zone_int_stage_u16, k1_zone_int.cu:247-250"""
    span = min(sy, ((1 << ib) + sx - 1) // sx + 1) if nchunks > 1 else sy
    return (ZI_TH + k - 1 + span - 1) * (32 + sx) + (ZI_TH + k - 1) * 32


def zone_int_class(need):
    """staging class of a zone-int tile, engine.cu:142"""
    return 0 if need <= ZI_CLS[0] else (1 if need <= ZI_CLS[1] else 2)


def generic_stage_floats(kx, ky, sx, sy, nchunks):
    """k1_generic_stage_floats, k1_generic.cu:259-262"""
    span = min(sy, (K1G_DCHUNK + sx - 1) // sx + 1) if nchunks > 1 else sy
    return (32 + kx - 1 + sx - 1) * (16 + ky - 1 + span - 1)


def zone_plan(cost, W, H, sx, sy, kx, ky, zone_int, vmin=0.0, vmax=0.0):
    """run_k1_zones (engine.cu:106-122) for the single zone of calc_disparity's general path: (kernel, nchunks), kernel
    "zone-int" or "generic"; nchunks > 1 means split over disparity chunks and finished by k1_generic_merge_kernel"""
    nd = sx * sy
    nchunks = (nd + K1G_DCHUNK - 1) // K1G_DCHUNK
    kind = "generic"
    if zone_int and k1_zone_int_mode(cost, kx, ky, int(vmax) - int(vmin)):
        nci = (nd + 255) >> 8
        if zone_int_stage_u16(kx, sx, sy, nci) <= ZI_MAX_U16 and (nci == 1 or W * H * nci < (1 << 29)):
            kind, nchunks = "zone-int", nci
    if not (nchunks > 1 and W * H * nchunks < (1 << 29)):
        nchunks = 1
    return kind, nchunks


@dataclass
class Expect:
    """what a calc_disparity call runs: the hot kernel family and its template arguments, and the passes after it"""
    family: str
    args: tuple
    merge: tuple = None          # the merge kernel (name, template arguments), or None when no merge runs
    seed: tuple = None           # screen: the template arguments of the seeding k1_fast_abs_kernel, or None
    seed_merge: bool = False     # screen: the seeding k1_fast problem runs with J > 1
    geom: dict = field(default_factory=dict)


def expected_kernels(cost, W, H, sx, sy, kx, ky, vmin, vmax, integer, zone_int=False):
    """calc_disparity_device, engine.cu:905-940: which kernel a raster takes, from its statistics"""
    if not (zone_int and integer):
        if k1_fast_supported(cost, kx, ky, sx, sy, vmin, vmax, integer):
            g = fast_geom(W, H, sx, sy, kx, ky)
            return Expect("k1_fast_abs_kernel", (kx, cost == SQ), ("k1_fast_merge_kernel", ()) if g.J > 1 else None,
                          geom=dict(J=g.J, th=g.th, NS=g.NS, NB=g.NB))
        if k1_screen_supported(cost, kx, ky, sx, sy, vmin, vmax, integer):
            g = screen_geom(W, H, sx, sy, kx, ky, cost)
            s = screen_seed(W, H, sx, sy, kx, ky, vmin, vmax)
            seed_merge = s is not None and fast_geom(s[4], s[5], s[2], s[3], s[0], s[1]).J > 1
            return Expect("k1_screen_kernel", (kx, 0 if cost == NCC else 1), ("k1_screen_merge_kernel", ()) if g.J > 1 else None,
                          (s[0], False) if s else None, seed_merge, dict(J=g.J, sd=g.sd, NS=g.NS, NB=g.NB))
    kind, nchunks = zone_plan(cost, W, H, sx, sy, kx, ky, zone_int and integer, vmin, vmax)
    merge = ("k1_generic_merge_kernel", (NCC if cost == NCC else ABS,)) if nchunks > 1 else None
    if kind == "zone-int":
        mode = k1_zone_int_mode(cost, kx, ky, int(vmax) - int(vmin))
        return Expect("k1_zone_int_kernel", (SQ if mode == 2 else cost, kx, mode == 2), merge,
                      geom=dict(nchunks=nchunks, cls=zone_int_class(zone_int_stage_u16(kx, sx, sy, nchunks))))
    stage = generic_stage_floats(kx, ky, sx, sy, nchunks) <= ZR_MAX
    # calc_disparity's zone reads stay inside the rasters: clamp_reads is false (engine.cu:120-121)
    return Expect("k1_generic_kernel", (cost, stage, stage), merge, geom=dict(nchunks=nchunks, stage=stage))


# ---- the instantiations the sources compile ------------------------------------------------------------------------------
def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _switch_widths(src, macro):
    """the widths of the `switch` that expands `macro`: its calls between the macro's #define and its #undef"""
    begin = src.index(f"#define {macro}(")
    end = src.index(f"#undef {macro}", begin)
    return sorted({int(k) for k in re.findall(rf"\b{macro}\((\d+)\)", src[begin:end])})


def compiled_instantiations():
    """every hot-kernel instantiation a dispatch switch can select, parsed from the sources"""
    inst = set()
    for k in _switch_widths(_read("k1_fast.cu"), "KCASE"):            # k1_fast.cu:480-486
        inst |= {("k1_fast_abs_kernel", (k, False)), ("k1_fast_abs_kernel", (k, True))}
    for k in _switch_widths(_read("k1_screen.cu"), "KCASE"):          # k1_screen.cu:766-772
        inst |= {("k1_screen_kernel", (k, 0)), ("k1_screen_kernel", (k, 1))}
    for k in _switch_widths(_read("k1_zone_int.cu"), "ZI_CASE"):      # k1_zone_int.cu:261-270
        inst |= {("k1_zone_int_kernel", (ABS, k, False)), ("k1_zone_int_kernel", (SQ, k, False)), ("k1_zone_int_kernel", (SQ, k, True))}
    gen = _read("k1_generic.cu")
    m = re.search(r"#define KSEL\(C\) (.*)", gen)                     # k1_generic.cu:273-278
    combos = [(a == "true", b == "true") for a, b in re.findall(r"k1_generic_kernel<C, (\w+), (\w+)>", m.group(1))]
    costs = {"VWB200_ABSOLUTE_DIFFERENCE": ABS, "VWB200_SQUARED_DIFFERENCE": SQ, "VWB200_CROSS_CORRELATION": NCC}
    for c in {costs[c] for c in re.findall(r"KSEL\((VWB200_\w+)\)", gen)}:
        inst |= {("k1_generic_kernel", (c, clamp, stage)) for clamp, stage in combos}
    for c in re.findall(r"k1_generic_merge_kernel<(\w+)><<<", gen):   # k1_generic.cu:244-245
        inst.add(("k1_generic_merge_kernel", (costs[c],)))
    return inst


# instantiations no calc_disparity or view call can select, and why
UNREACHABLE = {
    ("k1_screen_kernel", (3, 1)): "Sq on K1 screen needs r^2 * kx * ky >= 2^32 - 1 with r <= 4095, so kx * ky >= 257; "
                                  "at kx = 3 that is ky >= 86, past the ky <= 41 limit",
    ("k1_screen_kernel", (5, 1)): "as <3, 1>: at kx = 5, Sq on K1 screen needs ky >= 52 > 41",
}


# ---- imagery -----------------------------------------------------------------------------------------------------------------
def binary_raster(h, w, lo, hi, seed):
    """only lo and hi: random, with a checkerboard in the top-left quarter (windows that differ in every pixel from a
    one-pixel shift, the largest window sums)"""
    rng = np.random.default_rng(seed)
    v = np.where(rng.random((h, w)) < 0.5, lo, hi).astype(np.float64)
    yy, xx = np.mgrid[0:h // 2, 0:w // 2]
    v[:h // 2, :w // 2] = np.where((yy + xx) % 2 == 0, lo, hi)
    return v


def levels_raster(h, w, levels, step, seed, flat=None, zero=None):
    """values (0 .. levels-1) * step, so that many disparities tie; `flat` (y0, y1, x0, x1) is set to the top value, `zero`
    to 0"""
    rng = np.random.default_rng(seed)
    v = rng.integers(0, levels, size=(h, w)).astype(np.float64) * step
    if flat:
        v[flat[0]:flat[1], flat[2]:flat[3]] = (levels - 1) * step
    if zero:
        v[zero[0]:zero[1], zero[2]:zero[3]] = 0.0
    return v


def sparse_raster(h, w, density, seed):
    """1 with probability `density`, else 0: NCC window sums of a few units, so that a small error in box(l * r) reorders
    candidates whose right energies differ"""
    return (np.random.default_rng(seed).random((h, w)) < density).astype(np.float64)


def float_raster(h, w, seed):
    """multiples of 2^-8 in [0, 256): every box sum is an exact double"""
    rng = np.random.default_rng(seed)
    return np.floor(rng.random((h, w)) * 256 * 256) / 256


@dataclass
class Case:
    id: str
    cost: int
    W: int
    H: int
    search: tuple
    kernel: tuple
    image: dict                  # make_inputs() recipe
    zone_int: bool = False       # run with the integer zone kernel forced (VWB200_K1_ZONE_INT)

    def inputs(self):
        return make_inputs(self)

    def expect(self):
        left, right = self.inputs()
        vmin, vmax = float(min(left.min(), right.min())), float(max(left.max(), right.max()))
        integer = bool(np.all(left == np.rint(left)) and np.all(right == np.rint(right)))
        (sx, sy), (kx, ky) = self.search, self.kernel
        return expected_kernels(self.cost, self.W, self.H, sx, sy, kx, ky, vmin, vmax, integer, self.zone_int)


def make_inputs(case):
    """left, right (float32) for a case: `right` from the recipe, `left` its crop at the disparity `shift` (+ noise)"""
    (sx, sy), (kx, ky) = case.search, case.kernel
    rh, rw = case.H + ky - 1 + sy - 1, case.W + kx - 1 + sx - 1
    im = case.image
    seed = im.get("seed", 0)
    kind = im["kind"]
    if kind == "binary":
        right = binary_raster(rh, rw, im["lo"], im["hi"], seed)
    elif kind == "sparse":
        right = sparse_raster(rh, rw, im["density"], seed)
    elif kind == "levels":
        right = levels_raster(rh, rw, im["levels"], im.get("step", 1), seed, im.get("flat"), im.get("zero"))
    else:
        right = float_raster(rh, rw, seed)
        if im.get("zero"):
            z = im["zero"]
            right[z[0]:z[1], z[2]:z[3]] = 0.0
    dx, dy = im.get("shift", (sx // 2, sy // 2))
    left = right[dy:dy + case.H + ky - 1, dx:dx + case.W + kx - 1].copy()
    if im.get("independent"):                 # a left raster unrelated to the right: the best match is a near tie
        left = sparse_raster(left.shape[0], left.shape[1], im["density"], seed + 7)
    if im.get("noise"):
        n = np.random.default_rng(seed + 1).integers(-im["noise"], im["noise"], size=left.shape, endpoint=True)
        left = np.clip(left + n * im.get("step", 1), right.min(), right.max())
    if im.get("lzero"):
        z = im["lzero"]
        left[z[0]:z[1], z[2]:z[3]] = 0.0
    return np.ascontiguousarray(left, np.float32), np.ascontiguousarray(right, np.float32)


# ---- the case matrix ---------------------------------------------------------------------------------------------------------
WIDTHS = list(range(3, 32, 2))                # K1 fast / K1 screen: kx 3 .. 31
ZI_WIDTHS = list(range(3, 26, 2))             # zone-int: K 3 .. 25
KY_ROT = (1, 3, None, 41)                     # ky across the widths; None: ky = kx


def _sq_limit(n):
    """the largest r <= 4095 with r^2 * n < 2^32 - 1"""
    r = min(4095, math.isqrt(4294967294 // n))
    while r * r * n >= 4294967295:
        r -= 1
    return r


def _fast_cases():
    out = []
    for i, kx in enumerate(WIDTHS):
        ky = KY_ROT[i % 4] or kx
        W = (257 - kx) + 19 + i                # two strips, the second one partial
        sx, sy = 13 if i % 2 else 11, 6 + (i % 3) * 4      # sx % 8 != 0, sy <= 15: J = 1
        for cost in (ABS, SQ):
            hi = 8191 if cost == ABS else _sq_limit(kx * ky)
            out.append(Case(f"fast-{COST_NAMES[cost]}-k{kx}x{ky}-limit", cost, W, 24 + i, (sx, sy), (kx, ky),
                            dict(kind="binary", lo=0, hi=hi, seed=100 + kx, shift=(sx - 2, sy - 1))))
        # J > 1: 2-bit imagery with a flat block (ties across warps and dy chunks, all-equal pixels)
        kyb = max(1, min(41, (kx // 2) | 1))
        for cost in (ABS, SQ):
            out.append(Case(f"fast-{COST_NAMES[cost]}-k{kx}x{kyb}-ties", cost, 70, 30, (12, 24), (kx, kyb),
                            dict(kind="levels", levels=4, seed=200 + kx, flat=(8, 30, 10, 60), shift=(3, 17))))
    return out


def _screen_ncc_ky(kx, vmax=4095):
    """the tallest odd ky <= 41 that keeps maxc^2 * kx * ky < 2^31 at [0, vmax]"""
    maxc = max(vmax - math.floor(vmax * 0.5 + 0.5), math.floor(vmax * 0.5 + 0.5))
    ky = min(41, (2147483646 // (maxc * maxc * kx)))
    return ky if ky % 2 else ky - 1


def _screen_sq_ky(kx):
    """odd ky <= 41 with 4095^2 * kx * ky >= 2^32 - 1 (not K1 fast) and 2048^2 * kx * ky < 2^31 (K1 screen); None if none"""
    for ky in range(41, 0, -2):
        n = kx * ky
        if 16769025 * n >= 4294967295 and 4194304 * n < 2147483647:
            return ky
    return None


def _screen_cases():
    out = []
    for i, kx in enumerate(WIDTHS):
        for cost in (NCC, SQ):
            ky = _screen_ncc_ky(kx) if cost == NCC else _screen_sq_ky(kx)
            if ky is None:
                continue
            W = (257 - kx) + 11 + i
            sx = 13 if i % 2 else 15
            # (a) seeding (>= 64 x 64), two strips, partial octet, range at the limit
            out.append(Case(f"screen-{COST_NAMES[cost]}-k{kx}x{ky}-seeded", cost, W, 64, (sx, 15), (kx, ky),
                            dict(kind="binary", lo=0, hi=4095, seed=300 + kx, shift=(sx - 3, 9))))
            # (b) under 64 rows (no seeding), J > 1; NCC: zero-energy blocks; every third width: a flat region
            flat = (4, 40, 20, 90) if i % 3 == 0 else None
            if cost == NCC:
                im = dict(kind="levels", levels=4, step=1365, seed=400 + kx, flat=flat, zero=(30, 60, 100, 150),
                          lzero=(2, 20, 5, 40), shift=(5, 11))
            else:
                im = dict(kind="binary", lo=0, hi=4095, seed=400 + kx, shift=(5, 11))
                if flat:
                    im = dict(kind="levels", levels=2, step=4095, seed=400 + kx, flat=flat, shift=(5, 11))
            out.append(Case(f"screen-{COST_NAMES[cost]}-k{kx}x{ky}-J" + ("-flat" if flat else ""), cost, 120, 40, (12, 24),
                            (kx, ky), im))
        # NCC on unrelated sparse binary rasters: low-energy windows and near ties between disparities whose right energies
        # differ, so that an error of a few units in box(l * r) changes the winner
        ky = _screen_ncc_ky(kx)
        out.append(Case(f"screen-ncc-k{kx}x{ky}-sparse", NCC, 100, 40, (13, 9), (kx, ky),
                        dict(kind="sparse", density=0.08, seed=450 + kx, independent=True)))
    # ring depths 2 and 1: wide searches
    for cost, kx, ky in ((NCC, 9, 41), (SQ, 15, 19)):
        for sx in (_sx_for_sd(cost, kx, ky, 2), _sx_for_sd(cost, kx, ky, 1)):
            sd = screen_geom(256, 32, sx, 1, kx, ky, cost).sd
            out.append(Case(f"screen-{COST_NAMES[cost]}-k{kx}x{ky}-sd{sd}", cost, 70, 40, (sx, 2), (kx, ky),
                            dict(kind="binary", lo=0, hi=4095, seed=500 + sx, shift=(sx - 7, 1))))
    return out


def _sx_for_sd(cost, kx, ky, sd):
    """the smallest search width (not a multiple of 8) whose ring depth is sd"""
    for sx in range(8, 513):
        g = screen_geom(256, 32, sx, 2, kx, ky, cost)
        if g is not None and g.sd == sd and sx % 8:
            return sx
    raise AssertionError(f"no search width gives ring depth {sd}")


def _zone_int_limit(cost, wide, k):
    n = k * k
    if cost == ABS:
        return min(65535, ((1 << 24) - 1) // n)
    if not wide:
        r = min(255, math.isqrt(((1 << 24) - 1) // n))
        while r * r * n >= (1 << 24):
            r -= 1
        return r
    r = min(4095, math.isqrt(0xfffffffe // n))
    while r * r * n >= 0xffffffff:
        r -= 1
    return r


def _zone_int_cases():
    out = []
    for i, k in enumerate(ZI_WIDTHS):
        tw = 33 - k
        W = 2 * tw + 5 if (2 * tw + 5) % tw else 2 * tw + 6        # not a multiple of the tile width
        for cost, wide in ((ABS, False), (SQ, False), (SQ, True)):
            name = "wide" if wide else "narrow"
            hi = _zone_int_limit(cost, wide, k)
            # (a) just below the variant's limit, one zone of < 256 disparities
            out.append(Case(f"zint-{COST_NAMES[cost]}-{name}-k{k}-limit", cost, W, 37, (11, 9), (k, k),
                            dict(kind="binary", lo=0, hi=hi, seed=600 + k, shift=(7, 5)), zone_int=True))
            # (b) more than 256 disparities (two chunks), an odd count in the last one; a mid-range value set so that
            #     costs tie across the chunk boundary
            sx, sy = (11, 27) if i % 2 else (13, 21)              # 297 = 256 + 41, 273 = 256 + 17
            out.append(Case(f"zint-{COST_NAMES[cost]}-{name}-k{k}-split", cost, W, 21, (sx, sy), (k, k),
                            dict(kind="levels", levels=3, step=hi // 2, seed=700 + k, shift=(sx - 4, sy - 3), noise=1),
                            zone_int=True))
    # staging class 2 (> 12288 u16 of right patch per tile): a wide search split over chunks
    out.append(Case("zint-abs-narrow-k25-class2", ABS, 30, 20, (400, 3), (25, 25),
                    dict(kind="levels", levels=5, step=1, seed=800, shift=(333, 2)), zone_int=True))
    return out


def _generic_cases():
    out = []
    for cost in (ABS, SQ, NCC):
        c = COST_NAMES[cost]
        # staged, one chunk
        out.append(Case(f"generic-{c}-staged", cost, 70, 37, (13, 9), (7, 5), dict(kind="float", seed=900 + cost, shift=(9, 6))))
        # unstaged (right patch over ZR_MAX floats), one chunk
        out.append(Case(f"generic-{c}-unstaged", cost, 45, 21, (200, 1), (31, 41), dict(kind="float", seed=910 + cost, shift=(171, 0))))
        # split, staged: the true match lies in the last chunk
        out.append(Case(f"generic-{c}-split-staged", cost, 50, 33, (20, 20), (5, 5), dict(kind="float", seed=920 + cost, shift=(17, 18))))
        # split, unstaged
        out.append(Case(f"generic-{c}-split-unstaged", cost, 40, 18, (300, 2), (9, 41), dict(kind="float", seed=930 + cost, shift=(280, 1))))
    # NCC split with zero-energy right windows that only the last chunk's disparities reach: the NaN flag crosses chunks
    out.append(Case("generic-ncc-split-nan", NCC, 50, 33, (20, 20), (5, 5),
                    dict(kind="float", seed=940, shift=(3, 2), zero=(40, 58, 10, 40))))
    return out


CASES = _fast_cases() + _screen_cases() + _zone_int_cases() + _generic_cases()

# the clamped, unstaged generic variant <C, true, false> is selected by the view only (tests/test_gpu_kernel_matrix.py): a
# single-level pyramid_correlate on float imagery with the consistency check on.  The right-to-left zone starts at
# q.rx = z.lx - dsx < 0 (engine.cu:646), which sets clamp_reads (engine.cu:120-121), and its 201 x 5 search is split over
# chunks whose right patch does not fit ZR_MAX.  id, cost, (W, H), search BBox2i, kernel
VIEW_CASES = [(f"view-generic-{COST_NAMES[c]}-clamped", c, (150, 80), (-100, -2, 100, 2), (9, 41)) for c in (ABS, SQ, NCC)]


def view_expect(cost):
    """the instantiation a VIEW_CASES view runs for its right-to-left zone"""
    return Expect("k1_generic_kernel", (cost, True, False))
