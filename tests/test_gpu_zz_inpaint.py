"""fill_holes_grass on the device (k9_inpaint.cu) against the oracle (oracle/vw_inpaint_oracle.c), bit for bit: both pixel
types, 0-100 % invalid pixels, 1 x 1 to 50 x 147 images, len 0..64, whole-image, interior, edge and 1-pixel windows, the
warp, CTA and global-scratch workers, a 4096^2 field with thousands of holes, host and device rasters with padded pitches on
NULL and side streams, a view's float output as input, the rejected arguments, and which K9 kernels ran."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import inpaint as oi
from test_oracle_inpaint import field, same

pytestmark = pytest.mark.gpu
EARG = -1
I32, F32 = 0, 1


@pytest.fixture(scope="module")
def vwb():
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "GPU tests need a CUDA device: the engine has no CPU path"
    return v


def holes_field(w, h, dtype, seed, length, n, sprinkle=0.0):
    """a valid field with n round holes of diameter 1..len, plus a fraction `sprinkle` of single invalid pixels"""
    d = field(w, h, sprinkle, dtype, seed)
    rng = np.random.default_rng(seed + 1)
    yy, xx = np.mgrid[:h, :w]
    for _ in range(n):
        r = rng.uniform(0.0, max(length, 1) / 2.0)
        cx, cy = rng.uniform(0, w), rng.uniform(0, h)
        d[(xx - cx) ** 2 + (yy - cy) ** 2 <= r * r, 2] = 0
    return d


def engine(vwb, d, length, window, dev):
    import torch
    x0, y0, ow, oh = window if window is not None else (0, 0, d.shape[1], d.shape[0])
    x = torch.from_numpy(d).cuda() if dev else d
    got = vwb.fill_holes_grass(x, length, (x0, y0, x0 + ow, y0 + oh))
    return got.cpu().numpy() if dev else got


def check(vwb, d, length, window=None, devs=(False, True), label=""):
    want = oi.fill_holes_grass(d, length, window)
    for dev in devs:
        got = engine(vwb, d, length, window, dev)
        assert same(got, want), (label, length, window, dev, np.argwhere(np.any(got != want, axis=2))[:5])
    return want


def windows(w, h):
    out = [None, (w - 1, h - 1, 1, 1), (0, 0, 1, 1)]
    if w > 6 and h > 6:
        out += [(2, 3, w - 5, h - 6), (0, h // 2, w, h - h // 2), (w // 3, 0, w - w // 3, 3), (w // 2, h // 2, 1, 1)]
    return out


SIZES = [(1, 1), (1, 9), (9, 1), (23, 17), (50, 147)]


@pytest.mark.parametrize("dtype", [np.int32, np.float32], ids=["i32", "f32"])
@pytest.mark.parametrize("w,h", SIZES, ids=lambda s: str(s))
def test_density_matrix(vwb, w, h, dtype):
    for k, dens in enumerate([0.0, 0.02, 0.1, 0.3, 0.6, 0.9, 1.0]):
        d = field(w, h, dens, dtype, 10 * k + w)
        for length in (0, 1, 2, 3, 7, 64):
            for win in windows(w, h):
                check(vwb, d, length, win, devs=(True,) if win else (False, True), label=dens)


@pytest.mark.parametrize("dtype", [np.int32, np.float32], ids=["i32", "f32"])
@pytest.mark.parametrize("length", [1, 2, 3, 4, 5, 8, 13, 21, 34, 50, 64])
def test_round_holes_len(vwb, length, dtype):
    """holes of diameter 1..len (several distance levels, the warp and the shared-memory CTA workers)"""
    w, h = (50, 147) if length <= 21 else (150, 160)
    d = holes_field(w, h, dtype, 200 + length, length, 12 if length <= 21 else 5, sprinkle=0.01)
    for win in (None, (3, 5, w - 9, h - 20), (w // 2, h // 2, 1, 1), (0, 0, w // 2, h)):
        check(vwb, d, length, win, devs=(False, True) if win is None else (True,))


@pytest.mark.parametrize("dtype", [np.int32, np.float32], ids=["i32", "f32"])
def test_global_scratch_ring(vwb, dtype):
    """a one-pixel-wide square ring of a hole around a valid island: a 170 x 170 bbox whose bbox.expand(1) state (16 bytes a
    pixel) is beyond shared memory, while max_distance = 1 keeps it to 10 sweeps"""
    n = 170
    d = field(n + 20, n + 16, 0.0, dtype, 300)
    d[8, 10:10 + n, 2] = d[8 + n - 1, 10:10 + n, 2] = 0
    d[8:8 + n, 10, 2] = d[8:8 + n, 10 + n - 1, 2] = 0
    want = check(vwb, d, n)
    assert (want[..., 2] != 0).all()
    check(vwb, d, n + 7, (40, 40, 30, 30))
    want = check(vwb, d, n - 1)                       # one short: the ring is not filled
    assert (want[8, 10:10 + n, 2] == 0).all()


def test_special_values(vwb):
    d = holes_field(60, 50, np.float32, 400, 6, 15, sprinkle=0.05)
    rng = np.random.default_rng(401)
    bad = d[..., 2] == 0
    d[..., :2][bad] = rng.choice(np.array([np.nan, np.inf, -np.inf, -0.0, 1e30, 3.0], np.float32), (bad.sum(), 2))
    d[3, 4, :2] = (np.inf, -np.inf)                                  # valid infinities next to holes
    d[20, 20, 2] = np.nan                                            # a NaN valid word counts as valid
    d[21, 20, 2] = -0.0                                              # and -0.0 as invalid
    check(vwb, d, 6)
    di = holes_field(60, 50, np.int32, 402, 6, 15, sprinkle=0.05)
    di[..., :2] = np.random.default_rng(403).integers(-(1 << 30) + 1, 1 << 30, (50, 60, 2))
    check(vwb, di, 6)


def test_4096_field(vwb):
    import torch
    n = 4096
    d = holes_field(n, n, np.float32, 500, 12, 0, sprinkle=0.002)
    rng = np.random.default_rng(501)
    yy, xx = np.mgrid[:24, :24]
    for cx, cy, r in zip(rng.integers(20, n - 20, 3000), rng.integers(20, n - 20, 3000), rng.uniform(0.5, 6.0, 3000)):
        d[cy - 12:cy + 12, cx - 12:cx + 12, 2][(xx - 12) ** 2 + (yy - 12) ** 2 <= r * r] = 0
    want, st = oi.fill_holes_grass(d, 12, None, stats=True)
    got = vwb.fill_holes_grass(torch.from_numpy(d).cuda(), 12).cpu().numpy()
    assert same(got, want)
    s = vwb.last_fill_stats()
    assert s["holes"] == st[0] and s["filled"] == st[1] and s["max_sweeps"] == st[2] and st[1] > 3000, (s, st)
    win = (1000, 1500, 1024, 1024)
    got = vwb.fill_holes_grass(torch.from_numpy(d).cuda(), 12, (1000, 1500, 2024, 2524)).cpu().numpy()
    assert same(got, oi.fill_holes_grass(d, 12, win))


def test_view_output_as_input(vwb):
    """the float disparity the correlation view rasterises, holes and all, as fill_holes_grass's input"""
    import torch
    from visionworkbench_b200.synth import make_pair
    search, kernel = (-12, -8, 12, 8), (7, 7)
    left, right, lm, rm, _ = make_pair(256, 224, search, seed=5)
    view = vwb.pyramid_correlate(left, right, lm, rm, vwb.PREFILTER_NONE, 0.0, search, kernel, vwb.ABSOLUTE_DIFFERENCE,
                                 0, 0.0, 2.0, 0, 3, 3)
    disp = view.rasterize(None, (0, 0, 256, 224))
    disp = disp.cpu().numpy() if hasattr(disp, "cpu") else np.asarray(disp)
    assert disp.dtype == np.float32 and disp.shape == (224, 256, 3) and (disp[..., 2] == 0).any()
    for length in (3, 10):
        check(vwb, np.ascontiguousarray(disp), length)
    out = vwb.fill_holes_grass(torch.from_numpy(disp).cuda(), 5)          # and the output again as the input
    check(vwb, out.cpu().numpy(), 20)


# ---- the C ABI: host and device rasters, padded pitches, NULL and side streams --------------------------------------------------
def padded(a, pad, fill):
    b = np.full((a.shape[0], a.shape[1] + pad, 3), fill, a.dtype)
    b[:, :a.shape[1]] = a
    return b


@pytest.mark.parametrize("dtype", [np.int32, np.float32], ids=["i32", "f32"])
def test_abi_places_pitches_streams(vwb, dtype):
    import torch
    L = vwb.lib()
    w, h = 41, 37
    d = holes_field(w, h, dtype, 600, 6, 8, sprinkle=0.05)
    side = torch.cuda.Stream()
    ptype = I32 if dtype == np.int32 else F32
    for win in ((0, 0, w, h), (5, 4, 30, 25)):
        x0, y0, ow, oh = win
        want = oi.fill_holes_grass(d, 6, win)
        for dev in (0, 1):
            for ipad, opad in ((0, 0), (3, 0), (0, 5), (2, 1)):
                for stream in ((None, side) if dev else (None,)):
                    src, dst = padded(d, ipad, -77), padded(np.zeros((oh, ow, 3), dtype), opad, -77)
                    if dev:
                        src, dst = torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda()
                    ptr = (lambda a: a.data_ptr()) if dev else (lambda a: a.ctypes.data)
                    sp = C.c_void_p(stream.cuda_stream) if stream is not None else None
                    torch.cuda.synchronize()
                    rc = L.vwb200_fill_holes_grass(ptype, ptr(src), w, h, w + ipad, 6, x0, y0, ptr(dst), ow, oh, ow + opad, dev, sp)
                    assert rc == 0, L.vwb200_last_error()
                    if stream is not None:
                        stream.synchronize()
                    out = dst.cpu().numpy() if dev else dst
                    assert same(np.ascontiguousarray(out[:, :ow]), want), (win, dev, ipad, opad, stream)
                    assert (out[:, ow:] == -77).all(), "the pitch padding was written"
                    src_np = src.cpu().numpy() if dev else src
                    assert same(np.ascontiguousarray(src_np[:, :w]), d), "the input changed"


def test_abi_rejects(vwb):
    L = vwb.lib()
    d = np.zeros((8, 8, 3), np.float32)
    o = np.zeros((8, 8, 3), np.float32)
    ok = lambda *a: L.vwb200_fill_holes_grass(*a)  # noqa: E731
    assert ok(F32, d.ctypes.data, 8, 8, 8, 2, 0, 0, o.ctypes.data, 8, 8, 8, 0, None) == 0
    assert ok(F32, d.ctypes.data, 8, 8, 8, -1, 0, 0, o.ctypes.data, 8, 8, 8, 0, None) == EARG
    assert ok(F32, d.ctypes.data, 8, 8, 8, 46341, 0, 0, o.ctypes.data, 8, 8, 8, 0, None) == EARG
    assert ok(F32, d.ctypes.data, 8, 8, 8, 46340, 0, 0, o.ctypes.data, 8, 8, 8, 0, None) == 0
    assert ok(F32, d.ctypes.data, 8, 8, 8, 2, 0, 0, d[4:].ctypes.data, 8, 4, 8, 0, None) == EARG
    assert ok(F32, d.ctypes.data, 8, 8, 8, 2, 1, 0, o.ctypes.data, 8, 8, 8, 0, None) == EARG
    assert ok(7, d.ctypes.data, 8, 8, 8, 2, 0, 0, o.ctypes.data, 8, 8, 8, 0, None) == EARG
    with pytest.raises(vwb.ArgumentErr):
        vwb.fill_holes_grass(d, -3)
    with pytest.raises(vwb.ArgumentErr):
        vwb.fill_holes_grass(d, 2, (0, 0, 9, 8))


# Traced in a process of its own, so that its profiler sessions neither depend on nor add to the ones of the rest of the suite.
TRACE_SCRIPT = """
import numpy as np, torch
import visionworkbench_b200 as v
from kernel_trace import KernelTrace


class K9Trace(KernelTrace):
    def hot(self):
        return {n for n in self.raw if "k9_" in n}


torch.cuda.init()
for dt in (torch.int32, torch.float32):
    d = torch.zeros(240, 240, 3, dtype=dt, device="cuda")
    d[..., 2] = 1
    small = d.clone(); small[50, 60, 2] = 0; small[100:103, 100:104, 2] = 0
    big = d.clone(); yy, xx = torch.meshgrid(torch.arange(240), torch.arange(240), indexing="ij")
    big[((yy - 120) ** 2 + (xx - 120) ** 2 <= 400).cuda(), 2] = 0
    ring = d.clone(); ring[20, 20:210, 2] = 0; ring[209, 20:210, 2] = 0; ring[20:210, 20, 2] = 0; ring[20:210, 209, 2] = 0
    n0 = v.kernel_launches()
    v.fill_holes_grass(small, 0)
    print("LEN0", v.kernel_launches() - n0)
    for name, x, n in (("none", d, 5), ("warp", small, 5), ("cta", big, 50), ("global", ring, 200)):
        fn = lambda: v.fill_holes_grass(x, n)
        fn()
        tr = K9Trace()
        tr.run(fn)
        print("CASE", str(dt).split(".")[-1], name, "|".join(sorted(set(tr.raw))))
"""


def test_kernel_trace():
    """len 0 launches no kernel; otherwise the labelling kernels run, and each hole class runs its k9_fill_kernel<T, WARP, SMEM>
    worker"""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here]), PYTHONNOUSERSITE="1")
    r = subprocess.run([sys.executable, "-c", TRACE_SCRIPT], cwd=here, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    cases_ = [ln.split(" ", 3)[1:] for ln in r.stdout.splitlines() if ln.startswith("CASE ")]
    assert [ln for ln in r.stdout.splitlines() if ln.startswith("LEN0 ")] == ["LEN0 0"] * 2, r.stdout
    assert len(cases_) == 8, r.stdout
    labelling = ("k9_label_init_kernel", "k9_union_kernel", "k9_flatten_kernel", "k9_claim_kernel", "k9_stats_kernel", "k9_select_kernel")
    fills = {"none": set(), "warp": {"true, true"}, "cta": {"false, true"}, "global": {"false, false"}}
    for dt, name, names in cases_:
        k9 = {n for n in names.split("|") if "k9_" in n}
        ran = {k for k in labelling if any(k in n for n in k9)}
        assert ran == set(labelling), (dt, name, names)
        got = set()
        for n in k9:
            if "k9_fill_kernel" in n:
                assert ("vwb200_dispi" if dt == "int32" else "DispF") in n, n
                got.add(n.split("<", 1)[1].split(">")[0].split(", ", 1)[1].replace("(bool)1", "true").replace("(bool)0", "false"))
        assert got == fills[name], (dt, name, names)
