"""K12 on the device against the ipfind oracle, bit for bit: normalize, detect_interest_points with
IntegralAutoGainDetector, remove_ip_near_nodata and the SGrad descriptor, alone and composed as ipfind does, down to the
.vwip bytes.  Every field is compared as raw bits, in list order."""
import os

import numpy as np
import pytest

from oracle import ipfind as of

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def v():
    import visionworkbench_b200 as v
    if v.device_count() == 0:
        pytest.skip("no CUDA device")
    return v


def texture(h, w, seed=0, levels=255, cell=4):
    rng = np.random.default_rng(seed)
    base = rng.random((h // cell + 3, w // cell + 3))
    img = np.kron(base, np.ones((cell, cell)))[:h, :w]
    img = (img + np.roll(img, 1, 0) + np.roll(img, 1, 1) + np.roll(img, (1, 1), (0, 1))) / 4
    return np.floor(img * levels).astype(np.float32)


def periodic(h, w):
    tile = np.zeros((16, 16), np.float32)
    tile[6:9, 6:9] = 1                                               # hundreds of points with a handful of interests
    return np.tile(tile, (h // 16 + 1, w // 16 + 1))[:h, :w].copy()


def random_float(h, w, seed=3):
    return np.random.default_rng(seed).standard_normal((h, w)).astype(np.float32) * 100


def same_points(got, want):
    for f in ("x", "y", "ix", "iy", "scale", "interest", "orientation"):
        assert np.asarray(got[f]).tobytes() == np.asarray(want[f]).tobytes(), f


IMAGES = {
    "1x1": lambda: np.ones((1, 1), np.float32),
    "5x5": lambda: texture(5, 5),
    "64": lambda: texture(64, 64, 1),
    "1024": lambda: texture(1024, 1024, 2),
    "1025x1030": lambda: texture(1030, 1025, 4),
    "1x4096": lambda: texture(1, 4096, 5),
    # tiles 41..50 pixels wide: scale-6 candidates land in the last 1024 flag positions the cull kernel scans
    "45x700": lambda: texture(700, 45, 15, cell=3),
    "1069x1500": lambda: texture(1500, 1069, 16, cell=3),
    "50x300": lambda: texture(300, 50, 17, cell=2),
    "3000x2000": lambda: texture(2000, 3000, 6, levels=4095, cell=6),
    "random": lambda: random_float(700, 900),
    "constant": lambda: np.full((300, 200), 7, np.float32),
    "periodic": lambda: periodic(600, 500),
}


@pytest.mark.parametrize("name", sorted(IMAGES))
def test_normalize_and_detect(v, name):
    raw = IMAGES[name]()
    img = v.normalize(raw)
    want_img = of.normalize(raw)
    assert img.tobytes() == want_img.tobytes()
    for ipt in (250, 1, 0):
        got = v.detect_interest_points_iagd(img, ipt)
        want, stats = of.detect(want_img, ipt)
        same_points(got, want)
        s = v.last_ipfind_stats()
        assert [s["tiles"], s["extrema"], s["kept"], s["culled_tiles"]] == stats


@pytest.mark.parametrize("tile_size", [256, 2048])
def test_tile_sizes(v, tile_size):
    raw = texture(2100, 1300, 8)
    img = of.normalize(raw)
    got = v.detect_interest_points_iagd(img, 40, tile_size)
    want, _ = of.detect(img, 40, tile_size)
    same_points(got, want)


def test_cull_boundaries(v):
    img = of.normalize(texture(300, 280, 9))
    allp, _ = of.detect(img, 0)
    n = len(allp)
    assert n > 3
    # num_ip of this small tile is ceil(area fraction * ip_per_tile): pick ip_per_tile so num_ip is n and n - 1
    frac = 300 * 280 / 1024 ** 2
    for target in (n, n - 1):
        ipt = int(np.ceil(target / frac - 1e-9))
        while int(np.ceil(frac * ipt)) > target:
            ipt -= 1
        assert v.tile_num_ip(280, 300, ipt) == target           # count == num_ip, then count == num_ip + 1
        got = v.detect_interest_points_iagd(img, ipt)
        want, _ = of.detect(img, ipt)
        same_points(got, want)
        assert v.last_ipfind_stats()["culled_tiles"] == (1 if target < n else 0)


@pytest.mark.parametrize("nodata,radius", [(None, 1), (0.0, 2), (17.0, 3), (None, 0)])
def test_ipfind_chain(v, tmp_path, nodata, radius):
    raw = texture(1200, 1100, 11)
    raw[100:140, 200:260] = 0 if nodata is None else nodata
    raw[:, :3] = 0
    got = v.ipfind(raw, ip_per_tile=200, nodata=nodata, nodata_radius=radius)
    pts, desc = of.ipfind(raw, ip_per_tile=200, nodata=nodata, nodata_radius=radius)
    same_points(got, pts)
    assert got["descriptor"].tobytes() == desc.tobytes()
    want = v.interest_points(pts["x"], pts["y"], desc, scale=pts["scale"], interest=pts["interest"], orientation=pts["orientation"],
                             ix=pts["ix"], iy=pts["iy"])
    a, b = tmp_path / "a.vwip", tmp_path / "b.vwip"
    v.write_binary_ip_file(str(a), got)
    v.write_binary_ip_file(str(b), want)
    assert a.read_bytes() == b.read_bytes()


def test_ip_per_image(v):
    raw = texture(2000, 3000, 12, levels=4095)
    got = v.ipfind(raw, ip_per_image=500)
    pts, desc = of.ipfind(raw, ip_per_image=500)
    same_points(got, pts)
    assert got["descriptor"].tobytes() == desc.tobytes()


def test_describe_arbitrary_points(v):
    img = of.normalize(texture(1100, 1050, 2))
    rng = np.random.default_rng(5)
    n = 300
    pts = np.zeros(n, of.POINT)
    pts["x"] = rng.uniform(0, 1049.9, n).astype(np.float32)
    pts["y"] = rng.uniform(0, 1099.9, n).astype(np.float32)
    pts["x"][:4] = [0, 1049, 0.5, 1048.75]                         # the border: zero edge
    pts["ix"], pts["iy"] = pts["x"].astype(np.int32), pts["y"].astype(np.int32)
    pts["scale"] = rng.choice([1.5, 1.875, 2.34375, 5.722046], n)
    pts["orientation"] = rng.uniform(-3, 3, n).astype(np.float32)
    want, desc = of.describe(img, pts)
    rec = v.interest_points(pts["x"], pts["y"], np.zeros((n, 0), np.float32), scale=pts["scale"], orientation=pts["orientation"])
    got = v.describe_sgrad(img, rec)
    same_points(got, want)
    assert got["descriptor"].tobytes() == desc.tobytes()


def test_non_finite_is_argument_error(v):
    for bad in (np.nan, np.inf, -np.inf):
        raw = texture(64, 64)
        raw[3, 5] = bad
        with pytest.raises(v.ArgumentErr):
            v.normalize(raw)
    with pytest.raises(v.ArgumentErr):
        v.normalize(np.full((8, 8), 3, np.float32), nodata=3)


def test_cuda_tensors_and_pitch(v):
    import torch
    raw = texture(900, 1300, 13)
    pad = np.zeros((900, 1320), np.float32)
    pad[:, :1300] = raw
    t = torch.from_numpy(pad).cuda()[:, :1300]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = v.ipfind(t, ip_per_tile=100)
    s.synchronize()
    pts, desc = of.ipfind(raw, ip_per_tile=100)
    same_points(got, pts)
    assert got["descriptor"].tobytes() == desc.tobytes()
    img = v.normalize(t)
    assert isinstance(img, torch.Tensor) and img.cpu().numpy().tobytes() == of.normalize(raw).tobytes()


def test_8192_64_tiles(v):
    raw = texture(8192, 8192, 14, cell=8)
    got = v.ipfind(raw, ip_per_tile=250)
    pts, desc = of.ipfind(raw, ip_per_tile=250)
    assert v.last_ipfind_stats()["described"] == len(pts)
    same_points(got, pts)
    assert got["descriptor"].tobytes() == desc.tobytes()


def render_view(size, x0, y0, seed=21):
    """a window of one large rendered scene: two views overlap where their windows do"""
    scene = texture(size + 400, size + 400, seed, cell=5)
    return np.ascontiguousarray(scene[y0:y0 + size, x0:x0 + size])


def test_chain_to_match_file(v, tmp_path):
    """ipfind on two overlapping views -> ip_match (L2, 0.8) -> remove_duplicates -> .match, byte-identical to the oracle's
    chain (the oracle's ipfind with the matcher oracle)"""
    from oracle import ipmatch as om
    a, b = render_view(900, 0, 0), render_view(900, 37, 23)
    ga, gb = v.ipfind(a, ip_per_tile=400), v.ipfind(b, ip_per_tile=400)
    pa, da = of.ipfind(a, ip_per_tile=400)
    pb, db = of.ipfind(b, ip_per_tile=400)
    assert ga["descriptor"].tobytes() == da.tobytes() and gb["descriptor"].tobytes() == db.tobytes()
    idx = v.ip_match(ga["descriptor"], ga["polarity"].astype(bool), gb["descriptor"], gb["polarity"].astype(bool), 0.8)
    want_idx, _, _ = om.match(da, np.zeros(len(da), np.uint8), db, np.zeros(len(db), np.uint8), 0.8)
    assert np.array_equal(idx, want_idx)
    i1 = np.nonzero(idx >= 0)[0]
    m1, m2 = ga[i1], gb[idx[i1]]
    keep = v.remove_duplicates(np.stack([m1["x"], m1["y"]], 1), np.stack([m2["x"], m2["y"]], 1))
    okeep = om.remove_duplicates(np.stack([pa["x"][i1], pa["y"][i1]], 1), np.stack([pb["x"][want_idx[i1]], pb["y"][want_idx[i1]]], 1))
    assert np.array_equal(keep, okeep) and len(keep) > 20
    # the planted shift: most kept matches move by (-37, -23)
    shift = np.stack([m2["x"][keep] - m1["x"][keep], m2["y"][keep] - m1["y"][keep]], 1)
    assert np.mean(np.all(shift == [-37, -23], axis=1)) > 0.8
    def rec(p, d, sel):
        return v.interest_points(p["x"][sel], p["y"][sel], d[sel], scale=p["scale"][sel], interest=p["interest"][sel],
                                 orientation=p["orientation"][sel], ix=p["ix"][sel], iy=p["iy"][sel])
    got_file, want_file = tmp_path / "got.match", tmp_path / "want.match"
    v.write_binary_match_file(str(got_file), m1[keep], m2[keep])
    v.write_binary_match_file(str(want_file), rec(pa, da, i1[okeep]), rec(pb, db, want_idx[i1][okeep]))
    assert got_file.read_bytes() == want_file.read_bytes()


# Traced in a process of its own, so that its profiler sessions neither depend on nor add to the ones of the rest of the suite.
TRACE_SCRIPT = """
import numpy as np, torch
import visionworkbench_b200 as v
from kernel_trace import KernelTrace


class K12Trace(KernelTrace):
    def hot(self):
        return {n for n in self.raw if "k12_" in n}


torch.cuda.init()
rng = np.random.default_rng(0)
img = np.floor(np.kron(rng.random((300, 300)), np.ones((4, 4))) * 255).astype(np.float32)
t = torch.from_numpy(img).cuda()
pts = v.detect_interest_points_iagd(v.normalize(t), 250)
cases = [("ipfind", lambda: v.ipfind(t, ip_per_tile=250)), ("nodata", lambda: v.remove_ip_near_nodata(t, pts, 0.0, 2))]
for name, fn in cases:
    fn()
    tr = K12Trace()
    tr.run(fn)
    print("CASE", name, "|".join(n for n in tr.raw if "k12_" in n))
"""


def test_kernel_trace():
    """ipfind ran the normalize, integral, interest, extrema, cull, nodata and describe kernels (and no kernel outside K12);
    remove_ip_near_nodata the nodata kernel alone"""
    import re
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here]), PYTHONNOUSERSITE="1")
    r = subprocess.run([sys.executable, "-c", TRACE_SCRIPT], cwd=here, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    cases = {ln.split(" ")[1]: ln.split(" ", 2)[2].split("|") for ln in r.stdout.splitlines() if ln.startswith("CASE ")}
    assert len(cases) == 2, r.stdout
    fams = {k: {re.search(r"(k12_\w+?)\(", n).group(1) for n in names if n} for k, names in cases.items()}
    assert fams["ipfind"] == {"k12_norm_stats_kernel", "k12_norm_apply_kernel", "k12_integral_kernel", "k12_interest_kernel",
                              "k12_extrema_kernel", "k12_cull_kernel", "k12_nodata_kernel", "k12_describe_kernel"}, fams
    assert fams["nodata"] == {"k12_nodata_kernel"}, fams
