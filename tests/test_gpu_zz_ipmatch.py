"""K11 on the device against the oracle, bit for bit (indices, and first_pick / second_pick as float64): sizes from empty to
4097 x 5003, few queries against many candidates (the split path) and the reverse, descriptor lengths 0 to 1681, duplicated
candidates (ties, first == second), one polarity, no candidate and a single candidate, every threshold class, inf / NaN and
overflowing values, Hamming on ORB-like bytes and lengths that are not multiples of 8 or 4, CUDA tensors with padded rows on a
side stream; which kernels each case ran; and a planted correspondence through match -> remove_duplicates -> .match file."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from oracle import ipmatch as om

pytestmark = pytest.mark.gpu
THRESHOLDS = (0.0, 0.5, 0.8, 1.0, np.inf, np.nan)


@pytest.fixture(scope="module")
def vwb():
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "GPU tests need a CUDA device: the engine has no CPU path"
    return v


def lists(seed, n1, n2, dim, dup=False, pol="mix", kind="normal"):
    rng = np.random.default_rng(seed)
    if kind == "bytes":
        d1 = rng.integers(0, 256, (n1, dim)).astype(np.float32)
        d2 = rng.integers(0, 256, (n2, dim)).astype(np.float32)
    else:
        d1 = rng.normal(0, 1, (n1, dim)).astype(np.float32)
        d2 = rng.normal(0, 1, (n2, dim)).astype(np.float32)
    if dup and n2 > 3:
        d2[1::3] = d2[0::3][: len(d2[1::3])]
        m = min(n1, n2) // 2
        d1[:m] = d2[:m]
    if pol == "mix":
        p1, p2 = rng.random(n1) < 0.5, rng.random(n2) < 0.5
    elif pol == "one":
        p1, p2 = np.ones(n1, bool), np.ones(n2, bool)
    else:                                                            # "none": no candidate shares a query's polarity
        p1, p2 = np.ones(n1, bool), np.zeros(n2, bool)
    return d1, p1, d2, p2


def check(vwb, d1, p1, d2, p2, thr=0.5, metric="l2"):
    got = vwb.ip_match(d1, p1, d2, p2, threshold=thr, metric=metric, distances=True)
    want = om.match(d1, p1, d2, p2, thr, om.HAMMING if metric == "hamming" else om.L2)
    assert got[0].dtype == np.int32 and got[0].tolist() == want[0].tolist(), np.flatnonzero(got[0] != want[0])[:10]
    assert got[1].view(np.uint64).tolist() == want[1].view(np.uint64).tolist()
    assert got[2].view(np.uint64).tolist() == want[2].view(np.uint64).tolist()
    st = vwb.last_ipmatch_stats()
    assert st["pairs"] == len(d1) * len(d2) and st["matches"] == int((want[0] >= 0).sum()) and st["metric"] == metric
    return st


@pytest.mark.parametrize("n1,n2,dim", [(0, 5, 4), (5, 0, 4), (1, 1, 3), (2, 2, 1), (31, 33, 15), (33, 31, 64), (1000, 1000, 128),
                                       (4097, 5003, 15)])
def test_sizes(vwb, n1, n2, dim):
    check(vwb, *lists(n1 + n2, n1, n2, dim, dup=True))


@pytest.mark.parametrize("dim", [0, 1, 3, 15, 64, 128, 180, 1681])
def test_lengths(vwb, dim):
    n1, n2 = (150, 170) if dim < 1681 else (70, 90)
    check(vwb, *lists(dim, n1, n2, dim, dup=dim % 2 == 1))


def test_split_path(vwb):
    """few queries: the candidates are split over CTAs, and the split changes nothing"""
    st = check(vwb, *lists(1, 40, 20000, 64, dup=True))
    assert st["splits"] > 1
    st = check(vwb, *lists(2, 20000, 40, 3, dup=True))
    assert st["splits"] == 1


@pytest.mark.parametrize("thr", THRESHOLDS)
@pytest.mark.parametrize("pol", ["mix", "one", "none"])
def test_thresholds_and_polarity(vwb, thr, pol):
    check(vwb, *lists(7, 300, 257, 20, dup=True, pol=pol), thr=thr)


def test_single_candidate(vwb):
    d1, p1, d2, p2 = lists(3, 50, 1, 8)
    got = vwb.ip_match(d1, np.zeros(50, bool), d2, np.zeros(1, bool), distances=True)
    assert (got[0] == 0).all() and (got[2] == 1e100).all()
    check(vwb, d1, p1, d2, p2)


@pytest.mark.parametrize("case", ["inf", "nan", "overflow", "inf_minus_inf"])
def test_non_finite(vwb, case):
    d1, p1, d2, p2 = lists(11, 200, 230, 24, dup=True)
    rng = np.random.default_rng(5)
    rows1, rows2 = rng.integers(0, 200, 20), rng.integers(0, 230, 20)
    if case == "inf":
        d1[rows1, 3], d2[rows2, 7] = np.inf, -np.inf
    elif case == "nan":
        d1[rows1, 0], d2[rows2, 23] = np.nan, np.nan
    elif case == "overflow":
        d1[rows1, :] = 3e19                                          # squares of 3e19 overflow float: finite values, inf distance
        d2[rows2, 5] = -3e38
    else:
        d1[rows1, 2], d2[rows2, 2] = np.inf, np.inf
        d2[rows2, 9] = np.nan
    for thr in (0.8, 1.0, np.inf):
        check(vwb, d1, p1, d2, p2, thr=thr)


@pytest.mark.parametrize("dim", [32, 13, 6, 1, 0])
def test_hamming(vwb, dim):
    d1, p1, d2, p2 = lists(dim, 700, 900, dim, dup=True, kind="bytes")
    if dim:
        d1[::7, 0], d2[::5, -1] = 255.9, -0.5
        d1[1::9, -1] = 0.75
    for thr in (0.5, 0.8, 1.0):
        check(vwb, d1, p1, d2, p2, thr=thr, metric="hamming")


def test_hamming_rejects_non_byte_values(vwb):
    d1, p1, d2, p2 = lists(4, 20, 30, 32, kind="bytes")
    d2[17, 9] = 256.0
    d2[21, 0] = np.nan
    with pytest.raises(vwb.ArgumentErr, match=r"desc2\[17\]\[9\] = 256"):
        vwb.ip_match(d1, p1, d2, p2, metric="hamming")
    d1[3, 31] = -1.0
    with pytest.raises(vwb.ArgumentErr, match=r"desc1\[3\]\[31\] = -1"):
        vwb.ip_match(d1, p1, d2, p2, metric="hamming")


@pytest.mark.parametrize("metric", ["l2", "hamming"])
def test_cuda_tensors_on_a_side_stream(vwb, metric):
    import torch
    d1, p1, d2, p2 = lists(21, 1500, 1700, 40, dup=True, kind="bytes" if metric == "hamming" else "normal")
    want = om.match(d1, p1, d2, p2, 0.8, om.HAMMING if metric == "hamming" else om.L2)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        wide1 = torch.zeros(1500, 48, device="cuda")
        wide1[:, :40] = torch.from_numpy(d1).cuda()
        t1 = wide1[:, :40]                                           # padded rows: pitch 48
        t2 = torch.from_numpy(d2).cuda()
        idx, first, second = vwb.ip_match(t1, torch.from_numpy(p1).cuda(), t2, torch.from_numpy(p2).cuda(), 0.8, metric, distances=True)
    s.synchronize()
    assert idx.is_cuda and idx.dtype == torch.int32 and first.dtype == torch.float64
    assert idx.cpu().numpy().tolist() == want[0].tolist()
    assert np.array_equal(first.cpu().numpy(), want[1]) and np.array_equal(second.cpu().numpy(), want[2])


def test_planted_correspondence_through_a_match_file(vwb, tmp_path):
    """300 points seen in both images (shifted by (12.5, -3)) among 2000 / 2500 distractors: match -> remove_duplicates ->
    write_binary_match_file -> read_binary_match_file gives back exactly the planted pairs"""
    rng = np.random.default_rng(99)
    n, n1, n2, dim = 300, 2000, 2500, 64
    d1 = rng.normal(0, 1, (n1, dim)).astype(np.float32)
    d2 = rng.normal(0, 1, (n2, dim)).astype(np.float32)
    a, b = rng.choice(n1, n, replace=False), rng.choice(n2, n, replace=False)
    d2[b] = d1[a] + rng.normal(0, 0.01, (n, dim)).astype(np.float32)
    xy1 = rng.uniform(0, 1000, (n1, 2)).astype(np.float32)
    xy2 = rng.uniform(0, 1000, (n2, 2)).astype(np.float32)
    xy2[b] = xy1[a] + np.float32([12.5, -3.0])
    p1, p2 = np.zeros(n1, bool), np.zeros(n2, bool)
    p1[a] = p2[b] = rng.random(n) < 0.5
    idx = vwb.ip_match(d1, p1, d2, p2, threshold=0.5)
    i1 = np.flatnonzero(idx >= 0)
    i2 = idx[i1]
    keep = vwb.remove_duplicates(xy1[i1], xy2[i2])
    i1, i2 = i1[keep], i2[keep]
    ip1 = vwb.interest_points(xy1[i1, 0], xy1[i1, 1], d1[i1], polarity=p1[i1])
    ip2 = vwb.interest_points(xy2[i2, 0], xy2[i2, 1], d2[i2], polarity=p2[i2])
    path = str(tmp_path / "left__right.match")
    vwb.write_binary_match_file(path, ip1, ip2)
    r1, r2 = vwb.read_binary_match_file(path)
    got = sorted(zip(np.round(r1["x"], 3).tolist(), np.round(r1["y"], 3).tolist(), np.round(r2["x"], 3).tolist(), np.round(r2["y"], 3).tolist()))
    want = sorted(zip(np.round(xy1[a, 0], 3).tolist(), np.round(xy1[a, 1], 3).tolist(), np.round(xy2[b, 0], 3).tolist(), np.round(xy2[b, 1], 3).tolist()))
    assert got == want
    assert np.array_equal(r1["descriptor"], d1[i1]) and np.array_equal(r2["descriptor"], d2[i2])


# Traced in a process of its own, so that its profiler sessions neither depend on nor add to the ones of the rest of the suite.
TRACE_SCRIPT = """
import numpy as np, torch
import visionworkbench_b200 as v
from kernel_trace import KernelTrace


class K11Trace(KernelTrace):
    def hot(self):
        return {n for n in self.raw if "k11_" in n}


torch.cuda.init()
rng = np.random.default_rng(0)
a, b = rng.normal(0, 1, (3000, 64)).astype(np.float32), rng.normal(0, 1, (2000, 64)).astype(np.float32)
h1, h2 = rng.integers(0, 256, (3000, 32)).astype(np.float32), rng.integers(0, 256, (2000, 32)).astype(np.float32)
pa, pb = np.zeros(3000, bool), np.zeros(2000, bool)
cases = [("l2", lambda: v.ip_match(a, pa, b, pb)), ("hamming", lambda: v.ip_match(h1, pa, h2, pb, metric="hamming")),
         ("empty", lambda: v.ip_match(a, pa, b[:0], pb[:0]))]
for name, fn in cases:
    fn()
    tr = K11Trace()
    tr.run(fn)
    print("CASE", name, "|".join(n for n in tr.raw if "k11_" in n))
"""


def test_kernel_trace():
    """L2 ran the <false> match kernel and the finalize kernel; Hamming the pack kernel on both lists, the <true> match kernel
    and the finalize kernel; an empty candidate list the finalize kernel alone"""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here]), PYTHONNOUSERSITE="1")
    r = subprocess.run([sys.executable, "-c", TRACE_SCRIPT], cwd=here, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    cases = {ln.split(" ")[1]: ln.split(" ", 2)[2].split("|") for ln in r.stdout.splitlines() if ln.startswith("CASE ")}
    assert len(cases) == 3, r.stdout

    def kinds(names):
        out = []
        for n in names:
            m = re.search(r"k11_(match|finalize|pack)_kernel(?:<\(?(?:bool\)?)?(true|false|1|0)>)?", n)
            assert m, n
            out.append(m.group(1) + ({"true": "<1>", "1": "<1>", "false": "<0>", "0": "<0>"}.get(m.group(2), "")))
        return out
    assert kinds(cases["l2"]) == ["match<0>", "finalize"], cases["l2"]
    assert kinds(cases["hamming"]) == ["pack", "pack", "match<1>", "finalize"], cases["hamming"]
    assert kinds(cases["empty"]) == ["finalize"], cases["empty"]
