"""Time the neighbourhood outlier filters on an 8192 x 8192 device disparity: rm_outliers_using_{thresh,mean,stddev} and
disparity_cleanup_using_* for int32 and float32 pixels at half kernels 2 and 5 (CUDA events around the call on device
tensors, the median of --reps after a warm-up call).  The disparity is a smooth field with speckle and holes.  The CPU
baseline is the single-threaded oracle on a 1024 x 1024 crop, scaled per pixel.  Prints the card's name, power limit and
max SM clock with the numbers.

    python tools/time_outlier_filters.py [--size 8192] [--reps 3] [--no-cpu]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

FILTERS = [("rm_outliers_using_thresh", 0, 0), ("disparity_cleanup_using_thresh", 0, 1), ("rm_outliers_using_mean", 1, 0),
           ("disparity_cleanup_using_mean", 1, 1), ("rm_outliers_using_stddev", 2, 0), ("disparity_cleanup_using_stddev", 2, 1)]
PT, RT, RT_STD, MMD = 3.0, 0.5, 0.5, 3.0     # pixel_threshold, rejection_threshold (thresh / stddev), max_mean_diff


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi failed)"


def field(n, dtype, seed=1):
    """a smooth field with 2 % speckle and 5 % holes (plus invalid blobs)"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:n, 0:n].astype(np.float32)
    dx = 20 * np.sin(xx / 600) + 0.002 * yy + 0.3 * rng.standard_normal((n, n), np.float32)
    dy = 2 * np.cos(yy / 900) + 0.2 * rng.standard_normal((n, n), np.float32)
    speck = rng.random((n, n)) < 0.02
    dx[speck] += rng.uniform(-60, 60, int(speck.sum())).astype(np.float32)
    v = (rng.random((n, n)) >= 0.05).astype(np.float32)
    for _ in range(n // 8):
        cy, cx, r = rng.integers(0, n), rng.integers(0, n), rng.integers(2, 40)
        v[max(cy - r, 0):cy + r, max(cx - r, 0):cx + r] = 0
    d = np.stack([dx, dy, v], -1)
    return np.rint(d).astype(np.int32) if dtype == np.int32 else d


def args(method):
    return (PT, RT, 0.0) if method == 0 else (0.0, 0.0, MMD) if method == 1 else (PT, RT_STD, 0.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    import torch

    import visionworkbench_b200 as v
    assert v.device_count() > 0, "needs a CUDA device"
    N = a.size
    print(f"card: {card()}")

    def timed(fn):
        times = []
        for i in range(a.reps + 1):                                     # the first call warms up
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            if i:
                times.append(e0.elapsed_time(e1))
        return float(np.median(times))

    host = {}
    for dtype in (np.int32, np.float32):
        d = field(N, dtype)
        host[dtype] = d
        t = torch.from_numpy(d).cuda()
        for half in (2, 5):
            for name, m, cl in FILTERS:
                pt, rt, mmd = args(m)
                ms = timed(lambda: v.outlier_filter(m, cl, t, half, half, pt, rt, mmd))
                print(f"{np.dtype(dtype).name:<8s} h={half} {name:<32s} {ms:9.2f} ms  {N * N / ms / 1e3:9.1f} Mpix/s", flush=True)
        del t
    if a.no_cpu:
        return
    import oracle.outliers as oracle
    c = 1024
    print(f"CPU baseline: single-threaded oracle on a {c} x {c} crop (scaled to {N} x {N})")
    for dtype in (np.int32, np.float32):
        dc = np.ascontiguousarray(host[dtype][:c, :c])
        for half in (2, 5):
            for name, m, cl in FILTERS:
                pt, rt, mmd = args(m)
                t0 = time.perf_counter()
                oracle.outlier_filter(m, cl, dc, half, half, pt, rt, mmd)
                s = time.perf_counter() - t0
                print(f"  {np.dtype(dtype).name:<8s} h={half} {name:<32s} {s * 1e3:9.1f} ms on {c}^2  ~{s * (N / c) ** 2:8.1f} s at {N}^2",
                      flush=True)


if __name__ == "__main__":
    main()
