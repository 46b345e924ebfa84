"""Time the disparity resampling, range and transform operations on an 8192 x 8192 device disparity, int32 and float32:
disparity_subsample, disparity_upsample, get_disparity_range, disparity_range_mask and both transform_disparities forms
(CUDA events around the call on device tensors, the median of --reps after a warm-up call).  GB/s counts the algorithmic
bytes: each input and output pixel once (12 bytes).  The CPU baseline is the single-threaded oracle on a 1024 x 1024 crop,
scaled per pixel.  Prints the card's name, power limit and max SM clock with the numbers.

    python tools/time_dispmap.py [--size 8192] [--reps 3] [--no-cpu]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H = np.array([[0.98, 0.03, 12.5], [-0.02, 1.01, -7.25], [1.5e-5, -2e-5, 1.0]])


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi failed)"


def field(n, dtype, seed=1):
    """a smooth field with 10 % invalid pixels"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:n, 0:n].astype(np.float32)
    dx = 20 * np.sin(xx / 600) + 0.002 * yy + 0.3 * rng.standard_normal((n, n), np.float32)
    dy = 2 * np.cos(yy / 900) + 0.2 * rng.standard_normal((n, n), np.float32)
    v = (rng.random((n, n)) >= 0.1).astype(np.float32)
    d = np.stack([dx, dy, v], -1)
    return np.rint(d).astype(np.int32) if dtype == np.int32 else d


def ops(v, n):
    """(name, call on a disparity, output pixels per input pixel)"""
    return [("disparity_subsample", lambda d: v.disparity_subsample(d), 0.25),
            ("disparity_upsample", lambda d: v.disparity_upsample(d), 4.0),
            ("get_disparity_range", lambda d: v.get_disparity_range(d), 0.0),
            ("disparity_range_mask", lambda d: v.disparity_range_mask(d, (0, 0), (n, n)), 1.0),
            ("transform_disparities (lazy)", lambda d: v.transform_disparities(d, H), 1.0),
            ("transform_disparities (explicit)", lambda d: v.transform_disparities_explicit(True, (0, 0, n, n), H, d), 1.0)]


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
        for name, fn, out_ratio in ops(v, N):
            ms = timed(lambda: fn(t))
            gb = 12.0 * N * N * (1.0 + out_ratio) / 1e9
            print(f"{np.dtype(dtype).name:<8s} {name:<34s} {ms:8.3f} ms  {gb / ms * 1e3:7.0f} GB/s  ({100 * gb / ms * 1e3 / 3350:4.1f} % of 3.35 TB/s)",
                  flush=True)
        del t
    if a.no_cpu:
        return
    import oracle.dispmap as dm
    c = 1024
    print(f"CPU baseline: single-threaded oracle on a {c} x {c} crop (scaled to {N} x {N})")
    inv = np.linalg.inv(H)
    cpu = [("disparity_subsample", lambda d: dm.disparity_subsample(d)), ("disparity_upsample", lambda d: dm.disparity_upsample(d)),
           ("get_disparity_range", lambda d: dm.get_disparity_range(d)), ("disparity_range_mask", lambda d: dm.disparity_range_mask(d, (0, 0), (c, c))),
           ("transform_disparities (lazy)", lambda d: dm.transform_disparities(dm.LAZY, inv, d)),
           ("transform_disparities (explicit)", lambda d: dm.transform_disparities(dm.EXPLICIT, H, d, True))]
    for dtype in (np.int32, np.float32):
        dc = np.ascontiguousarray(host[dtype][:c, :c])
        for name, fn in cpu:
            t0 = time.perf_counter()
            fn(dc)
            s = time.perf_counter() - t0
            print(f"  {np.dtype(dtype).name:<8s} {name:<34s} {s * 1e3:8.1f} ms on {c}^2  ~{s * (N / c) ** 2 * 1e3:9.0f} ms at {N}^2", flush=True)


if __name__ == "__main__":
    main()
