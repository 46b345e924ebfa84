"""Time transform(image, tx, edge, interp) on an 8192 x 8192 float32 device image (CUDA events around the call on device
tensors, the median of --reps after a warm-up call): a projective HomographyTransform with bilinear, bicubic and nearest-pixel
interpolation, and a DisparityTransform with bilinear interpolation.  GB/s counts 4 bytes read and 4 written per output pixel
(the gathers that hit cache are not counted; a DisparityTransform also reads 12 bytes of disparity, listed beside it), against
the 3.35 TB/s data-sheet bandwidth; the fp64 operations per pixel are the explicitly rounded double steps of the kernel.  The
CPU baseline is the single-threaded oracle on a 1024 x 1024 crop, scaled per pixel.  Prints the card's name, power limit and
max SM clock with the numbers.

    python tools/time_warp.py [--size 8192] [--reps 3] [--no-cpu]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H = np.array([[1.01, 0.02, -12.5], [-0.015, 0.995, 7.25], [2e-6, -3e-6, 1.0]])
# fp64 operations per pixel: the homography's reverse is 6 mul + 6 add + 2 div; bicubic adds 2 offsets, 2 x 17 weight steps,
# 4 rows of 4 mul + 3 add, 4 mul + 3 add across rows and the final * 0.25; nearest adds the two +-0.5 of _round; the
# disparity's reverse is 2 adds; bilinear interpolates in float
CASES = (("homography", "bilinear", 14), ("homography", "bicubic", 14 + 2 + 34 + 28 + 7 + 1), ("homography", "nearest", 16),
         ("disparity", "bilinear", 2))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi failed)"


def inputs(n, seed=1):
    """a smooth image and a smooth disparity with 10 % invalid pixels"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:n, 0:n].astype(np.float32)
    im = (100 * np.sin(xx / 97) * np.cos(yy / 61) + 5 * rng.standard_normal((n, n), np.float32)).astype(np.float32)
    dx = 20 * np.sin(xx / 600) + 0.002 * yy + 0.3 * rng.standard_normal((n, n), np.float32)
    dy = 2 * np.cos(yy / 900) + 0.2 * rng.standard_normal((n, n), np.float32)
    v = (rng.random((n, n)) >= 0.1).astype(np.float32)
    return im, np.stack([dx, dy, v], -1).astype(np.float32)


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
    interp = {"bilinear": v.INTERP_BILINEAR, "bicubic": v.INTERP_BICUBIC, "nearest": v.INTERP_NEAREST}

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

    im, d = inputs(N)
    ti, td = torch.from_numpy(im).cuda(), torch.from_numpy(d).cuda()
    txs = {"homography": v.HomographyTransform(H), "disparity": v.DisparityTransform(td)}
    for kind, ip, flops in CASES:
        ms = timed(lambda: v.transform(ti, txs[kind], None, v.EDGE_ZERO, interp[ip]))
        gb = 8.0 * N * N / 1e9
        extra = f"  (+{12.0 * N * N / 1e9:.2f} GB of disparity read)" if kind == "disparity" else ""
        print(f"{kind:<10s} {ip:<8s} {ms:8.3f} ms  {gb / ms * 1e3:7.0f} GB/s ({100 * gb / ms * 1e3 / 3350:4.1f} % of 3.35 TB/s)  "
              f"{flops:3d} fp64 op/px = {flops * N * N / ms / 1e6:7.1f} GFLOP/s{extra}", flush=True)
    del ti, td
    if a.no_cpu:
        return
    import oracle.warp as wo
    c = 1024
    print(f"CPU baseline: single-threaded oracle on a {c} x {c} crop (scaled to {N} x {N})")
    ic, dc = np.ascontiguousarray(im[:c, :c]), np.ascontiguousarray(d[:c, :c])
    kinds = {"homography": wo.HOMOGRAPHY, "disparity": wo.DISPARITY}
    winterp = {"bilinear": wo.BILINEAR, "bicubic": wo.BICUBIC, "nearest": wo.NEAREST}
    for kind, ip, _ in CASES:
        t0 = time.perf_counter()
        wo.transform(ic, kinds[kind], winterp[ip], wo.ZERO, (0, 0, c, c), matrix=txs["homography"].H_inverse, disparity=dc)
        s = time.perf_counter() - t0
        print(f"  {kind:<10s} {ip:<8s} {s * 1e3:8.1f} ms on {c}^2  ~{s * (N / c) ** 2 * 1e3:9.0f} ms at {N}^2", flush=True)


if __name__ == "__main__":
    main()
