"""Time the dense triangulation calls on an 8192 x 8192 float32 device disparity with 10 % invalid pixels, from a seeded
rectified pinhole pair (f = 8192 px, baseline 1): (a) stereo_triangulate with the NULL lens, (a) with a TSAI lens, (b)
StereoModel on the image with the TSAI lens, and (c) universe radius in place on (b)'s points.  CUDA events around whole calls
on device tensors, the median of --reps (min, max) after a warm-up.  Bytes are algorithmic: 12 B in and 24 B out a pixel, plus
8 B of error for (b); 24 B in and 24 B out for (c); the rate is against 3.35 TB/s of HBM3.  The Tsai rows also give the mean
Newton-Raphson iterations per undistorted ray.  The CPU baseline is the single-threaded oracle on the top-left 1024 x 1024
tile, scaled per pixel.  Prints the card's name, power limit and max SM clock.

    python tools/time_triangulate.py [--size 8192] [--reps 3] [--no-cpu]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM = 3.35e12
TSAI = (-0.12, 0.03, 1e-3, -2e-3, 0.01)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi failed)"


def cameras(n, tsai):
    """a rectified pair: rotation about a tilted axis, f = n pixels, principal point at the centre, baseline 1 along the rows"""
    a = 0.3
    R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    c1 = np.array([0.5, -0.2, 1.0])
    c2 = c1 + R @ np.array([1.0, 0.0, 0.0])
    f = float(n)
    return [dict(center=tuple(c), rotation=R, fu=f, fv=f, cu=n / 2.0, cv=n / 2.0, u=(1, 0, 0), v=(0, 1, 0), w=(0, 0, 1), pixel_pitch=1.0,
                 tsai=tsai) for c in (c1, c2)]


def field(n, seed=1):
    """float32 (n, n, 3) device disparity: a smooth surface 150 .. 250 pixels of disparity, 10 % invalid"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(n, device="cuda", dtype=torch.float32), torch.arange(n, device="cuda", dtype=torch.float32),
                            indexing="ij")
    d = torch.stack([-200 - 50 * torch.sin(xx / 900) * torch.cos(yy / 700), 0.01 * torch.randn(n, n, device="cuda", generator=g),
                     torch.ones_like(xx)], -1)
    d[..., 0] += 0.2 * torch.randn(n, n, device="cuda", generator=g)
    d[..., 2][torch.rand(n, n, device="cuda", generator=g) < 0.1] = 0
    return d.contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--tile", type=int, default=1024)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    import torch

    import visionworkbench_b200 as v
    assert v.device_count() > 0, "needs a CUDA device"
    N, T = a.size, a.tile
    print(f"card: {card()}")

    def api(c):
        return v.PinholeModel(c["center"], c["rotation"], c["fu"], c["fv"], c["cu"], c["cv"], c["u"], c["v"], c["w"],
                              None if c["tsai"] is None else v.TsaiLensDistortion(c["tsai"]), c["pixel_pitch"])

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
        return float(np.median(times)), float(min(times)), float(max(times))

    d = field(N)
    null, tsai = cameras(N, None), cameras(N, TSAI)
    nv = int((d[..., 2] != 0).sum())
    pts = {}

    def run_b():
        pts["xyz"] = v.stereo_model_points(d, api(tsai[0]), api(tsai[1]))[0]

    rows = [("(a) stereo_triangulate, NULL lens", lambda: v.stereo_triangulate(d, api(null[0]), api(null[1])), 36, None),
            ("(a) stereo_triangulate, TSAI lens", lambda: v.stereo_triangulate(d, api(tsai[0]), api(tsai[1])), 36, "a"),
            ("(b) StereoModel image, TSAI lens", run_b, 44, "b"),
            ("(c) universe radius, in place", lambda: v.universe_radius(pts["xyz"], (0.5, -0.2, 1.0), 1.0, 1e4, out=pts["xyz"]), 48, None)]
    results = []
    for name, fn, bpp, nr in rows:
        ms, lo, hi = timed(fn)
        gbs = bpp * N * N / (ms * 1e-3)
        extra = ""
        if nr:
            it = v.last_triangulation_stats()["tsai_iterations"]
            extra = f"  mean NR iterations {it / (2.0 * nv):.2f} per ray"
        results.append((name, ms))
        print(f"{name:<36s} {ms:8.2f} ms (min {lo:.2f}, max {hi:.2f})  {bpp} B/px  {gbs / 1e9:7.0f} GB/s = {100 * gbs / HBM:5.1f} % of 3.35 TB/s{extra}",
              flush=True)
    if a.no_cpu:
        return
    import oracle.triangulate as ot
    print(f"CPU baseline: single-threaded oracle on the top-left {T} x {T} tile (scaled to {N} x {N})")
    dc = np.ascontiguousarray(d[:T, :T].cpu().numpy())
    scale = (N / T) ** 2
    t0 = time.perf_counter(); ot.stereo_triangulate(dc, null[0], null[1]); s1 = time.perf_counter() - t0
    t0 = time.perf_counter(); ot.stereo_triangulate(dc, tsai[0], tsai[1]); s2 = time.perf_counter() - t0
    t0 = time.perf_counter(); xyz = ot.stereo_model(dc, tsai[0], tsai[1])[0]; s3 = time.perf_counter() - t0
    t0 = time.perf_counter(); ot.universe_radius(xyz, (0.5, -0.2, 1.0), 1.0, 1e4); s4 = time.perf_counter() - t0
    for (name, ms), s in zip(results, (s1, s2, s3, s4)):
        print(f"  {name:<36s} {s * 1e3:9.1f} ms on {T}^2  ~{s * scale * 1e3:10.0f} ms at {N}^2  ({s * scale * 1e3 / ms:7.0f} x the device)", flush=True)


if __name__ == "__main__":
    main()
