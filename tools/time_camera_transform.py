"""Time epipolar rectification on an 8192 x 8192 image: camera_transform from a TSAI source camera into its NULL-lens epipolar
camera with (1) float bilinear, (2) float bicubic and (3) PixelMask<float> bilinear with a value edge, and (4)
resize_epipolar_cameras_to_fit over two 8192^2 ROIs.  CUDA events around whole calls on device tensors, the median of --reps
(min, max) after a warm-up.  Bytes are algorithmic: 4 B read and 4 B written a float pixel, 8 + 8 for a masked one, against
3.35 TB/s of HBM3.  fp64 operations a pixel are counted from pinhole.cuh for this pair (NULL pixel_to_vector, TSAI
point_to_pixel and its check): 156 plus 121 per Newton-Raphson iteration of the check's undistortion; the mean iteration count
comes from the oracle on 4096 sampled pixels, and the rate is against 34 TFLOP/s (H100 SXM fp64, non-tensor).  The CPU
baseline is the single-threaded oracle on the top-left 1024 x 1024 tile, scaled per pixel.  Prints the card's name, power
limit and max SM clock.

    python tools/time_camera_transform.py [--size 8192] [--reps 3] [--no-cpu]
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
FP64 = 34e12
TSAI = (-0.12, 0.03, 1e-3, -2e-3, 0.01)
FP64_FIXED, FP64_PER_NR = 156, 121


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi failed)"


def cameras(n):
    """a pair f = 0.9 n px apart by 1 along x with small tilts; the left one has the TSAI lens"""
    from scipy.spatial.transform import Rotation
    out = []
    for k, rv in enumerate(((0.01, -0.02, 0.005), (-0.015, 0.01, 0.0))):
        out.append(dict(center=(float(k), 0.02 * k, 0.0), rotation=Rotation.from_rotvec(rv).as_matrix(), fu=0.9 * n, fv=0.9 * n, cu=n / 2.0,
                        cv=n / 2.0, u=(1, 0, 0), v=(0, 1, 0), w=(0, 0, 1), pixel_pitch=1.0, tsai=TSAI if k == 0 else None))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--tile", type=int, default=1024)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    import torch

    import visionworkbench_b200 as v
    from oracle import epipolar as oe
    from oracle import triangulate as ot
    from oracle import warp as ow
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

    cams = cameras(N)
    e0, e1 = oe.epipolar(*cams)
    e0, e1, s0, _ = oe.resize_epipolar(*cams, e0, e1, (0, 0, N, N), (0, 0, N, N))
    src, dst, dst1 = api(cams[0]), api(e0), api(e1)
    g = torch.Generator(device="cuda").manual_seed(1)
    gray = torch.rand(N, N, device="cuda", generator=g) * 255
    masked = torch.stack([gray, (torch.rand(N, N, device="cuda", generator=g) > 0.1).float()], -1).contiguous()
    win = (0, 0, N, N)

    rng = np.random.default_rng(0)
    its = []
    for p in rng.uniform((0, 0), (N, N), (4096, 2)):
        q = oe.camera_reverse(cams[0], e0, p)
        its.append(ot.tsai_undistort(cams[0], q * cams[0]["pixel_pitch"])[2])
    nr = float(np.mean(its))
    flops = FP64_FIXED + FP64_PER_NR * nr
    print(f"epipolar output {s0[0]} x {s0[1]}; timed window {N} x {N}; mean NR iterations of the check {nr:.2f} a pixel -> {flops:.0f} fp64 ops a pixel")

    rows = [("float bilinear, TSAI -> NULL", lambda: v.camera_transform(gray, src, dst, bbox=win), 8, True),
            ("float bicubic, TSAI -> NULL", lambda: v.camera_transform(gray, src, dst, bbox=win, interp=v.INTERP_BICUBIC), 8, True),
            ("masked bilinear, value edge", lambda: v.camera_transform(masked, src, dst, bbox=win, edge=v.EDGE_VALUE, edge_value=(0.0, 0.0)), 16, True),
            ("resize_epipolar_cameras_to_fit", lambda: v.resize_epipolar_cameras_to_fit(src, api(cams[1]), dst, dst1, win, win), 0, False)]
    results = []
    for name, fn, bpp, per_px in rows:
        ms, lo, hi = timed(fn)
        extra = ""
        if per_px:
            gbs = bpp * N * N / (ms * 1e-3)
            gf = flops * N * N / (ms * 1e-3)
            extra = f"  {bpp} B/px {gbs / 1e9:6.0f} GB/s = {100 * gbs / HBM:4.1f} % of 3.35 TB/s;  {gf / 1e12:5.2f} TFLOP/s fp64 = {100 * gf / FP64:4.1f} % of 34"
        results.append((name, ms))
        print(f"{name:<32s} {ms:9.2f} ms (min {lo:.2f}, max {hi:.2f}){extra}", flush=True)
    if a.no_cpu:
        return
    print(f"CPU baseline: single-threaded oracle on the top-left {T} x {T} tile (scaled to {N} x {N}; resize: the perimeter scaled)")
    img = gray[:T, :T].cpu().numpy()
    mimg = masked[:T, :T].cpu().numpy()
    scale = (N / T) ** 2
    t0 = time.perf_counter(); oe.camera_transform(img, cams[0], e0, (0, 0, T, T), ow.BILINEAR, ow.ZERO); s1 = time.perf_counter() - t0
    t0 = time.perf_counter(); oe.camera_transform(img, cams[0], e0, (0, 0, T, T), ow.BICUBIC, ow.ZERO); s2 = time.perf_counter() - t0
    t0 = time.perf_counter(); oe.camera_transform(mimg, cams[0], e0, (0, 0, T, T), ow.BILINEAR, oe.VALUE); s3 = time.perf_counter() - t0
    t0 = time.perf_counter(); oe.resize_epipolar(*cams, e0, e1, (0, 0, T, T), (0, 0, T, T)); s4 = time.perf_counter() - t0
    for (name, ms), s, sc in zip(results, (s1, s2, s3, s4), (scale, scale, scale, N / T)):
        print(f"  {name:<32s} {s * 1e3:9.1f} ms on {T}^2  ~{s * sc * 1e3:10.0f} ms at {N}^2  ({s * sc * 1e3 / ms:7.0f} x the device)", flush=True)


if __name__ == "__main__":
    main()
