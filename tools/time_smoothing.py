"""Time the disparity smoothing filters on an 8192 x 8192 raster on the GPU: disparity_median_filter at k = 3 / 5 / 11,
texture_measure at k = 9 / 15 and texture_preserving_disparity_filter at max_kernel_size = 13, each on device tensors
(CUDA events around the call, the median of --reps).  For the two in-place wavefront sweeps it also prints the critical
path W + (h + 1)(H - 1) in pixel steps and the time per step.  The CPU baseline is the single-threaded oracle on a
1024 x 1024 crop, scaled per pixel.  Prints the card's name and power limit with the numbers.

    python tools/time_smoothing.py [--size 8192] [--reps 3] [--no-cpu]
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


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi failed)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    import torch

    import smoothing_reference as S
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "needs a CUDA device"
    N = a.size
    print(f"card: {card()}")
    disp = S.random_disparity(1, (N, N), 0.1)
    rng = np.random.default_rng(2)
    img = (rng.random((N, N)) * 255).astype(np.float32)
    img[: N // 2, : N // 2] = 128.0                                    # a flat quarter: the texture filter smooths there
    d0 = torch.from_numpy(disp).cuda()
    im = torch.from_numpy(img).cuda()
    work = torch.empty_like(d0)

    def timed(fn, reset=None):
        times = []
        for i in range(a.reps + 1):                                     # the first call warms up
            if reset:
                reset()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            if i:
                times.append(e0.elapsed_time(e1))
        return float(np.median(times))

    def line(name, ms, h=None):
        s = f"{name:<44s} {ms:9.2f} ms  {N * N / ms / 1e3:9.1f} Mpix/s"
        if h is not None:
            steps = N + (h + 1) * (N - 1)
            s += f"  critical path {steps} steps, {ms * 1e6 / steps:7.1f} ns/step"
        print(s, flush=True)

    for k in (3, 5, 11):
        line(f"disparity_median_filter k={k}", timed(lambda: v.disparity_median_filter(work, k), lambda: work.copy_(d0)), (k - 1) // 2)
    tex = {}
    for k in (9, 15):
        ms = timed(lambda: tex.__setitem__(k, v.texture_measure(im, k)))
        line(f"texture_measure k={k}", ms)
    t15 = tex[15]
    tmax = float(np.float32(0.85) * np.float32(t15.max().item()))
    print(f"texture_max = 0.85 * max(texture_measure k=15) = {tmax:.6g}; pixels with a kernel >= 3: "
          f"{int(((tmax - t15) * (13 / tmax) >= 2).sum().item())} of {N * N}")
    line("texture_preserving_disparity_filter max_k=13",
         timed(lambda: v.texture_preserving_disparity_filter(work, t15, tmax, 13), lambda: work.copy_(d0)), 6)

    if a.no_cpu:
        return
    import oracle.smoothing as oracle
    c = 1024
    dc, ic = np.ascontiguousarray(disp[:c, :c]), np.ascontiguousarray(img[:c, :c])
    tc = t15[:c, :c].cpu().numpy()
    print(f"CPU baseline: single-threaded oracle on a {c} x {c} crop (scaled to {N} x {N})")
    for name, fn in ([(f"disparity_median_filter k={k}", lambda k=k: oracle.disparity_median_filter(dc, k)) for k in (3, 5, 11)]
                     + [(f"texture_measure k={k}", lambda k=k: oracle.texture_measure(ic, k)) for k in (9, 15)]
                     + [("texture_preserving_disparity_filter max_k=13", lambda: oracle.texture_preserving_disparity_filter(dc, tc, tmax, 13))]):
        t = time.perf_counter()
        fn()
        s = time.perf_counter() - t
        print(f"  {name:<44s} {s * 1e3:9.1f} ms on {c}^2  ~{s * (N / c) ** 2:8.1f} s at {N}^2", flush=True)


if __name__ == "__main__":
    main()
