"""Time K12 (ipfind's iagd + sgrad path) on seeded 8-bit texture imagery held in device tensors: CUDA events around whole
ipfind calls and around its three stages (normalize, detect, describe), the median of --reps (min, max) after a warm-up.
With --split, the device time of each K12 kernel in one detection, from torch.profiler (CUDA activity).  The CPU baseline
is the single-threaded oracle's ipfind on a --cpu-size square crop, scaled by area.  Prints the card's
name, power limit and max SM clock.

    python tools/time_ipfind.py [--sizes 8192 16384] [--reps 5] [--cpu-size 2048] [--no-cpu] [--split]
"""
import argparse
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi failed)"


def texture(n, seed=1, cell=8):
    rng = np.random.default_rng(seed)
    base = rng.random((n // cell + 2, n // cell + 2)).astype(np.float32)
    img = np.kron(base, np.ones((cell, cell), np.float32))[:n, :n]
    img = (img + np.roll(img, 1, 0) + np.roll(img, 1, 1) + np.roll(img, (1, 1), (0, 1))) / 4
    return np.floor(img * 255).astype(np.float32)


def time_call(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms)), min(ms), max(ms)


def kernel_split(fn, reps=3):
    """{kernel: mean device ms per call} of the k12 kernels fn() launches"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        m = re.search(r"k12_\w+?(?=\()", e.name)
        if m:
            tot[m.group(0)] = tot.get(m.group(0), 0.0) + e.device_time / reps / 1000.0
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[8192, 16384])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-size", type=int, default=2048)
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--split", action="store_true")
    a = ap.parse_args()
    import torch
    import visionworkbench_b200 as v
    print(f"card: {card()}")
    for n in a.sizes:
        t = torch.from_numpy(texture(n)).cuda()
        img = v.normalize(t)
        pts = v.detect_interest_points_iagd(img, 250)
        stages = {
            "normalize": lambda: v.normalize(t),
            "detect": lambda: v.detect_interest_points_iagd(img, 250),
            "describe": lambda: v.describe_sgrad(img, pts),
            "ipfind": lambda: v.ipfind(t, ip_per_tile=250),
        }
        for name, fn in stages.items():
            med, lo, hi = time_call(fn, a.reps)
            print(f"{n}^2 {name:9s} {med:9.2f} ms (min {lo:.2f}, max {hi:.2f}); points {len(pts)}")
        if a.split:
            for k, ms in sorted(kernel_split(lambda: v.detect_interest_points_iagd(img, 250)).items(), key=lambda kv: -kv[1]):
                print(f"{n}^2 detect kernel {k}: {ms:.2f} ms")
        if not a.no_cpu:
            from oracle import ipfind as of
            c = a.cpu_size
            crop = np.ascontiguousarray(texture(n)[:c, :c])
            t0 = time.perf_counter()
            of.ipfind(crop, ip_per_tile=250)
            s = (time.perf_counter() - t0) * (n * n) / float(c * c)
            print(f"{n}^2 oracle ipfind, single thread, scaled from {c}^2: {s:.1f} s")


if __name__ == "__main__":
    main()
