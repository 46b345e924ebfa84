"""Time K11 interest point matching on device tensors: L2 at --n x --n x 128 floats (SIFT-sized) and Hamming at --n x --n x 32
bytes (ORB-sized), both lists of one polarity, seeded.  CUDA events around whole ip_match calls, the median of --reps (min,
max) after a warm-up.  Element pairs are n^2 D; the L2 floor is the FP32 issue bound: 3 instructions (sub, mul, add) per
element pair at 128 lanes x 132 SMs x the max SM clock.  The CPU baseline is the single-threaded oracle on the first --cpu-rows
queries against all candidates, scaled per element pair.  Prints the card's name, power limit and max SM clock.

    python tools/time_ipmatch.py [--n 50000] [--reps 5] [--cpu-rows 20] [--no-cpu]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi failed)"


def max_sm_mhz(line):
    try:
        return float(line.split(",")[2].split()[0])
    except (IndexError, ValueError):
        return 1980.0


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-rows", type=int, default=20)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    import torch
    import visionworkbench_b200 as v
    line = card()
    print(f"card: {line}")
    n = a.n
    rng = np.random.default_rng(0)
    cases = {"l2": rng.normal(0, 1, (2, n, 128)).astype(np.float32), "hamming": rng.integers(0, 256, (2, n, 32)).astype(np.float32)}
    pol = torch.zeros(n, dtype=torch.uint8, device="cuda")
    floor_rate = 128 * 132 * max_sm_mhz(line) * 1e6 / 3                 # element pairs / s at 3 FP32 instructions each
    for metric, d in cases.items():
        t1, t2 = torch.from_numpy(d[0]).cuda(), torch.from_numpy(d[1]).cuda()
        med, lo, hi = time_call(lambda: v.ip_match(t1, pol, t2, pol, 0.8, metric), a.reps)
        st = v.last_ipmatch_stats()
        pairs = float(n) * n * d.shape[2]
        msg = f"{metric:8s} {n} x {n} x {d.shape[2]}: {med:9.2f} ms (min {lo:.2f}, max {hi:.2f})  {pairs / med / 1e9:8.1f} G element-pairs/s"
        msg += f"  splits {st['splits']}  matches {st['matches']}"
        if metric == "l2":
            msg += f"  FP32 floor {pairs / floor_rate * 1e3:.1f} ms ({pairs / floor_rate * 1e3 / med:.2f} of it)"
        if not a.no_cpu:
            from oracle import ipmatch as om
            k = min(a.cpu_rows, n)
            t0 = time.perf_counter()
            om.match(d[0][:k], np.zeros(k, bool), d[1], np.zeros(n, bool), 0.8, om.HAMMING if metric == "hamming" else om.L2)
            cpu = (time.perf_counter() - t0) / (k * float(n) * d.shape[2])
            msg += f"  oracle 1 core {1 / cpu / 1e9:.2f} G element-pairs/s (full size ~{cpu * pairs:.0f} s)"
        print(msg, flush=True)


if __name__ == "__main__":
    main()
