"""Time fill_holes_grass on an 8192 x 8192 float32 device disparity with round holes of diameter 1..len (one hole per
128 x 128 pixels on average, placed at random) plus 0.1 % single invalid pixels, for len 5, 21 and 50: once over the whole
image and once as 1024 x 1024 tiles (each tile is its own call, so it also reads the len border around it).  CUDA events
around the calls on device tensors, the median of --reps after a warm-up.  Each line also gives the holes found, the holes
filled, the largest 10 * max_distance^2 (sweeps) and the longest chain of synchronised steps (sweeps x levels) of one hole,
which bounds a call from below however many SMs there are.  The CPU baseline is the single-threaded oracle on the top-left
1024 x 1024 tile of the same field, scaled per pixel.  Prints the card's name, power limit and max SM clock.

    python tools/time_inpaint.py [--size 8192] [--reps 3] [--lens 5 21 50] [--no-cpu]
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


def field(n, length, seed=1):
    """a smooth float32 disparity (n, n, 3) on the device with the holes painted in"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(n, device="cuda", dtype=torch.float32), torch.arange(n, device="cuda", dtype=torch.float32),
                            indexing="ij")
    d = torch.stack([20 * torch.sin(xx / 600) + 0.002 * yy, 2 * torch.cos(yy / 900), torch.ones_like(xx)], -1)
    d[..., :2] += 0.3 * torch.randn(n, n, 2, device="cuda", generator=g)
    d[..., 2][torch.rand(n, n, device="cuda", generator=g) < 0.001] = 0
    k = (n // 128) ** 2
    r = torch.rand(k, device="cuda", generator=g) * (length / 2.0)
    cx = torch.randint(0, n, (k,), device="cuda", generator=g)
    cy = torch.randint(0, n, (k,), device="cuda", generator=g)
    h = length // 2 + 1
    oy, ox = torch.meshgrid(torch.arange(-h, h + 1, device="cuda"), torch.arange(-h, h + 1, device="cuda"), indexing="ij")
    inside = (ox[None] ** 2 + oy[None] ** 2).float() <= (r ** 2)[:, None, None]
    px, py = (cx[:, None, None] + ox[None]).expand_as(inside)[inside], (cy[:, None, None] + oy[None]).expand_as(inside)[inside]
    ok = (px >= 0) & (px < n) & (py >= 0) & (py < n)
    d[py[ok], px[ok], 2] = 0
    return d.contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--lens", type=int, nargs="+", default=[5, 21, 50])
    ap.add_argument("--tile", type=int, default=1024)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    import torch

    import visionworkbench_b200 as v
    assert v.device_count() > 0, "needs a CUDA device"
    N, T = a.size, a.tile
    print(f"card: {card()}")

    def timed(fn):
        times = []
        for i in range(a.reps + 1):                                     # the first call warms up
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            st = fn()
            e1.record()
            e1.synchronize()
            if i:
                times.append(e0.elapsed_time(e1))
        return float(np.median(times)), float(min(times)), float(max(times)), st

    def whole(d, length):
        v.fill_holes_grass(d, length)
        return v.last_fill_stats()

    def tiled(d, length):
        agg = {"holes": 0, "filled": 0, "max_sweeps": 0, "max_levels": 0, "critical_steps": 0}
        for y in range(0, N, T):
            for x in range(0, N, T):
                v.fill_holes_grass(d, length, (x, y, min(x + T, N), min(y + T, N)))
                s = v.last_fill_stats()
                for k in agg:
                    agg[k] = agg[k] + s[k] if k in ("holes", "filled") else max(agg[k], s[k])
        return agg

    fields = {}
    for length in a.lens:
        d = field(N, length, seed=length)
        fields[length] = d
        for name, fn in (("whole", whole), (f"{T}^2 tiles", tiled)):
            ms, lo, hi, st = timed(lambda: fn(d, length))
            print(f"len {length:3d} {name:<12s} {ms:9.2f} ms (min {lo:.2f}, max {hi:.2f})  holes {st['holes']:7d}  filled {st['filled']:7d}  "
                  f"max 10*dmax^2 {st['max_sweeps']:6d}  max levels {st['max_levels']:4d}  critical path {st['critical_steps']:9d} steps",
                  flush=True)
    if a.no_cpu:
        return
    import oracle.inpaint as oi
    print(f"CPU baseline: single-threaded oracle on the top-left {T} x {T} tile (scaled to {N} x {N})")
    for length in a.lens:
        d = fields[length].cpu().numpy()
        t0 = time.perf_counter()
        _, st = oi.fill_holes_grass(d, length, (0, 0, T, T), stats=True)
        s = time.perf_counter() - t0
        print(f"  len {length:3d} {s * 1e3:10.1f} ms on {T}^2 ({st[1]} holes filled)  ~{s * (N / T) ** 2 * 1e3:11.0f} ms at {N}^2", flush=True)


if __name__ == "__main__":
    main()
