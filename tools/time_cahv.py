"""Time the CAHV / CAHVOR device paths on 8192 x 8192 rasters: (1) a PixelMask<float> bilinear camera_transform from a CAHVOR
camera into its linearized CAHV camera, (2) a float bicubic camera_transform between two CAHV cameras (an epipolar pair's
left camera), and (3) stereo_triangulate of a float disparity through a CAHVOR pair; alternated with (4) the float bilinear
camera_transform from a TSAI pinhole into its epipolar camera, the figure DESIGN gives for the pinhole path.  CUDA events
around whole calls on device tensors, the median (min, max) of --reps calls after a warm-up.  The FP64 issue floor counts the
rounded double operations a pixel from cahv.cuh (none of them can fuse: the code is explicitly unfused) against the H100
SXM's DADD / DMUL issue rate, 132 SMs x 64 fp64 lanes x the card's max SM clock -- half the data sheet's 34 TFLOP/s, which
counts an FMA as two.  A divide or square root is counted as one operation although each issues a sequence of several
instructions, so the floor is a lower bound and the ratios to it overstate how far a kernel is from its fp64 issue limit.
The CAHVOR Newton passes come from the call's own counter where there is one, else from the oracle on sampled pixels.
Prints the card's name, power limit and max SM clock from the same process.

    python tools/time_cahv.py [--size 8192] [--reps 5]
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
FP64_LANES = 132 * 64                                        # H100 SXM: SMs x fp64 lanes (one DADD / DMUL a lane a clock)
# rounded double operations, counted from cahv.cuh
P2V_CAHV, P2V_CAHVOR_FIXED, P2V_PER_PASS = 31, 77, 16        # pixel_to_vector; CAHVOR adds the distortion terms and the passes
P2P_CAHV, P2P_CAHVOR = 23, 54                                # point_to_pixel
INTERSECT = 95                                               # the parallel test, triangulate_pair and the reflection test


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi failed)"


def max_sm_hz(line):
    """the max SM clock of card()'s line (\"..., 1980 MHz\"), or the H100 SXM's 1980 MHz when nvidia-smi did not say"""
    try:
        return float(line.rsplit(",", 1)[1].split()[0]) * 1e6
    except (IndexError, ValueError):
        return 1.98e9


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    import visionworkbench_b200 as v
    from cahv_reference import rover
    from oracle import cahv as oc
    n = args.size
    line = card()
    rate = FP64_LANES * max_sm_hz(line)
    print(f"card: {line}; fp64 DADD / DMUL issue rate {rate / 1e12:.1f} T/s")
    api = lambda c: v.CAHVModel(c["C"], c["A"], c["H"], c["V"]) if c["model"] == 1 else v.CAHVORModel(c["C"], c["A"], c["H"], c["V"], c["O"], c["R"])
    src = rover(1, n, n)
    lin = v.linearize_camera(api(src), (n, n), (n, n))
    l0, l1 = rover(2, n, n, model=1), rover(3, n, n, center=(0.0, -0.5, 0.0), model=1)
    e0, _ = v.epipolar(api(l0), api(l1))
    c0, c1 = rover(4, n, n), rover(5, n, n, center=(0.0, -0.5, 0.0))
    gen = torch.Generator(device="cuda").manual_seed(0)
    masked = torch.rand(n, n, 2, device="cuda", generator=gen)
    masked[..., 1] = 1.0
    gray = torch.rand(n, n, device="cuda", generator=gen)
    disp = torch.zeros(n, n, 3, device="cuda")
    disp[..., 0] = -20.0 + torch.rand(n, n, device="cuda", generator=gen)
    disp[..., 2] = 1.0
    pin0 = v.PinholeModel((0, 0, 0), np.eye(3), 0.9 * n, 0.9 * n, n / 2, n / 2, distortion_model=v.TsaiLensDistortion((-0.12, 0.03, 1e-3, -2e-3, 0.01)))
    pin1 = v.PinholeModel((1, 0, 0), np.eye(3), 0.9 * n, 0.9 * n, n / 2, n / 2)
    pe0, _ = v.epipolar(pin0, pin1)
    rng = np.random.default_rng(0)
    samples = rng.uniform(0, n - 1, (2048, 2))
    passes = np.mean([oc.pixel_to_vector(src, p)[2] for p in samples])
    v.stereo_triangulate(disp, api(c0), api(c1))
    tri_passes = v.last_triangulation_stats()["cahvor_iterations"] / (n * n)
    cases = [
        ("masked bilinear CAHVOR -> CAHV", lambda: v.camera_transform(masked, api(src), lin, edge=v.EDGE_VALUE, edge_value=(0.0, 0.0)),
         P2V_CAHV + 3 + P2P_CAHVOR),
        ("gray bicubic CAHV -> CAHV", lambda: v.camera_transform(gray, api(l0), e0, interp=v.INTERP_BICUBIC), P2V_CAHV + 3 + P2P_CAHV + 40),
        ("float-disparity triangulation, CAHVOR pair", lambda: v.stereo_triangulate(disp, api(c0), api(c1)),
         2 * P2V_CAHVOR_FIXED + P2V_PER_PASS * tri_passes + INTERSECT),
        ("gray bilinear TSAI pinhole -> epipolar (DESIGN's pinhole figure)", lambda: v.camera_transform(gray, pin0, pe0), None),
    ]
    times = {name: [] for name, _, _ in cases}
    for name, fn, _ in cases:                                # warm every shape first
        fn()
    for _ in range(args.reps):                               # alternate the cases call by call
        for name, fn, _ in cases:
            times[name] += timed(fn, 1)
    print(f"size {n} x {n}; CAHVOR Newton passes a ray: {passes:.2f} (transform source, oracle, 2048 samples), "
          f"{tri_passes / 2:.2f} (triangulation, device counter)")
    for name, _, ops in cases:
        t = np.array(times[name])
        out = f"{name}: median {np.median(t):.2f} ms (min {t.min():.2f}, max {t.max():.2f})"
        if ops is not None:
            floor = n * n * ops / rate * 1e3
            out += f"; FP64 issue floor {floor:.2f} ms ({ops:.0f} ops a pixel), {np.median(t) / floor:.2f}x the floor"
        print(out)


if __name__ == "__main__":
    main()
