"""K1 fast runs 12 warps per SM (384 threads, one CTA), which leaves each thread at most 65536 / 384 -> 168 registers.
Every instantiation of k1_fast_abs_kernel in the built library must fit that without a stack frame: a spill would put
local-memory traffic into the row step.  Read from the compiled code with cuobjdump; no GPU is needed."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "visionworkbench_b200", "libvwb200.so")
KX = (3, 5, 7, 9, 11, 13, 15, 17, 19, 21, 23, 25, 27, 29, 31)


def _cuobjdump():
    for p in (shutil.which("cuobjdump"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")):
        if p and os.path.exists(p):
            return p
    pytest.skip("cuobjdump not found")


def _fast_kernel_usage():
    """{(KX, SQ): (REG, STACK)} of every k1_fast_abs_kernel in the library"""
    assert os.path.exists(SO), f"{SO} is not built"
    r = subprocess.run([_cuobjdump(), "-res-usage", SO], capture_output=True, text=True, check=True)
    usage, fn = {}, None
    for line in r.stdout.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            fn = re.search(r"k1_fast_abs_kernelILi(\d+)ELb([01])E", m.group(1))
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and fn:
            usage[(int(fn.group(1)), fn.group(2) == "1")] = (int(m.group(1)), int(m.group(2)))
            fn = None
    return usage


def test_k1_fast_fits_twelve_warps():
    usage = _fast_kernel_usage()
    assert set(usage) == {(k, sq) for k in KX for sq in (False, True)}, sorted(usage)
    over = {k: v for k, v in usage.items() if v[0] > 168 or v[1] != 0}
    assert not over, f"(KX, SQ): (registers, stack bytes) over 168 registers or with a stack frame: {over}"
