"""K11's L2 distances must round every sub, mul and add as the reference's x86-64 float code does, with no fused
multiply-add (nvcc contracts a * b + c into FFMA by default).  Read the compiled match kernels with cuobjdump: the L2
instantiation issues FADD and FMUL and no FFMA; the Hamming one counts bits with POPC.  No GPU is needed."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "build", "obj", "k11_ipmatch.o")


@pytest.fixture(scope="module")
def kernels():
    from visionworkbench_b200 import build
    build.build()
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not found")
    sass = subprocess.run([tool, "-sass", OBJ], capture_output=True, text=True, check=True).stdout
    out = {}
    for block in re.split(r"\n\s*Function : ", sass)[1:]:
        name = block.split("\n", 1)[0].strip()
        out[name] = re.findall(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", block)
    return out


def _one(kernels, pattern):
    names = [n for n in kernels if re.search(pattern, n)]
    assert len(names) == 1, (pattern, list(kernels))
    return kernels[names[0]]


def test_l2_kernel_has_no_ffma(kernels):
    ops = _one(kernels, r"k11_match_kernelILb0E")
    assert not [o for o in ops if o.startswith("FFMA")], sorted(set(ops))
    assert sum(o.startswith("FADD") for o in ops) >= 16 * 16 and sum(o.startswith("FMUL") for o in ops) >= 16 * 16


def test_finalize_kernel_has_no_dfma(kernels):
    ops = _one(kernels, r"k11_finalize_kernel")
    assert not [o for o in ops if o.startswith(("FFMA", "DFMA"))], sorted(set(ops))


def test_hamming_kernel_counts_bits(kernels):
    ops = _one(kernels, r"k11_match_kernelILb1E")
    assert sum(o.startswith("POPC") for o in ops) >= 16 * 16
