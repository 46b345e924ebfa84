"""K12 restates the reference's float and double arithmetic operation by operation: nvcc would contract a * b + c into an
FFMA / DFMA by default.  Read the compiled kernels with cuobjdump: the integral, box-filter and normalize kernels issue no
FFMA or DFMA at all.  The extrema kernel's Harris ratio and the descriptor's 1 / sqrt are IEEE-rounded divisions and square
roots, whose device sequences refine with fused operations internally; those kernels hold only those few.  No GPU is needed."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "build", "obj", "k12_ipfind.o")


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


def _fused(ops):
    return [o for o in ops if o.startswith(("FFMA", "DFMA"))]


@pytest.mark.parametrize("name", ["k12_integral_kernel", "k12_interest_kernel", "k12_norm_apply_kernel"])
def test_restated_kernels_have_no_fma(kernels, name):
    ops = _one(kernels, name)
    assert not _fused(ops), sorted(set(ops))
    assert any(o.startswith("FADD") for o in ops)


def test_box_filter_rounds_each_step(kernels):
    ops = _one(kernels, "k12_interest_kernel")
    # 8 scales x 6 boxes: 3 box adds / subs and one weighted add each, plus the weight's FMUL
    assert sum(o.startswith("FADD") for o in ops) >= 8 * 6 * 4 and sum(o.startswith("FMUL") for o in ops) >= 8 * 6


def test_division_kernels_hold_only_the_division_sequences(kernels):
    ext = _one(kernels, "k12_extrema_kernel")
    assert not [o for o in ext if o.startswith("DFMA")] and len(_fused(ext)) <= 20, sorted(set(ext))
    desc = _one(kernels, "k12_describe_kernel")
    assert not [o for o in desc if o.startswith("FFMA")] and len(_fused(desc)) <= 32, sorted(set(desc))
