"""K1 fast's row step is paced by the integer ALU pipe (DESIGN section 4): the u16 unpack runs on the FMA pipe as
IMAD.HI / IMAD, the ring rows are pointers that wrap with one compare-and-subtract, and the common path keeps a single
candidate predicate.  Hold the <21, false> row-step loop of the built library to the ALU-pipe count that reached, so
a change that moves work back onto that pipe shows up here.  Read from the compiled code with cuobjdump; no GPU is
needed."""
import importlib.util
import os
import shutil

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "visionworkbench_b200", "libvwb200.so")
ALU_MAX = 310           # 305 instructions in the loop (the rare offer path included), plus a small margin
TOTAL_MAX = 662         # the loop before the unpack moved to the FMA pipe


def _census_tool():
    spec = importlib.util.spec_from_file_location("k1_sass_census", os.path.join(ROOT, "tools", "k1_sass_census.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def census21():
    assert os.path.exists(SO), f"{SO} is not built"
    tool = _census_tool()
    try:
        tool._cuobjdump()
    except RuntimeError:
        pytest.skip("cuobjdump not found")
    return tool.census(tool.disassemble(SO, 21, False))


def test_row_step_alu_pipe_count(census21):
    alu = census21["pipes"].get("alu", 0)
    assert alu <= ALU_MAX, f"<21, false> row-step loop: {alu} ALU-pipe instructions (at most {ALU_MAX}): {census21['opcodes']}"


def test_row_step_total_count(census21):
    assert census21["total"] <= TOTAL_MAX, f"<21, false> row-step loop: {census21['total']} instructions"


def test_unpack_on_fma_pipe(census21):
    ops = census21["opcodes"]
    # 6 LDS.128 per row step = 24 words, each split into two u16 halves
    assert ops.get("IMAD.HI.U32", 0) >= 24, ops
    assert not any(op.split(".")[0] == "SHF" for op in ops), ops
