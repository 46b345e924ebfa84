"""Opcode census of K1 fast's row-step loop, read from the compiled SASS (no GPU needed).

    python tools/k1_sass_census.py [--kx 21] [--sq] [--so visionworkbench_b200/libvwb200.so]

Compiles csrc/k1_fast.cu for sm_90a with the library's nvcc flags (or reads an already built library or cubin with
--so), disassembles k1_fast_abs_kernel<KX, SQ> with cuobjdump, takes the row-step loop -- the shortest innermost loop
that holds a warp shuffle (for <KX, false> that is fast_pass<KX, true>, the octets of 8 dx) -- and prints its opcodes grouped by the pipe that runs them.  The half-rate integer ALU pipe sets the pace of this loop
(DESIGN section 4), so `alu` is the count to watch; tests/test_k1_fast_sass.py holds it to a ceiling."""
import argparse
import collections
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "visionworkbench_b200", "csrc", "k1_fast.cu")

# base opcode (text before the first '.') -> pipe.  alu: the integer ALU pipe (half rate per sub-partition, 2 cycles per
# warp instruction); fma: the FMA pipes (IMAD forms, half rate); mio: shared memory, shuffles and atomics; ctrl: branches
# and convergence barriers; uniform: the uniform datapath (one per warp, off the vector pipes).
PIPES = {
    "alu": ("VABSDIFF", "VABSDIFF4", "IADD3", "LOP3", "VIADDMNMX", "VIMNMX", "IMNMX", "SHF", "LEA", "ISETP", "SEL",
            "PRMT", "PLOP3", "IABS", "FLO", "POPC", "BMSK", "SGXT", "VIADD", "P2R", "R2P", "FSEL", "ICMP"),
    "fma": ("IMAD", "IMUL", "FFMA", "FADD", "FMUL", "IDP", "I2FP", "F2IP"),
    "mio": ("SHFL", "LDS", "STS", "ATOMS", "LD", "ST", "LDG", "STG", "RED", "REDG", "ATOM", "ATOMG", "LDSM"),
    "ctrl": ("BRA", "BSSY", "BSYNC", "WARPSYNC", "EXIT", "RET", "CALL", "NOP", "YIELD", "BAR"),
}
PIPE_OF = {op: pipe for pipe, ops in PIPES.items() for op in ops}
INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_.]*)(.*?);")


def pipe_of(opcode):
    base = opcode.split(".")[0]
    if base.startswith("U") and base not in PIPE_OF:
        return "uniform"
    return PIPE_OF.get(base, "other")


def mangled(kx, sq):
    return f"_ZN6vwb20018k1_fast_abs_kernelILi{kx}ELb{int(sq)}EEEvPKtS2_NS_8FastGeomEP12vwb200_dispilPjPtPy"


def _cuobjdump():
    for p in (shutil.which("cuobjdump"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")):
        if p and os.path.exists(p):
            return p
    raise RuntimeError("cuobjdump not found")


def compile_cubin(out_dir):
    sys.path.insert(0, ROOT)
    from visionworkbench_b200 import build
    cubin = os.path.join(out_dir, "k1_fast.cubin")
    cmd = [build.nvcc()] + build.NVCC_FLAGS + ["-cubin", SRC, "-o", cubin]
    subprocess.run(cmd, check=True, capture_output=True, text=True)
    return cubin


def disassemble(binary, kx, sq):
    r = subprocess.run([_cuobjdump(), "-sass", "-fun", mangled(kx, sq), binary], capture_output=True, text=True, check=True)
    return r.stdout


def parse(sass):
    """[(address, opcode, operands)] in address order"""
    out = []
    for line in sass.splitlines():
        m = INSN.match(line)
        if m:
            out.append((int(m.group(1), 16), m.group(3), m.group(4)))
    return out


def loops(insns):
    """[(target, branch address)] of every backward branch"""
    out = []
    for addr, op, args in insns:
        m = re.search(r"0x([0-9a-f]+)\s*$", args.strip())
        if op.split(".")[0] == "BRA" and m and int(m.group(1), 16) < addr:
            out.append((int(m.group(1), 16), addr))
    return out


def row_loop(insns):
    """the instructions of the row-step loop: of the innermost loops (no other backward branch inside) that hold a SHFL,
    the shortest.  The outer loops over work units and bands hold the passes; fast_pass<KX, false> runs the same row
    step plus a width check per dx, so the shortest is fast_pass<KX, true>."""
    ls = loops(insns)
    best = None
    for lo, hi in ls:
        if any((a, b) != (lo, hi) and lo <= a and b <= hi for a, b in ls):
            continue
        body = [x for x in insns if lo <= x[0] <= hi]
        if any(x[1].startswith("SHFL") for x in body) and (best is None or len(body) < len(best)):
            best = body
    if best is None:
        raise RuntimeError("no innermost loop with a SHFL found")
    return best


def census(sass):
    """{"pipes": {pipe: count}, "opcodes": {opcode: count}, "total": n} of the row-step loop"""
    body = row_loop(parse(sass))
    ops = collections.Counter(op for _, op, _ in body)
    pipes = collections.Counter()
    for op, n in ops.items():
        pipes[pipe_of(op)] += n
    return {"pipes": dict(pipes), "opcodes": dict(ops), "total": len(body), "start": body[0][0], "end": body[-1][0]}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--kx", type=int, default=21)
    ap.add_argument("--sq", action="store_true", help="the SquaredCost instantiation")
    ap.add_argument("--so", help="read this library or cubin instead of compiling k1_fast.cu")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        binary = a.so or compile_cubin(tmp)
        c = census(disassemble(binary, a.kx, a.sq))
    print(f"k1_fast_abs_kernel<{a.kx}, {str(a.sq).lower()}> row-step loop: {c['total']} instructions "
          f"(0x{c['start']:x} .. 0x{c['end']:x})")
    for pipe in ("alu", "fma", "mio", "ctrl", "uniform", "other"):
        ops = sorted(((n, op) for op, n in c["opcodes"].items() if pipe_of(op) == pipe), reverse=True)
        if ops:
            print(f"  {pipe:8s} {c['pipes'][pipe]:4d}: " + ", ".join(f"{op} {n}" for n, op in ops))
    p = c["pipes"]
    print(f"  floors (cycles per warp row step, one sub-partition): alu {2 * p.get('alu', 0)}, "
          f"fma {2 * p.get('fma', 0)}, dispatch {c['total']}")


if __name__ == "__main__":
    main()
