"""Build visionworkbench_b200/libvwb200.so (sm_90a only) with nvcc, in-tree (git-ignored build products)."""
import concurrent.futures
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(ROOT, "build", "obj")
SO = os.path.join(HERE, "libvwb200.so")
SOURCES = ["engine.cu", "cameras.cu", "k1_generic.cu", "k1_zone_int.cu", "k1_fast.cu", "k1_screen.cu", "k2_pyramid.cu", "k34_filters.cu", "k5_sgm.cu", "k5_sgm_paths.cu", "k6_smoothing.cu", "k7_dispmap.cu", "k8_warp.cu", "k9_inpaint.cu", "k10_triangulate.cu", "k11_ipmatch.cu", "k12_ipfind.cu", "shard.cu"]
# -ffp-contract=off: the host camera math (cameras.cu, with pinhole.cuh / cahv.cuh) rounds every product and sum as the
# reference does, never fused into an FMA; the device side uses explicitly rounded intrinsics instead
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-ffp-contract=off", "--expt-relaxed-constexpr"] + os.environ.get("VWB200_NVCC_EXTRA", "").split()


def nvcc():
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(p):
        raise RuntimeError("nvcc not found")
    return p


def _deps(src):
    hdr = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdr.append(os.path.join(ROOT, "include", "vwb200.h"))
    return [src, os.path.abspath(__file__)] + hdr      # this file holds the flags: objects built with other flags are stale


def _compile(name, verbose):
    src = os.path.join(CSRC, name)
    obj = os.path.join(OBJ, name.replace(".cu", ".o"))
    if os.path.exists(obj) and all(os.path.getmtime(d) <= os.path.getmtime(obj) for d in _deps(src)):
        return obj, False
    cmd = [nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {name}:\n{r.stdout}\n{r.stderr}")
    if verbose:
        sys.stderr.write(r.stderr)
    return obj, True


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    if force:
        for f in os.listdir(OBJ):
            os.remove(os.path.join(OBJ, f))
    with concurrent.futures.ThreadPoolExecutor(max_workers=8) as ex:
        res = list(ex.map(lambda n: _compile(n, verbose), SOURCES))
    objs = [o for o, _ in res]
    if any(ch for _, ch in res) or not os.path.exists(SO):
        # exported symbols are the extern "C" ABI only (default visibility is set in the header macro below)
        cmd = [nvcc(), "-shared", "-o", SO] + objs + ["-Xcompiler", "-fPIC", "-lcudart_static", "-ldl", "-lrt", "-lpthread"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
