"""Build libdeepim_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python mx-deepim_b200/build.py [--force] [--verbose]

raster.cu / zoom.cu / geom.cu / icp.cu / vsd.cu / bop.cu are compiled with -fmad=false: their float32 (icp.cu, vsd.cu, bop.cu:
float64)
sequences are specified operation by operation (the CPU checker used by tests/ is built with -ffp-contract=off) so that integer
outputs (bbox, masks, coverage) and the rendered images are bit-exact against the oracle.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libdeepim_b200.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
          "-Xcudafe", "--diag_suppress=177"]
UNITS = {
    "raster.cu": ["-fmad=false"],
    "zoom.cu": ["-fmad=false"],
    "geom.cu": ["-fmad=false"],
    "augment.cu": ["-fmad=false"],
    "icp.cu": ["-fmad=false"],
    "vsd.cu": ["-fmad=false"],
    "bop.cu": ["-fmad=false"],
    "net.cu": [],
    "train.cu": [],
    "capi.cu": [],
}


def _newer(src_list, target):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in src_list)


def build(force=False, verbose=False):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(HERE, "..", "include", "deepim_b200.h"))
    objs = []
    procs = []
    for unit, extra in UNITS.items():
        src = os.path.join(CSRC, unit)
        obj = os.path.join(CSRC, unit.replace(".cu", ".o"))
        objs.append(obj)
        if force or _newer([src] + headers, obj):
            cmd = [nvcc] + ARCH + COMMON + extra + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
            procs.append((unit, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for unit, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write("---- %s\n%s\n" % (unit, out))
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    if force or procs or _newer(objs, OUT):
        cmd = [nvcc] + ARCH + ["-shared", "-cudart", "static", "-o", OUT] + objs
        subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
