"""oracle/_ref: the reference's OWN native code on this path, compiled where it lies (test infrastructure only).

The one native source of the hot path is the reprojection-flow CUDA kernel lib/flow_c/gpu_flow_kernel.cu (row a13; kernel
l.32-69, host launcher `_flow` l.82-148).  It is compiled unmodified from /root/reference with the reference's own nvcc
flags (lib/flow_c/setup_linux.py:128: default -fmad, -fPIC) except the architecture, into oracle/_ref/libgpu_flow_ref.so.
oracle/_ref/ is git-ignored (no reference code enters the history) but travels to the GPU box with the snapshot, where
tests/golden/make_golden_flow_cuda.py runs it on seeded inputs and writes the fixture tests/golden/ref_flow_cuda.npz.
Nothing else of the reference is compilable here: cpu_flow_kernel.cpp is dead code that does not link (SURVEY 2 row 10),
the rest of the path is Python on MXNet / glumpy.

    python oracle/build_ref.py        # no-op (returns None) where /root/reference does not exist
"""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = "/root/reference/lib/flow_c/gpu_flow_kernel.cu"
OUT = os.path.join(HERE, "_ref", "libgpu_flow_ref.so")
SYMBOL = b"_Z5_flowPfS_S_S_S_S_iiii"  # void _flow(float*, float*, float*, float*, float*, float*, int, int, int, int)  (gpu_flow.hpp)


def build_ref(force=False):
    if not os.path.exists(REF_SRC):
        return OUT if os.path.exists(OUT) else None
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= os.path.getmtime(REF_SRC):
        return OUT
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-shared", "--compiler-options", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-I", os.path.dirname(REF_SRC), REF_SRC, "-o", OUT])
    return OUT


if __name__ == "__main__":
    print(build_ref(force=True))
