"""Build libfsb200.so (sm_90a) in-tree with nvcc.  Used by __graft_entry__.build() and `python -m fasterseg_b200.build`."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libfsb200.so")
SOURCES = ["api.cu", "conv_tc.cu", "conv_direct.cu", "resize.cu", "bn.cu", "train.cu", "wgrad_tc.cu", "train_fused.cu", "loss.cu", "optim.cu", "dp.cu", "peer.cu", "latency.cu", "stem_fused.cu"]
HEADERS = ["fsb_common.cuh", "fsb_internal.h", os.path.join("..", "..", "include", "fsb200.h")]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    for f in SOURCES + HEADERS:
        p = os.path.join(CSRC, f)
        if os.path.exists(p) and os.path.getmtime(p) > t:
            return True
    return False


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
           "-shared", "-Xcompiler", "-fPIC", "-o", LIB] + SOURCES + ["-ldl"]
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
    subprocess.run(cmd, cwd=CSRC, check=True)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
