"""Builds libvtts.so (the C-ABI library, include/vtts.h) in-tree with nvcc for sm_90a (H100)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libvtts.so")
SOURCES = ["engine.cu", "st_gather.cu", "st_tc.cu", "t2s.cu"]
DEPS = ["engine.cu", "st_gather.cu", "st_tc.cu", "t2s.cu", "t2s.cuh", "kernels.cuh", "conv_tc.cuh", "attn_tc.cuh", "wgmma.cuh", "mas.cuh", "vc.cuh", "spk.cuh", "contentvec.cuh", "sovits.cuh", "bert.cuh", "dit.cuh", "stabletts.cuh", "hifigan.cuh", "resample.cuh", "owned.cuh", os.path.join("..", "..", "include", "vtts.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-shared",
]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, d)) > t for d in DEPS if os.path.exists(os.path.join(CSRC, d)))


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
          [os.path.join(CSRC, s) for s in SOURCES] + ["-o", LIB, "-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed building libvtts.so")
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose="-v" in sys.argv))
