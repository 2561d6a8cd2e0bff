"""Build the C-ABI shared library ``libfqb200.so`` in-tree with nvcc for sm_90a (H100; no torch headers needed).

    python cnn-quantization_b200/build.py

The built ``.so`` is git-ignored.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libfqb200.so")
SOURCES = [os.path.join(CSRC, "fqb200.cu")]
HEADERS = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))) + [
    os.path.join(os.path.dirname(HERE), "include", "fqb200.h")]
STAMP = LIB + ".flags"  # the nvcc flags the existing library was built with: one built with other flags is stale

# -fmad=false: the reference's arithmetic is a chain of separately rounded fp32 torch ops; the kernels spell out
# every fused multiply-add they want (__fmaf_rn) and must not get any other.  No fast-math anywhere.
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-fmad=false", "-std=c++17",
              "-shared", "-Xcompiler", "-fPIC", "-Xcompiler", "-O2"]


def nvcc_path():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return "nvcc"


def is_stale():
    if not os.path.exists(LIB):
        return True
    try:
        with open(STAMP) as f:
            if f.read().strip() != " ".join(NVCC_FLAGS):
                return True
    except OSError:
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(p) > t for p in SOURCES + HEADERS)


def build(force=False, verbose=False):
    """Compile csrc/fqb200.cu -> libfqb200.so (skipped when up to date).  Returns the library path."""
    if not force and not is_stale():
        return LIB
    cmd = [nvcc_path()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB + ".tmp"] + SOURCES
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n%s\n%s" % (" ".join(cmd), res.stderr))
    if verbose:
        sys.stderr.write(res.stderr)
    os.replace(LIB + ".tmp", LIB)
    with open(STAMP, "w") as f:
        f.write(" ".join(NVCC_FLAGS) + "\n")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
