"""Build the test-infrastructure binaries under oracle/ (never loaded by the product):

  oracle/_build/liboracle_leaf.so   gcc build of oracle/fq_leaf.c (plain-C leaf restatement, OpenMP)
  oracle/_ref/sm_90a/int_quantization*.so  the REFERENCE's own extension (kernels/int_quantization.cpp + gemmlowp.cu),
                                    compiled unmodified for sm_90a from where the sources lie under
                                    REF_ROOT - only when that directory exists.
                                    It is the on-GPU oracle for the compiled leaf and the "kernel to beat".
  oracle/_ref/pyref/                the REFERENCE's Python hot path (pytorch_quantizer/, utils/), staged unmodified at
                                    build() time so that a GPU machine without the reference can run it (oracle/_ref is
                                    git-ignored): the live on-GPU oracle for every row of SURVEY 8a
                                    (oracle/ref_live.py imports it next to the compiled extension above).  Nothing of it
                                    is ever committed; the product never imports it.
"""
import glob
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
BUILD = os.path.join(HERE, "_build")
REFDIR = os.path.join(HERE, "_ref")
REF_ROOT = "/root/reference"
REF_KERNELS = os.path.join(REF_ROOT, "kernels")
PYREF = os.path.join(REFDIR, "pyref")
PYREF_PACKAGES = ("pytorch_quantizer", "utils")


def build_leaf(force=False):
    os.makedirs(BUILD, exist_ok=True)
    src = os.path.join(HERE, "fq_leaf.c")
    lib = os.path.join(BUILD, "liboracle_leaf.so")
    if force or not os.path.exists(lib) or os.path.getmtime(lib) < os.path.getmtime(src):
        cmd = ["gcc", "-O2", "-fopenmp", "-ffp-contract=off", "-shared", "-fPIC", "-o", lib, src, "-lm"]
        subprocess.run(cmd, check=True)
    return lib


REF_ARCH = "9.0a"                                  # TORCH_CUDA_ARCH_LIST of the reference extension
REF_EXT_DIR = os.path.join(REFDIR, "sm_90a")       # the extension lives in a directory named for its architecture


def build_reference_ext(force=False):
    """Compile the reference's CUDA extension as is (torch C++ extension, sm_90a) into oracle/_ref/sm_90a/.  Returns the
    .so path or None.  Only that directory is ever loaded (oracle/ref_live.py): a binary left elsewhere under oracle/_ref
    by a build for another architecture is never picked up."""
    found = glob.glob(os.path.join(REF_EXT_DIR, "int_quantization*.so"))
    if found and not force:
        return found[0]
    if not os.path.isdir(REF_KERNELS):
        return None
    for old in found:
        os.remove(old)
    os.makedirs(REF_EXT_DIR, exist_ok=True)
    work = os.path.join(REF_EXT_DIR, "_work")
    os.makedirs(work, exist_ok=True)
    # setup script lives in OUR tree and points at the reference sources in place (nothing is copied)
    setup_py = os.path.join(work, "setup_ref.py")
    with open(setup_py, "w") as f:
        f.write(
            "from setuptools import setup\n"
            "from torch.utils.cpp_extension import CUDAExtension, BuildExtension\n"
            "setup(name='int_quantization', ext_modules=[CUDAExtension('int_quantization', "
            "['%s/int_quantization.cpp', '%s/gemmlowp.cu'])], cmdclass={'build_ext': BuildExtension})\n"
            % (REF_KERNELS, REF_KERNELS))
    env = dict(os.environ, TORCH_CUDA_ARCH_LIST=REF_ARCH, MAX_JOBS="4")
    res = subprocess.run([sys.executable, setup_py, "build_ext", "--build-lib", REF_EXT_DIR, "--build-temp",
                          os.path.join(work, "tmp")], cwd=work, env=env, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout[-2000:] + res.stderr[-4000:])
        return None
    shutil.rmtree(work, ignore_errors=True)
    found = glob.glob(os.path.join(REF_EXT_DIR, "int_quantization*.so"))
    return found[0] if found else None


def stage_reference_python(force=False):
    """Stage the reference's Python packages (unmodified) under oracle/_ref/pyref.  Returns the directory, or None when
    neither the reference nor an earlier staging exists."""
    marker = os.path.join(PYREF, "pytorch_quantizer", "quantization", "qtypes", "int_quantizer.py")
    if not os.path.isdir(REF_ROOT):
        return PYREF if os.path.exists(marker) else None
    if os.path.exists(marker) and not force:
        return PYREF
    os.makedirs(PYREF, exist_ok=True)
    for pkg in PYREF_PACKAGES:
        dst = os.path.join(PYREF, pkg)
        shutil.rmtree(dst, ignore_errors=True)
        shutil.copytree(os.path.join(REF_ROOT, pkg), dst, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    return PYREF


if __name__ == "__main__":
    print(build_leaf(force=True))
    print(build_reference_ext(force="--force" in sys.argv))
    print(stage_reference_python(force="--force" in sys.argv))
