"""Build libfcma_b200.so (sm_90a) in-tree with nvcc.  `python -m brainiak_b200.build`"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "fcma_b200.cu")
DEPS = [SRC, os.path.join(HERE, "csrc", "ptx_sm90.cuh"),
        os.path.join(os.path.dirname(HERE), "include", "fcma_b200.h")]
OUT = os.path.join(HERE, "libfcma_b200.so")
# diagnostic build for tools/ only: same source with -DFCMA_DIAG, which compiles the A/B tuning knobs
# (FCMA_GEMM_STAGES, FCMA_COLS_CPW, ...) in; the product library above never reads the environment
OUT_DIAG = os.path.join(HERE, "libfcma_b200_diag.so")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]


def find_nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"),
                 os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libfcma_b200.so")


def needs_build(out=OUT):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False, diag=False):
    out = OUT_DIAG if diag else OUT
    if not force and not needs_build(out):
        return out
    cmd = [find_nvcc()] + NVCC_FLAGS + (["-DFCMA_DIAG"] if diag else []) + \
        (["-Xptxas", "-v"] if verbose else []) + [SRC, "-o", out]
    env = dict(os.environ)
    # the image exports CC/CXX=/opt/gcc/bin/*, wrappers nvcc does not need: use the system g++
    if os.path.exists("/usr/bin/g++"):
        cmd[1:1] = ["-ccbin", "/usr/bin/g++"]
    res = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout)
    if verbose:
        print(res.stdout)
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, diag="--diag" in sys.argv))
