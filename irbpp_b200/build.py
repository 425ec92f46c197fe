"""Build the CUDA library (in-tree, sm_90a only).  ``python -m irbpp_b200.build``"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "csrc", "irbpp.cu")
import glob  # noqa: E402
# every source the library is compiled from (all of csrc/ + the public header) + this file's flags
DEPS = sorted(glob.glob(os.path.join(HERE, "csrc", "*.cu")) + glob.glob(os.path.join(HERE, "csrc", "*.cuh"))) + \
    [os.path.join(ROOT, "include", "irbpp.h"), os.path.abspath(__file__)]
OUT_DIR = os.path.join(HERE, "lib")
OUT = os.path.join(OUT_DIR, "libirbpp.so")
# experiment hook: extra -D flags and an alternative output name (IRBPP_LIB selects it at load time)
EXTRA_DEFS = os.environ.get("IRBPP_BUILD_DEFS", "").split()

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-fmad=false",                      # float64 must round exactly like NumPy: no FMA contraction
              "-Xcompiler", "-fPIC", "-shared"]


def nvcc_path():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def up_to_date():
    if not os.path.exists(OUT):
        return False
    t = os.path.getmtime(OUT)
    return all(os.path.getmtime(d) <= t for d in DEPS)


def build(force=False, verbose=False, out=None, defs=None):
    """Compile ``csrc/irbpp.cu`` -> ``lib/libirbpp.so`` (nvcc cross-compiles without a GPU)."""
    defs = EXTRA_DEFS if defs is None else defs
    if out is None:
        out = OUT
        if not force and not defs and up_to_date():
            return OUT
    os.makedirs(OUT_DIR, exist_ok=True)
    cmd = [nvcc_path()] + NVCC_FLAGS + list(defs) + (["-Xptxas", "-v"] if verbose else []) + ["-o", out, SRC]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose:
        sys.stderr.write(res.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n%s\n%s" % (" ".join(cmd), res.stderr))
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
