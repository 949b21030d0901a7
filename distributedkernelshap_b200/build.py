"""Builds ``libdks.so`` (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100)."""
import os
import shutil
import subprocess

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
REPO_ROOT = os.path.dirname(PKG_DIR)
CSRC = os.path.join(PKG_DIR, "csrc")
INCLUDE = os.path.join(REPO_ROOT, "include")
LIB_PATH = os.path.join(PKG_DIR, "libdks.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-shared", "-Xcompiler", "-fPIC",
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh"))) + \
        [os.path.join(INCLUDE, "dks.h")]


def is_stale():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(s) > t for s in sources())


def find_nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def build_library(force=False, verbose=False):
    """Compile csrc/dks.cu -> libdks.so if missing or older than its sources.  Returns the library path."""
    if not force and not is_stale():
        return LIB_PATH
    nvcc = find_nvcc()
    if nvcc is None:
        raise RuntimeError("nvcc not found: cannot build libdks.so (expected a prebuilt library next to the package)")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
        ["-I" + INCLUDE, "-I" + CSRC, os.path.join(CSRC, "dks.cu"), "-o", LIB_PATH + ".tmp"]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + proc.stdout + proc.stderr)
    os.replace(LIB_PATH + ".tmp", LIB_PATH)
    if verbose:
        print(proc.stderr)
    return LIB_PATH


if __name__ == "__main__":
    print(build_library(force=True, verbose=True))
