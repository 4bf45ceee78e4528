"""Builds the in-tree native artefacts.

    libepropnp_b200.so   nvcc, sm_90a only (cross-compiles without a GPU)
    libhost_emul.so      g++ build of csrc/pnp_math.cuh + tests/host_emul.cpp (CPU tests only)

The .so files stay in the tree (epro-pnp_b200/lib/, git-ignored) so they travel to the GPU box.
"""
import os
import shutil
import subprocess

PKG_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))      # .../epro-pnp_b200
REPO_ROOT = os.path.dirname(PKG_ROOT)
CSRC = os.path.join(PKG_ROOT, "csrc")
LIB_DIR = os.path.join(PKG_ROOT, "lib")
INCLUDE = os.path.join(REPO_ROOT, "include")
LIB_PATH = os.path.join(LIB_DIR, "libepropnp_b200.so")
EMUL_PATH = os.path.join(LIB_DIR, "libhost_emul.so")

NVCC_FLAGS = ["-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC", "-shared", "-I", INCLUDE]

# kept for the test-side build helpers (tests/simt_native.py): the shipped library has no build options
DEFAULT_OPTIONS = []


def kernel_sources():
    """Everything the native library is compiled from (dependency list of every in-tree build)."""
    import glob
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh"))) + \
        [os.path.join(INCLUDE, "epropnp_b200.h")]


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libepropnp_b200.so")


def build_library(force=False, verbose=False):
    srcs = [os.path.join(CSRC, "pnp_kernels.cu")]
    deps = kernel_sources()
    os.makedirs(LIB_DIR, exist_ok=True)
    if force or _newer(LIB_PATH, deps):
        cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB_PATH] + srcs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
        if verbose:
            print(r.stderr)
    return LIB_PATH


def build_host_emul(force=False):
    src = os.path.join(REPO_ROOT, "tests", "host_emul.cpp")
    deps = [src, os.path.join(CSRC, "pnp_math.cuh"), os.path.join(INCLUDE, "epropnp_b200.h")]
    os.makedirs(LIB_DIR, exist_ok=True)
    if force or _newer(EMUL_PATH, deps):
        cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I", INCLUDE, "-o", EMUL_PATH, src]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("g++ failed:\n" + r.stdout + r.stderr)
    return EMUL_PATH


if __name__ == "__main__":
    print(build_library(force=True, verbose=True))
    print(build_host_emul(force=True))
