"""Build libfear_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m feartracker_b200.build [--force]

The shared object is a build product and is not tracked by git.
"""
import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "libfear_b200.so")
SOURCES = ["fear_context.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]


def _newest_source_mtime() -> float:
    newest = 0.0
    for root in (CSRC, os.path.join(os.path.dirname(PKG_DIR), "include")):
        for dirpath, _, files in os.walk(root):
            for f in files:
                if f.endswith((".cu", ".cuh", ".h")):
                    newest = max(newest, os.path.getmtime(os.path.join(dirpath, f)))
    return newest


def needs_build() -> bool:
    return not os.path.isfile(LIB_PATH) or os.path.getmtime(LIB_PATH) < _newest_source_mtime()


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB_PATH
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.isfile(nvcc):
        raise RuntimeError("nvcc not found: cannot build libfear_b200.so")
    extra = os.environ.get("FEAR_NVCC_FLAGS", "").split()  # build-time only (profiling builds); nothing is read at run time
    cmd = [nvcc, *NVCC_FLAGS, *extra, "-o", LIB_PATH + ".tmp", *SOURCES]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    proc = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError(f"nvcc failed ({proc.returncode}):\n{proc.stdout}\n{proc.stderr}")
    if verbose:
        sys.stderr.write(proc.stderr)
    os.replace(LIB_PATH + ".tmp", LIB_PATH)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
