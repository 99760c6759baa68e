"""Build the C-ABI CUDA library (sm_90a, H100) in-tree with nvcc.

    python -m dolomite_engine_b200.build [--force] [--verbose]

Produces dolomite_engine_b200/lib/libdolomite_b200.so (and the host library libdolomite_data.so).  nvcc cross-compiles
without a GPU; the built libraries are git-ignored build products.
"""

from __future__ import annotations

import argparse
import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_DIR = os.path.join(_HERE, "lib")
OBJ_DIR = os.path.join(LIB_DIR, "obj")
LIB_PATH = os.path.join(LIB_DIR, "libdolomite_b200.so")
INCLUDE = os.path.join(os.path.dirname(_HERE), "include")

NVCC_FLAGS = [
    "-gencode",
    "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "-O3",
    "-std=c++17",
    "--expt-relaxed-constexpr",
    "-Xcompiler",
    "-fPIC",
    "-Xptxas",
    "-v",
]


def _nvcc() -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; the dolomite_b200 CUDA library cannot be built")
    return nvcc


def _sources() -> list[str]:
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(path: str) -> str:
    h = hashlib.sha256()
    for dep in [path] + sorted(
        [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
        + [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    ):
        with open(dep, "rb") as f:
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _compile_one(src: str, force: bool, verbose: bool) -> tuple[str, bool, str]:
    name = os.path.splitext(os.path.basename(src))[0]
    obj = os.path.join(OBJ_DIR, name + ".o")
    stamp = obj + ".sha"
    dig = _digest(src)
    if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
        return obj, False, ""
    cmd = [_nvcc(), *NVCC_FLAGS, "-I", INCLUDE, "-c", src, "-o", obj]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{proc.stdout}\n{proc.stderr}")
    with open(stamp, "w") as f:
        f.write(dig)
    log = proc.stderr if verbose else ""
    return obj, True, log


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ_DIR, exist_ok=True)
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile_one(s, force, verbose), srcs))
    objs = [r[0] for r in results]
    rebuilt = any(r[1] for r in results)
    for r in results:
        if r[2]:
            sys.stderr.write(r[2])
    if rebuilt or not os.path.exists(LIB_PATH):
        cmd = [_nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB_PATH, *objs]
        proc = subprocess.run(cmd, capture_output=True, text=True)
        if proc.returncode != 0:
            raise RuntimeError(f"link failed:\n{proc.stdout}\n{proc.stderr}")
    build_host_library(force)
    return LIB_PATH


HOST_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc_host", "data_helpers.cpp")
HOST_LIB_PATH = os.path.join(os.path.dirname(LIB_PATH), "libdolomite_data.so")


def build_host_library(force: bool = False) -> str:
    """the data-feed index builders (plain C++, no CUDA): lib/libdolomite_data.so"""
    stamp = HOST_LIB_PATH + ".sha"
    digest = _digest(HOST_SRC)
    if not force and os.path.exists(HOST_LIB_PATH) and os.path.exists(stamp) and open(stamp).read() == digest:
        return HOST_LIB_PATH
    cxx = shutil.which("g++") or "g++"
    proc = subprocess.run([cxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-fvisibility=hidden", "-o", HOST_LIB_PATH, HOST_SRC],
                          capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError(f"g++ failed for {HOST_SRC}:\n{proc.stdout}\n{proc.stderr}")
    with open(stamp, "w") as f:
        f.write(digest)
    return HOST_LIB_PATH


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    a = ap.parse_args()
    print(build(a.force, a.verbose))
