"""Build liballegro_b200.so in-tree with nvcc for sm_90a (no torch types, plain C ABI).

    python -m allegro_b200.build [--force] [--verbose]

The .so and its object files are build products (git-ignored); build() rebuilds whenever a source or flag changes.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from typing import List

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "liballegro_b200.so")
STAMP = os.path.join(LIBDIR, "build.stamp")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def sources() -> List[str]:
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest() -> str:
    h = hashlib.sha256()
    root = os.path.dirname(HERE)
    files = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))] + [os.path.join(root, "include", "allegro_b200.h")]
    for f in files:
        with open(f, "rb") as fh:
            h.update(f.encode())
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def nvcc_path() -> str:
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(p):
        raise RuntimeError("nvcc not found; the CUDA extension cannot be built here")
    return p


def is_current() -> bool:
    if not (os.path.exists(LIB) and os.path.exists(STAMP)):
        return False
    try:
        return open(STAMP).read().strip() == _digest()
    except OSError:
        return False


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    if not force and is_current():
        return LIB
    nvcc = nvcc_path()
    objs = []
    procs = []
    objdir = os.path.join(LIBDIR, "obj")
    os.makedirs(objdir, exist_ok=True)
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(f"--- {os.path.basename(src)} ---\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed; see output above")
    # export only the extern "C" ab2_* symbols
    # link into a temporary name and move it into place: a failed link must not take the previous library with it
    tmp = LIB + ".tmp"
    cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", tmp] + objs
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        if os.path.exists(tmp):
            os.remove(tmp)
        raise RuntimeError("link failed")
    os.replace(tmp, LIB)
    with open(STAMP, "w") as f:
        f.write(_digest())
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
