"""Builds pvnet_b200/_lib/libpvnet_b200.so in-tree with nvcc for sm_90a (H100).

nvcc cross-compiles without a GPU; the resulting .so (git-ignored) is loaded from the
source tree.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "_lib")
LIB = os.path.join(LIBDIR, "libpvnet_b200.so")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

NVCC_FLAGS = [
    "-std=c++17", "-O3", "-lineinfo",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    "-Xptxas", "-v", "-Xptxas", "-warn-spills",
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
           [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not stale():
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    os.makedirs(LIBDIR, exist_ok=True)
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(LIBDIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [nvcc, *NVCC_FLAGS, "-I", INCLUDE, "-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append(out)
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f"nvcc failed on {src}")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", LIB + ".tmp", *objs, "-ldl"]
    subprocess.check_call(cmd)
    os.replace(LIB + ".tmp", LIB)
    with open(os.path.join(LIBDIR, "build.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
