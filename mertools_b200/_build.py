"""Build libmer_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

Called by ``__graft_entry__.build()`` and by ``python -m mertools_b200._build``.  The shared
library lands in ``mertools_b200/lib/`` (git-ignored: build() recreates it).
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "build")
LIB = os.path.join(LIBDIR, "libmer_b200.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr",
    "-DMER_BUILD=1",
]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(path, deps):
    h = hashlib.sha256()
    h.update(" ".join(FLAGS).encode())
    for p in [path] + deps:
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _compile(src, verbose):
    path = os.path.join(CSRC, src)
    obj = os.path.join(OBJDIR, src[:-3] + ".o")
    deps = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cuh", ".h"))]
    deps.append(os.path.join(HERE, "..", "include", "mer_b200.h"))
    stamp = obj + ".sha"
    dig = _digest(path, deps)
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
        return obj, ""
    cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", path, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(dig)
    return obj, r.stderr


def build(verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    srcs = _sources()
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile(s, verbose), srcs))
    objs = [o for o, _ in results]
    if verbose:
        for _, log in results:
            if log:
                print(log)
    newest = max(os.path.getmtime(o) for o in objs)
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < newest:
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a",
                                                     "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv))
