"""In-tree build of the sm_90a kernel library (plain nvcc, C ABI, loaded with ctypes).

``python -m torchrec_b200.ops.build`` (or ``__graft_entry__.build()``) compiles every ``csrc/*.cu``
with ``-gencode arch=compute_90a,code=sm_90a -lineinfo`` into ``torchrec_b200/ops/_lib/``.
Objects are rebuilt only when a source or header is newer; objects, compiler logs and the shared
object are build products (git-ignored).
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import shutil
import subprocess
import sys
from typing import List

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "_lib")
LIB_NAME = "libtrb200_ops.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; the torchrec_b200 kernel library needs the CUDA toolkit to build")


def _sources() -> List[str]:
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers_mtime() -> float:
    m = 0.0
    for f in os.listdir(CSRC):
        if f.endswith((".cuh", ".h", ".hpp")):
            m = max(m, os.path.getmtime(os.path.join(CSRC, f)))
    return m


def _compile_one(src: str, obj: str, verbose: bool) -> str:
    cmd = [_nvcc(), *NVCC_FLAGS, "-I", CSRC, "-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log = obj + ".log"
    with open(log, "w") as f:
        f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    if verbose:
        print(f"[trb200 build] {os.path.basename(src)} ok")
    return obj


def lib_path() -> str:
    return os.path.join(OUT, LIB_NAME)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OUT, exist_ok=True)
    srcs = _sources()
    hm = _headers_mtime()
    todo = []
    objs = []
    for s in srcs:
        o = os.path.join(OUT, os.path.basename(s)[:-3] + ".o")
        objs.append(o)
        if force or not os.path.exists(o) or os.path.getmtime(o) < max(os.path.getmtime(s), hm):
            todo.append((s, o))
    if todo:
        with cf.ThreadPoolExecutor(max_workers=min(8, len(todo))) as ex:
            list(ex.map(lambda so: _compile_one(so[0], so[1], verbose), todo))
    lib = lib_path()
    if todo or not os.path.exists(lib) or any(os.path.getmtime(o) > os.path.getmtime(lib) for o in objs):
        cmd = [_nvcc(), "-shared", "-o", lib + ".tmp", *objs, "-gencode", "arch=compute_90a,code=sm_90a",
               "-Xcompiler", "-fPIC"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
        os.replace(lib + ".tmp", lib)
        if verbose:
            print(f"[trb200 build] linked {lib}")
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
