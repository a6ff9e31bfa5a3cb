"""Builds libserl_b200.so (all hand-written sm_90a kernels + the C-ABI) in-tree with nvcc.

    python -m serl_b200.build            # incremental
    python -m serl_b200.build --force
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "lib", "obj")
LIB = os.path.join(HERE, "lib", "libserl_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]          # H100 (Hopper): wgmma, TMA, mbarrier
FLAGS = [*ARCH, "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "-I", os.path.join(ROOT, "include"), "-I", CSRC]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stamp(path):
    h = hashlib.sha1()
    for f in sorted(os.listdir(CSRC)) + ["../../include/serl_b200.h"]:
        p = os.path.join(CSRC, f)
        if os.path.isfile(p) and (f.endswith((".cuh", ".h")) or p == path):
            h.update(open(p, "rb").read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    todo, objs = [], []
    for s in sources():
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s[:-3] + ".o")
        st = obj + ".stamp"
        objs.append(obj)
        stamp = _stamp(src)
        if force or not os.path.exists(obj) or not os.path.exists(st) or open(st).read() != stamp:
            todo.append((src, obj, st, stamp))

    def compile_one(item):
        src, obj, st, stamp = item
        tmp = obj + ".tmp.o"                               # every file appears atomically (a repo snapshot may be taken mid-build)
        cmd = [NVCC, *FLAGS, "-c", src, "-o", tmp] + (["-Xptxas", "-v"] if verbose else [])
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr)
        os.replace(tmp, obj)
        open(st + ".tmp", "w").write(stamp)
        os.replace(st + ".tmp", st)
        return src

    if todo:
        with ThreadPoolExecutor(max_workers=min(8, len(todo))) as ex:
            for done in ex.map(compile_one, todo):
                print("compiled", os.path.relpath(done, ROOT))
    if todo or not os.path.exists(LIB):
        r = subprocess.run([NVCC, "-shared", "-o", LIB + ".tmp", *objs, *ARCH],
                           capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
        os.replace(LIB + ".tmp", LIB)
        print("linked", os.path.relpath(LIB, ROOT))
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="-v" in sys.argv)
