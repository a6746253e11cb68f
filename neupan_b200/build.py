"""Builds libneupan_b200.so in-tree with nvcc for sm_90a (H100; no torch involved).

    python -m neupan_b200.build [--force] [-v]

Each translation unit of UNITS compiles to its own object, in parallel.  The .so lands in neupan_b200/lib/ (git-ignored).
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "build")
LIB = os.path.join(LIBDIR, "libneupan_b200.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC"]
UNITS = ["nrmp.cu", "dune_tc.cu", "pan_api.cu", "world_api.cu", "aux_api.cu"]  # translation units under csrc/, linked in this order


def obj_path(unit: str) -> str:
    return os.path.join(OBJDIR, os.path.splitext(unit)[0] + ".o")


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _sources_digest() -> str:
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for name in sorted(os.listdir(root)):
            if name.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(root, name), "rb") as f:
                    h.update(name.encode()); h.update(f.read())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, "build.stamp")
    digest = _sources_digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == digest:
        return LIB
    nvcc = _nvcc()
    extra = ["-Xptxas", "-v"] if verbose else []
    jobs = [([nvcc, *ARCH, *COMMON, *extra, "-c", os.path.join(CSRC, u), "-o", obj_path(u)], u) for u in UNITS]

    def run(job):
        cmd, what = job
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {what}:\n{r.stdout}\n{r.stderr}")
        return what, r.stderr

    with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
        for what, log in ex.map(run, jobs):
            if verbose:
                print(f"--- {what}\n{log}")
    r = subprocess.run([nvcc, *ARCH, "-shared", "-o", LIB, *map(obj_path, UNITS)], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(digest)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
