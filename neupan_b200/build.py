"""Builds libneupan_b200.so in-tree with nvcc for sm_90a (H100; no torch involved).

    python -m neupan_b200.build            # all edge counts 3..8
    NB_EDGE_DIMS=4 python -m neupan_b200.build   # quick developer build

The DUNE kernel is instantiated once per polygon edge count E; each instantiation is its own
translation unit so they compile in parallel.  The .so lands in neupan_b200/lib/ (git-ignored).
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


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _sources_digest(edge_dims) -> str:
    h = hashlib.sha256(repr(sorted(edge_dims)).encode())
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for name in sorted(os.listdir(root)):
            if name.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(root, name), "rb") as f:
                    h.update(name.encode()); h.update(f.read())
    return h.hexdigest()


def build(edge_dims=None, force: bool = False, verbose: bool = False) -> str:
    if edge_dims is None:
        env = os.environ.get("NB_EDGE_DIMS", "3,4,5,6,7,8")
        edge_dims = [int(x) for x in env.split(",") if x]
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, "build.stamp")
    digest = _sources_digest(edge_dims)
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == digest:
        return LIB
    nvcc = _nvcc()
    mask = sum(1 << e for e in edge_dims)
    extra = ["-Xptxas", "-v"] if verbose else []
    jobs = [([nvcc, *ARCH, *COMMON, *extra, f"-DNB_E={e}", "-c", os.path.join(CSRC, "dune_inst.cu"), "-o", os.path.join(OBJDIR, f"dune_e{e}.o")], f"dune E={e}")
            for e in edge_dims]
    jobs.append(([nvcc, *ARCH, *COMMON, *extra, "-c", os.path.join(CSRC, "dune_mma.cu"), "-o", os.path.join(OBJDIR, "dune_mma.o")], "dune_mma"))
    jobs.append(([nvcc, *ARCH, *COMMON, *extra, "-c", os.path.join(CSRC, "dune_tc.cu"), "-o", os.path.join(OBJDIR, "dune_tc.o")], "dune_tc"))
    jobs.append(([nvcc, *ARCH, *COMMON, *extra, f"-DNB_EDGE_MASK={mask}", "-c", os.path.join(CSRC, "pan_api.cu"), "-o", os.path.join(OBJDIR, "pan_api.o")], "pan_api"))

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
    objs = [os.path.join(OBJDIR, f"dune_e{e}.o") for e in edge_dims] + [os.path.join(OBJDIR, "dune_mma.o"), os.path.join(OBJDIR, "dune_tc.o"), os.path.join(OBJDIR, "pan_api.o")]
    r = subprocess.run([nvcc, *ARCH, "-shared", "-o", LIB, *objs], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(digest)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
