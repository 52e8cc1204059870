"""Build liblatte_b200.so (hand-written sm_90a CUDA + C ABI) in-tree with nvcc.

The .so is a build product (git-ignored).  nvcc cross-compiles for sm_90a without a GPU, so this also runs on a
machine without one (`__graft_entry__.build()`).
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(CSRC, "build")
LIB = os.path.join(HERE, "liblatte_b200.so")
SOURCES = ["runtime.cu", "gemm.cu", "attention.cu", "elementwise.cu", "vae.cu", "sampler.cu", "train.cu", "api.cu"]
HEADERS = [os.path.join(CSRC, "common.h"), os.path.join(CSRC, "ptx.cuh"), os.path.join(CSRC, "wgmma.cuh"),
           os.path.join(os.path.dirname(HERE), "include", "latte_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: liblatte_b200.so cannot be built")


def _stale(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force: bool = False, verbose: bool = False) -> str:
    """Compile what is stale and link in place.  Safe under concurrent callers (every torchrun rank imports the package):
    a library newer than all sources is returned untouched; otherwise ONE process builds under a file lock, links to a
    temporary name and renames it into place, so nobody ever dlopens a half-written file."""
    import fcntl
    sources = [os.path.join(CSRC, s) for s in SOURCES]
    if not force and os.path.exists(LIB) and not _stale(LIB, sources + HEADERS):
        return LIB
    os.makedirs(BUILD, exist_ok=True)
    nvcc = _nvcc()

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
        if verbose and r.stderr:
            sys.stderr.write(r.stderr)

    with open(os.path.join(BUILD, ".lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and os.path.exists(LIB) and not _stale(LIB, sources + HEADERS):
                return LIB              # another process built it while we waited
            objs, jobs = [], []
            for sp in sources:
                op = os.path.join(BUILD, os.path.basename(sp).replace(".cu", ".o"))
                objs.append(op)
                if force or _stale(op, [sp] + HEADERS):
                    jobs.append([nvcc, *NVCC_FLAGS, "-c", sp, "-o", op])
            if jobs:
                with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
                    list(ex.map(run, jobs))
            # cudart is linked statically (nvcc default); the driver API is resolved at run time, so the
            # library loads on machines without libcuda (CPU-only build machines)
            tmp = f"{LIB}.tmp.{os.getpid()}"
            run([nvcc, "-shared", "-o", tmp, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC"])
            os.replace(tmp, LIB)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose=True))
