"""Build libgpbbmm.so in-tree with nvcc for sm_90a (no torch headers involved: pure C ABI).

    python -m gpytorch_b200.build            # incremental
    python -m gpytorch_b200.build --force

The .so lands in gpytorch_b200/lib/ (git-ignored build product).
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "build")
SOURCES = ["api.cu", "pack.cu", "kmv_simt.cu", "kmv_tc.cu", "cg.cu", "pivchol.cu", "slq.cu", "lanczos.cu", "comm.cu", "ski.cu", "sum.cu", "minres.cu", "lowrank.cu", "xgrad.cu", "tasks.cu", "kron.cu", "deriv.cu", "product.cu", "additive.cu", "spectral.cu", "periodic.cu", "compact.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v"]
LIB = os.path.join(LIBDIR, "libgpbbmm.so")


def nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _digest(paths):
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.encode())
        h.update(open(p, "rb").read())
    return h.hexdigest()


def _deps():
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(HERE, "..", "include", "gp_bbmm.h"))
    return hdrs


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    hdr_digest = _digest(_deps())
    cc = nvcc()
    jobs = []
    objs = []
    for src in SOURCES:
        sp = os.path.join(CSRC, src)
        obj = os.path.join(OBJDIR, src.replace(".cu", ".o"))
        stamp = obj + ".sha"
        dg = hashlib.sha256((hdr_digest + _digest([sp]) + " ".join(FLAGS + ARCH)).encode()).hexdigest()
        objs.append(obj)
        if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dg:
            continue
        jobs.append((sp, obj, stamp, dg))

    def run(job):
        sp, obj, stamp, dg = job
        cmd = [cc, *ARCH, *FLAGS, "-c", sp, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {sp}:\n{r.stdout}\n{r.stderr}")
        with open(obj + ".log", "w") as f:
            f.write(r.stdout + r.stderr)
        with open(stamp, "w") as f:
            f.write(dg)
        return r.stderr

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        for out in ex.map(run, jobs):
            if verbose:
                print(out)
    if jobs or force or not os.path.exists(LIB):
        cmd = [cc, *ARCH, "-shared", "-Xcompiler", "-fPIC", "-o", LIB, *objs, "-lcudart", "-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
