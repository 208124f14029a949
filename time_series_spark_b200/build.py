"""Builds libprophet_b200.so (hand-written sm_90a CUDA + C ABI) in-tree with nvcc.

    python -m time_series_spark_b200.build [--force]

nvcc cross-compiles without a GPU.  The eight seasonality-class translation units
(fit_inst.cu with -DPB200_MASK=0..7), capi.cu, the grouped-lanes kernels (fit_group_inst.cu) and the
seasonality-table class (fit_table.cu) are compiled in parallel, then linked.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
_VARIANT = os.environ.get("PB200_VARIANT", "")          # dev only: A/B builds with PB200_NVCC_EXTRA flags
OBJ = os.path.join(CSRC, "_build", _VARIANT) if _VARIANT else os.path.join(CSRC, "_build")
LIB = os.path.join(HERE, f"libprophet_b200{'_' + _VARIANT if _VARIANT else ''}.so")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]     # H100 (Hopper)
NVCC_FLAGS = [
    *ARCH, "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr",
] + [f for f in os.environ.get("PB200_NVCC_EXTRA", "").split() if f]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def _sources_digest() -> str:
    h = hashlib.sha256()
    for root in (CSRC, INCLUDE):
        for fn in sorted(os.listdir(root)):
            p = os.path.join(root, fn)
            if os.path.isfile(p) and fn.endswith((".cu", ".cuh", ".h")):
                h.update(fn.encode())
                with open(p, "rb") as f:
                    h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    # the stamp lives next to the library, not in _build/: a copy of the tree that leaves the object files behind still
    # finds the library up to date instead of recompiling it
    stamp = LIB + ".digest"
    digest = _sources_digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == digest:
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    nvcc = _nvcc()
    jobs = []
    for m in range(8):
        jobs.append(([nvcc, *NVCC_FLAGS, f"-DPB200_MASK={m}", "-c", os.path.join(CSRC, "fit_inst.cu"),
                      "-o", os.path.join(OBJ, f"fit_inst_{m}.o")]))
    jobs.append([nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, "capi.cu"), "-o", os.path.join(OBJ, "capi.o")])
    jobs.append([nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, "fit_group_inst.cu"), "-o", os.path.join(OBJ, "fit_group_inst.o")])
    jobs.append([nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, "fit_table.cu"), "-o", os.path.join(OBJ, "fit_table.o")])
    if verbose:
        jobs = [j[:1] + ["-Xptxas", "-v"] + j[1:] for j in jobs]

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        return cmd, r

    with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
        for cmd, r in ex.map(run, jobs):
            if verbose or r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
            if r.returncode != 0:
                raise RuntimeError("nvcc failed: " + " ".join(cmd))
    objs = [os.path.join(OBJ, f"fit_inst_{m}.o") for m in range(8)] + [os.path.join(OBJ, "capi.o"),
                                                                      os.path.join(OBJ, "fit_group_inst.o"),
                                                                      os.path.join(OBJ, "fit_table.o")]
    link = [nvcc, "-shared", *ARCH, "-o", LIB, *objs, "-lcudart"]
    r = subprocess.run(link, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    with open(stamp, "w") as f:
        f.write(digest)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
