"""Compiles oracle/prophet_oracle.c (the plain-C restatement used as checker and CPU baseline)
into oracle/_build/libprophet_oracle.so with gcc.  Test infrastructure only."""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_build")
LIB = os.path.join(OUT, "libprophet_oracle.so")
SRC = os.path.join(HERE, "prophet_oracle.c")
CMD = ["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-fopenmp", "-fno-fast-math", "-o", LIB, SRC, "-lm"]


def _digest() -> str:
    with open(SRC, "rb") as f:
        return hashlib.sha256(f.read() + " ".join(CMD).encode()).hexdigest()


def build(force: bool = False) -> str:
    # a digest stamp, not file times: a copied tree does not keep them in order, and the benchmark must find the
    # library up to date in a tree it may not write to
    stamp = LIB + ".digest"
    digest = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == digest:
        return LIB
    os.makedirs(OUT, exist_ok=True)
    r = subprocess.run(CMD, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("gcc failed building the C oracle")
    with open(stamp, "w") as f:
        f.write(digest)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
