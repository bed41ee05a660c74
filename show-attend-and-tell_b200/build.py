"""Build libsat_b200.so in-tree with nvcc for sm_90a (no GPU needed: nvcc cross-compiles).

    python show-attend-and-tell_b200/build.py [--force] [--verbose]

The library is self-contained (static cudart, no torch/cuBLAS/CUTLASS dependency) and is
loaded by `sat_b200.lib` through ctypes.
"""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libsat_b200.so")
STAMP = os.path.join(HERE, "build", "stamp.txt")
SOURCES = ["sat_api.cu", "sat_linear.cu", "sat_chain.cu", "sat_attention.cu", "sat_rows.cu", "sat_train.cu", "sat_cider.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-O3", "--expt-relaxed-constexpr",
]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _digest():
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for fn in sorted(os.listdir(root)):
            if fn.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(root, fn), "rb") as f:
                    h.update(fn.encode())
                    h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    dig = _digest()
    if not force and os.path.exists(OUT) and os.path.exists(STAMP):
        if open(STAMP).read().strip() == dig:
            return OUT
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    nvcc = _nvcc()
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"---- nvcc failed on {src} ----\n{out}\n")
        elif verbose or "warning" in out:
            sys.stderr.write(out)
    if failed:
        raise RuntimeError("nvcc compilation failed")
    link = [nvcc, "-shared", "-o", OUT, *objs, "-gencode", "arch=compute_90a,code=sm_90a",
            "-Xcompiler", "-fPIC", "-cudart", "static", "-Xlinker", "--exclude-libs,ALL"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    with open(STAMP, "w") as f:
        f.write(dig)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
