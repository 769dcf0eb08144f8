"""Build libquimb_b200.so in-tree with nvcc for sm_90a (H100).

Usage: python -m quimb_b200.csrc.build [--force] [--verbose]
The shared object lands next to the sources (git-ignored build product).
"""

import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
import glob

# every translation unit and every header next to this file is part of the
# build (and of the rebuild digest: a stale .so after a header edit would be a
# silent ABI mismatch between objects on the GPU box)
SOURCES = sorted(os.path.basename(p) for p in glob.glob(os.path.join(HERE, "*.cu")))
HEADERS = sorted(os.path.basename(p) for p in glob.glob(os.path.join(HERE, "*.h"))
                 + glob.glob(os.path.join(HERE, "*.cuh"))) + ["../../include/quimb_b200.h"]
LIB = os.path.join(HERE, "libquimb_b200.so")
STAMP = os.path.join(HERE, ".build_stamp")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]

NVCC_FLAGS = [
    *ARCH,
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "-cudart", "static",
]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libquimb_b200.so")


def _digest(sources):
    h = hashlib.sha256()
    for f in sources + HEADERS:
        p = os.path.join(HERE, f)
        if os.path.exists(p):
            with open(p, "rb") as fh:
                h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    sources = [s for s in SOURCES if os.path.exists(os.path.join(HERE, s))]
    dig = _digest(sources)
    if not force and os.path.exists(LIB) and os.path.exists(STAMP):
        with open(STAMP) as fh:
            if fh.read().strip() == dig:
                return LIB
    nvcc = _nvcc()
    objs = []
    procs = []
    for s in sources:
        obj = os.path.join(HERE, s.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(HERE, s), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas")
            cmd.insert(2, "-v")
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE,
                                          stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for s, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0:
            failed = True
            sys.stderr.write(f"[quimb_b200.build] {s} failed:\n{out}\n")
        elif verbose or out.strip():
            sys.stderr.write(f"[quimb_b200.build] {s}:\n{out}\n")
    if failed:
        raise RuntimeError("nvcc compilation failed")
    # link next to the target and rename: the library is replaced atomically
    # (a snapshot of the tree never sees a half-written .so)
    tmp = LIB + ".tmp"
    cmd = [nvcc, "-shared", *ARCH, "-cudart", "static", "-o", tmp, *objs]
    subprocess.run(cmd, check=True)
    os.replace(tmp, LIB)
    with open(STAMP, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(LIB)
