"""Builds libb200kge.so (sm_90a) in-tree with nvcc.  No torch headers, no CPU fallback."""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200kge.so")
SOURCES = ["capi.cu", "fold.cu", "pairwise_simt.cu", "pairwise_tc.cu", "presplit.cu", "rowwise.cu", "epilogue_dense.cu", "hostindex.cu", "grad.cu", "grad_distance.cu", "csr_loss.cu", "ns_loss.cu", "dropout.cu", "ns_dropout.cu", "rowset.cu", "optim.cu", "ns_p.cu", "ns_shared.cu"]
HEADERS = ["common.cuh", "dropmask.cuh", "fold.cuh", "philox.cuh", "ptx.cuh", "tc_common.cuh", os.path.join("..", "..", "include", "b200kge.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; cannot build libb200kge.so")


def _digest() -> str:
    h = hashlib.sha256()
    for f in SOURCES + HEADERS:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build_native(force: bool = False, verbose: bool = False) -> str:
    stamp = LIB + ".stamp"
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    procs = []
    objs = []
    for s in SOURCES:
        o = os.path.join(objdir, s.replace(".cu", ".o"))
        objs.append(o)
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, s), "-o", o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"--- nvcc {s} failed ---\n{out}\n")
        elif verbose and out.strip():
            print(f"--- nvcc {s} ---\n{out}")
    if failed:
        raise RuntimeError("nvcc failed building libb200kge.so")
    cmd = [nvcc, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed for libb200kge.so")
    with open(stamp, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    print(build_native(force="--force" in sys.argv, verbose=True))
