"""Build the C-ABI library in-tree with nvcc for sm_90a (H100; no torch dependency in the .so).

    python -m nerrf_b200.build            # -> nerrf_b200/csrc/libnerrf_b200.so
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(CSRC, "libnerrf_b200.so")
SOURCES = ["api.cu", "sage.cu", "sage_umma.cu", "sage_bwd.cu", "sage_edge_bwd.cu", "explain.cu", "incident.cu", "taint.cu", "mcts.cu", "lstm.cu", "lstm_bwd.cu", "lstm_umma.cu", "graph.cu", "ingest.cu", "intern_device.cu", "live_stream.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def nvcc_path():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _stale(out, deps):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    nvcc = nvcc_path()
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(HERE, "..", "include", "nerrf_b200.h"))
    objs = []
    procs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(CSRC, s.replace(".cu", ".o"))
        objs.append(obj)
        if force or _stale(obj, [src] + headers):
            cmd = [nvcc, *ARCH, *FLAGS, "-c", src, "-o", obj] + (["-Xptxas", "-v"] if verbose else [])
            procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"--- nvcc failed on {s}\n{out}\n")
        elif verbose or out.strip():
            sys.stderr.write(f"--- {s}\n{out}\n")
    if failed:
        raise RuntimeError("nvcc compilation failed")
    if force or procs or _stale(LIB, objs):
        cmd = [nvcc, *ARCH, "-shared", "-o", LIB, *objs, "-cudart", "static"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
