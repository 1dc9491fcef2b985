"""ctypes wrapper of the C restatement of the spec-v2 planner oracle (oracle/c/restore_oracle.c) -- TEST INFRASTRUCTURE.

Built on demand with gcc into oracle/_build/ (git-ignored).  Pins oracle/restore_ref.py bit for bit against a second,
independent implementation.  Never imported by the product (nerrf_b200/)."""
import ctypes as C
import os
import subprocess

import numpy as np

from . import rewards_ref as RW
from . import restore_ref as V2
from .mcts_ref import ln_table, best_child

_HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(_HERE, "c", "restore_oracle.c")
OUT_DIR = os.path.join(_HERE, "_build")
LIB = os.path.join(OUT_DIR, "librestore_oracle.so")
_lib = None


def build(force=False):
    os.makedirs(OUT_DIR, exist_ok=True)
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(SRC):
        cmd = ["gcc", "-O2", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", SRC, "-o", LIB, "-lm"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("gcc failed on the spec-v2 C oracle:\n" + r.stdout + r.stderr)
    return LIB


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _i32(a):
    return None if a is None else np.ascontiguousarray(a, np.int32)


def score(states, p, size, cost, guard=None, cover=None):
    p = np.ascontiguousarray(p, np.float32); size = np.ascontiguousarray(size, np.float32); cost = np.ascontiguousarray(cost, np.float32)
    A = p.shape[0]
    V2.check_cover(cover, guard, A)
    st = np.ascontiguousarray(states, np.uint32).reshape(-1, RW.layout(A)[3])
    out = np.zeros(st.shape[0], np.float32)
    g, cv = _i32(guard), _i32(cover)
    lib().nerrf_oracle_v2_score(_p(st), C.c_int64(st.shape[0]), _p(p), _p(size), _p(cost), _p(g), _p(cv), C.c_int(A), _p(out))
    return out


def search(p, size, cost, R=4096, D=50, T=64, seed=0, c=np.sqrt(2.0), root_state=None, guard=None, cover=None):
    p = np.ascontiguousarray(p, np.float32); size = np.ascontiguousarray(size, np.float32); cost = np.ascontiguousarray(cost, np.float32)
    A = p.shape[0]
    _, _, A_pad, _ = RW.layout(A)
    root = RW.empty_state(A) if root_state is None else (np.asarray(root_state, np.uint32) | RW.empty_state(A))
    root = np.ascontiguousarray(root, np.uint32)
    lo, inv = V2.reward_bounds(p, size, cost, root, guard, cover)
    g, cv = _i32(guard), _i32(cover)
    lnN = ln_table(T, R)
    root_n = np.zeros(A_pad, np.int32); root_w = np.zeros(A_pad, np.float32); nn = np.zeros(1, np.int32)
    lib().nerrf_oracle_v2_mcts(_p(p), _p(size), _p(cost), _p(g), _p(cv), C.c_int(A), _p(root), C.c_int(R), C.c_int(D), C.c_int(T),
                               C.c_uint64(seed), C.c_float(np.float32(c)), C.c_float(lo), C.c_float(inv), _p(lnN), _p(root_n),
                               _p(root_w), _p(nn))
    return {"root_n": root_n[:A].copy(), "root_w": root_w[:A].copy(), "best": best_child(root_n[:A], root_w[:A]),
            "num_nodes": int(nn[0]), "lo": lo, "inv_range": inv}
