"""The C-ABI library builds, loads, and exports every symbol include/nerrf_b200.h declares.
No compute calls here (CPU box)."""
import ctypes
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "nerrf_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(nerrf_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_the_path():
    syms = _declared_symbols()
    for want in ("nerrf_sage_layer_fwd", "nerrf_sage_forward", "nerrf_lstm_forward", "nerrf_mcts_search",
                 "nerrf_reward_score", "nerrf_last_error", "nerrf_sage_session_forward_host"):
        assert want in syms


def test_library_exports_every_declared_symbol(lib_built):
    h = ctypes.CDLL(lib_built)
    for s in _declared_symbols():
        assert hasattr(h, s), f"libnerrf_b200.so does not export {s}"
    assert h.nerrf_abi_version() == 2


def test_python_binding_covers_header(lib_built):
    from nerrf_b200 import _lib
    assert sorted(_lib.SIGNATURES) == _declared_symbols()
    _lib.lib()          # loads and type-annotates every entry point


def test_invalid_arguments_return_error_not_crash(lib_built):
    from nerrf_b200 import _lib
    h = _lib.lib()
    n = ctypes.c_size_t()
    assert h.nerrf_mcts_workspace_bytes(0, 4, 64, ctypes.byref(n)) == -1
    assert b"1..4096" in h.nerrf_last_error()
    assert h.nerrf_mcts_workspace_bytes(10, 4, 48, ctypes.byref(n)) == -1      # R not a power of two
    assert h.nerrf_mcts_workspace_bytes(10, 4, 64, ctypes.byref(n)) == 0 and n.value > 0
    assert h.nerrf_lstm_workspace_bytes(4, 100, 128, ctypes.byref(n)) == -1     # H != 256
    # the layer reads node_w 8 bytes at a time: a misaligned head vector is refused before anything is touched
    p = lambda a: ctypes.c_void_p(a)
    args = [p(1 << 20), p(2 << 20), 0, p(3 << 20), p(4 << 20), p(5 << 20), p(6 << 20), p(7 << 20), 10, 0, 10, 32, 128, 1, 0]
    assert h.nerrf_sage_layer_head_fwd(*args, p((8 << 20) + 4), 0.0, p(9 << 20), None) == -1
    assert b"node_w" in h.nerrf_last_error()


def test_product_never_imports_oracle():
    bad = []
    for d, _, files in os.walk(os.path.join(ROOT, "nerrf_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(d, f)).read()
                if re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M) or "from .. import oracle" in src:
                    bad.append(os.path.join(d, f))
    for d, _, files in os.walk(os.path.join(ROOT, "ai")):
        for f in files:
            if f.endswith(".py") and re.search(r"\boracle\b", open(os.path.join(d, f)).read()):
                bad.append(os.path.join(d, f))
    assert not bad, bad


def test_missing_library_fails_loudly(tmp_path):
    code = ("import nerrf_b200._lib as L; L.LIB_PATH = r'%s/nope.so'\n"
            "try:\n    L.lib()\nexcept L.NerrfError as e:\n    print('LOUD', e)\n" % tmp_path)
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert "LOUD" in out.stdout and "no cpu fallback" in out.stdout.lower()


def test_cpu_tensors_are_rejected(lib_built):
    import torch
    from nerrf_b200.ai.models import GraphSAGE_T
    from nerrf_b200._lib import NerrfError
    m = GraphSAGE_T(32, 128, 2)
    x = torch.zeros(4, 32); rp = torch.zeros(5, dtype=torch.int32)
    col = torch.zeros(0, dtype=torch.int32); ew = torch.zeros(0)
    with pytest.raises(NerrfError):
        m(x, rp, col, ew)


def test_reference_named_surface_imports():
    import ai.models, ai.planner                          # noqa: E401
    from ai.models import GraphSAGE_T, lstm               # noqa: F401
    from ai.planner import mcts, rewards
    assert callable(mcts.search) and callable(rewards.score) and callable(lstm.forward)
    assert hasattr(GraphSAGE_T, "forward")


def test_header_is_plain_c99(tmp_path, lib_built):
    """The boundary is a C ABI: the header must compile as C (no C++-isms), and a C program must link against the
    library with nothing but -lnerrf_b200 (static cudart inside)."""
    src = tmp_path / "use.c"
    src.write_text('#include "nerrf_b200.h"\n#include <stdio.h>\n'
                   'int main(void) { printf("%d %s\\n", nerrf_abi_version(), nerrf_last_error()); return 0; }\n')
    inc = os.path.join(ROOT, "include")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-I", inc, str(src)], check=True)
    exe = tmp_path / "use"
    libdir = os.path.dirname(lib_built)
    subprocess.run(["gcc", "-std=c99", "-I", inc, str(src), "-o", str(exe), "-L", libdir, "-lnerrf_b200",
                    "-Wl,-rpath," + libdir], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert out[0] == "2"
