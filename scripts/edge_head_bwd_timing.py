"""Edge head backward timing on the benchmark graph (1M nodes / 10M edges, hub sources: dist.gpu_synthetic_graph, the
largest source rows have ~10^5 out-edges): `nerrf_sage_edge_head_bwd` against one `nerrf_sage_layer_bwd` at F=128 (the
cost of one GraphSAGE-T layer's backward, for scale).  CUDA events, after warm-up, median of --reps calls each.  Also: the
bytes the edge head backward has to move, from the shapes (dL read twice -- once along the CSR rows, once gathered
through t_eid --, t_eid, the row pointers, h read, dh written), and whether two calls give the same bits.

    python scripts/edge_head_bwd_timing.py [--out DIR] [--reps 20]     # one JSON line -> stdout and DIR/edge_head_bwd_timing.json
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from nerrf_b200 import _lib as L, dist as ND
from nerrf_b200.ai import autograd as AG


def card():
    """Name and power limit, by read-only queries."""
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["nvidia_smi"] = q
    except Exception as e:                   # the timing stands without it; say why it is missing
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def timed(fn, reps):
    """Median ms of fn() over reps runs, each bracketed by CUDA events."""
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out)), [round(x, 3) for x in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="edge_head_bwd_timing_out"); ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--N", type=int, default=1_000_000); ap.add_argument("--E", type=int, default=10_000_000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda")
    N, E, H, F = a.N, a.E, 128, 128
    rowptr, col, ew, _ = ND.gpu_synthetic_graph(N, E, seed=20250115, device=dev)
    tg = AG.TrainGraph(rowptr, col, ew)
    gen = torch.Generator(device=dev).manual_seed(1)
    h = torch.relu(torch.randn(N, H, generator=gen, device=dev))
    We = torch.randn(2 * H, 2, generator=gen, device=dev) * 0.1
    dL = torch.randn(E, 2, generator=gen, device=dev)
    dh, dWe, dbe = torch.empty_like(h), torch.empty(2 * H, 2, device=dev), torch.empty(2, device=dev)
    lib = L.lib()
    s = L.current_stream_ptr()
    ws = tg.edge_workspace(H)
    is64 = int(tg.rowptr.dtype == torch.int64)
    edge = lambda: L.check(lib.nerrf_sage_edge_head_bwd(L.ptr(h), L.ptr(We), L.ptr(dL), L.ptr(tg.rowptr), is64,
                                                        L.ptr(tg.t_rowptr), L.ptr(tg.t_eid), is64, L.ptr(dh), L.ptr(dWe),
                                                        L.ptr(dbe), L.ptr(ws), ws.numel() * 4, N, H, s),
                           "nerrf_sage_edge_head_bwd")
    # one layer backward at F=128 (input, aggregate, output, upstream gradient; all gradients)
    x = torch.relu(torch.randn(N, F, generator=gen, device=dev))
    W = torch.randn(2 * F, H, generator=gen, device=dev) * 0.05
    m = AG.aggregate(x, tg)
    y = torch.relu(torch.cat([x, m], 1) @ W)
    dy = torch.randn(N, H, generator=gen, device=dev)
    ldh, ldW, ldb = torch.empty_like(x), torch.empty_like(W), torch.empty(H, device=dev)
    lws = tg.workspace(F)
    layer = lambda: L.check(lib.nerrf_sage_layer_bwd(L.ptr(x), L.ptr(m), L.ptr(y), L.ptr(dy), L.ptr(W), L.ptr(tg.t_rowptr),
                                                     is64, L.ptr(tg.t_col), L.ptr(tg.t_w), L.ptr(ldh), L.ptr(ldW),
                                                     L.ptr(ldb), L.ptr(lws), lws.numel() * 4, N, F, H, 1, s),
                            "nerrf_sage_layer_bwd")
    for _ in range(3):                                                 # warm-up
        edge(); layer()
    torch.cuda.synchronize()
    first = (dh.clone(), dWe.clone(), dbe.clone())
    edge_ms, edge_all = timed(edge, a.reps)
    layer_ms, layer_all = timed(layer, a.reps)
    edge_ms2, _ = timed(edge, a.reps)                                  # again, after the layer: the spread of the two runs
    same_bits = bool(torch.equal(first[0], dh) and torch.equal(first[1], dWe) and torch.equal(first[2], dbe))
    ib = tg.rowptr.element_size()
    out_deg = torch.diff(tg.t_rowptr.long())
    bytes_moved = (2 * E * 2 * 4 + E * tg.t_eid.element_size() + 2 * (N + 1) * ib + N * H * 4 + N * H * 4
                   + N * 16 * 2)                                     # + g [N,4] written and read back by the dW pass
    res = {"script": "edge_head_bwd_timing", "card": card(), "nodes": N, "edges": E, "H": H,
           "graph": "dist.gpu_synthetic_graph hub_src (dst uniform, src = floor(N u^3))",
           "max_out_degree": int(out_deg.max()), "max_in_degree": int(torch.diff(tg.rowptr.long()).max()),
           "reps": a.reps, "edge_head_bwd_ms": round(edge_ms, 4), "edge_head_bwd_ms_repeat": round(edge_ms2, 4),
           "layer_bwd_f128_ms": round(layer_ms, 4), "edge_over_layer": round(edge_ms / layer_ms, 4),
           "edge_head_bwd_bytes": int(bytes_moved), "edge_head_bwd_GBps": round(bytes_moved / edge_ms * 1e-6, 1),
           "samples_ms": {"edge_head_bwd": edge_all, "layer_bwd": layer_all}, "bitwise_repeatable": same_bits}
    line = json.dumps(res)
    print(line)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "edge_head_bwd_timing.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
