"""Training on device-built stream windows, timed on one GPU, and what it buys the cfg-5 stream.

  * windows built per second: ai.train.stream_examples over a cfg-5-size fleet with bystanders (window graph, node and
    edge labels, sequences of 512 class-balanced files), and the window graph alone with and without edge labels;
    the edge-label call itself (nerrf_trace_edge_labels) by CUDA events;
  * one training step (GraphSAGE-T + edge head + BiLSTM through the library's kernels) at fleet-window size;
  * the cfg-5 stream of bench.py (fleet_columns(10400, 40, seed=5), 60-s window, 30-s tick, kill candidates): precision,
    recall and kills with the toy-trained weights bench.py uses next to weights trained on fleet windows (seed 0, with
    bystanders; held-out AUCs on seed-1 windows).
Reports the GPU's name, power limit and max SM clock with the numbers.

    python scripts/stream_train_timing.py [--procs 10400] [--attacked 40] [--windows 8] [--epochs 30] [--out f.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from nerrf_b200 import graph as G, stream  # noqa: E402
from nerrf_b200.ai import train as T  # noqa: E402
from nerrf_b200.ai.models import GraphSAGE_T  # noqa: E402
from nerrf_b200.ai.models.lstm import LSTMScorer  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0)


def synced(fn):
    torch.cuda.synchronize()
    a = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - a


def cfg5(model, scorer, cols, enc, bad):
    sp = stream.StreamingPlanner(model, scorer, window_s=60.0, tick_s=30.0, top_a=4096, n_rollouts=1024, depth=32, iterations=8,
                                 commit_per_search=64, kill_candidates=True, device="cuda")
    _, s = synced(lambda: sp.run(cols))
    planned = set(sp.reverted)
    tp = len(planned & enc)
    return {"precision": tp / max(len(planned), 1), "recall": tp / max(len(enc), 1), "reversions": len(planned),
            "encrypted_files": len(enc), "kills_correct": len(sp.killed & bad), "kills_wrong": len(sp.killed - bad),
            "ransomware_processes": len(bad), "seconds": s}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--procs", type=int, default=10400); ap.add_argument("--attacked", type=int, default=40)
    ap.add_argument("--bystanders", type=int, default=2); ap.add_argument("--windows", type=int, default=8)
    ap.add_argument("--epochs", type=int, default=30); ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"gpu": gpu_info(), "fleet": [a.procs, a.attacked, a.bystanders]}

    ds = stream.DeviceStream(stream.fleet_columns(a.procs, a.attacked, seed=0, bystanders=a.bystanders)[0], "cuda", observable=True)
    T.stream_examples(ds, 2, seed=99)                                  # warm-up: kernels, allocator
    ex, s = synced(lambda: T.stream_examples(ds, a.windows, seed=0))
    res["stream_examples"] = {"windows": a.windows, "windows_per_s": a.windows / s,
                              "mean_nodes": float(np.mean([e["graph"].num_nodes for e in ex])),
                              "mean_edges": float(np.mean([e["graph"].num_edges for e in ex]))}
    wins = [e["window"] for e in ex]
    _, s_off = synced(lambda: [ds.window_graph(lo, hi, 60.0) for lo, hi in wins])
    _, s_on = synced(lambda: [ds.window_graph(lo, hi, 60.0, edge_labels=True) for lo, hi in wins])
    res["window_graph_ms"] = {"without_edge_labels": s_off / len(wins) * 1e3, "with_edge_labels": s_on / len(wins) * 1e3}
    g = max((e["graph"] for e in ex), key=lambda g_: g_.num_edges)
    lo, hi = g.meta["window_ranks"]
    sel = ds.d_order[lo:hi]
    P, F, raw = ds.node_p[sel], ds.node_f[sel], ds.d_raw_slot[sel]
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        G.edge_labels_device(P, F, raw, g.rowptr, g.col, g.num_nodes)
    ts = []
    for _ in range(20):
        ev0.record(); G.edge_labels_device(P, F, raw, g.rowptr, g.col, g.num_nodes); ev1.record(); ev1.synchronize()
        ts.append(ev0.elapsed_time(ev1))
    res["edge_labels_call_ms"] = {"median": float(np.median(ts)), "events": int(hi - lo), "edges": g.num_edges,
                                  "nodes": g.num_nodes}

    # training on fleet windows: one warm-up epoch, then the timed run whose weights are used below
    torch.manual_seed(0)
    fm, fs = GraphSAGE_T(G.F_IN, 128, 2), LSTMScorer()
    T.train(fm, fs, ex[:1], epochs=1, device="cuda", lstm_backward="library", edge_weight=1.0)
    torch.manual_seed(0)
    fm, fs = GraphSAGE_T(G.F_IN, 128, 2), LSTMScorer()
    _, s = synced(lambda: T.train(fm, fs, ex, epochs=a.epochs, lr=3e-3, device="cuda", lstm_backward="library", edge_weight=1.0))
    res["train"] = {"steps": a.epochs * len(ex), "step_ms": s / (a.epochs * len(ex)) * 1e3, "seconds": s}
    held = T.stream_examples(stream.fleet_columns(a.procs, a.attacked, seed=1, bystanders=a.bystanders)[0], 4, seed=1)
    res["held_out_auc"] = T.evaluate(fm, fs, held, device="cuda", edges=True)
    del ex, held, ds, g
    torch.cuda.empty_cache()

    # the cfg-5 stream: toy-trained weights (bench.py's) next to the fleet-trained ones
    torch.manual_seed(0)
    tm, tsc = GraphSAGE_T(G.F_IN, 128, 2), LSTMScorer()
    T.train(tm, tsc, T.toy_set(range(100, 104)), epochs=25, lr=3e-3, device="cuda")
    cols, enc, bad = stream.fleet_columns(10400, 40, seed=5, return_pids=True)
    res["cfg5_toy_trained"] = cfg5(tm.cuda(), tsc.cuda(), cols, enc, bad)
    res["cfg5_fleet_trained"] = cfg5(fm.cuda(), fs.cuda(), cols, enc, bad)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
