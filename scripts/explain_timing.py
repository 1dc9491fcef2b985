"""Time the explanation of a cfg-5-size plan, stage by stage (DESIGN.md 1.1.1 / 6).

    python scripts/explain_timing.py [--procs 10400] [--attacked 40] [--k 8] [--reps 5] [--out f.json]

The cfg-5 fleet trace of bench.py (fleet_columns(procs, attacked, seed=5)), toy-trained weights as bench.py trains them.
A StreamingPlanner run (kill candidates, explain=0) gives the ticks; every tick's window graph is rebuilt, planned once
(pipeline.run, kill candidates) and its planned nodes explained: extraction (nerrf_explain_subgraph_count / _fill),
forward (the fused layers), backward (nerrf_sage_layer_bwd_ex), top-k (nerrf_explain_topk), event gather
(explain.attach_events).  Each stage ends in a device synchronise; per tick the median of --reps timed runs after one
warm-up.  Printed beside the tick's own graphsage_t + lstm + mcts_plan time, with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nerrf_b200 import explain as EX, graph as G, pipeline, stream  # noqa: E402
from nerrf_b200.ai import train as T  # noqa: E402
from nerrf_b200.ai.models import GraphSAGE_T  # noqa: E402
from nerrf_b200.ai.models.lstm import LSTMScorer  # noqa: E402


def stages(gd, g, model, nodes, k):
    sync = torch.cuda.synchronize
    tm = {}
    a = time.perf_counter()
    sg = EX.subgraphs(gd.rowptr, gd.col, gd.ew, gd.x, nodes, model.num_layers)
    sync(); tm["extract"] = (time.perf_counter() - a) * 1e3
    a = time.perf_counter()
    hs = EX.forward_saved(model, sg["x"], sg["rowptr"], sg["col"], sg["ew"])
    sync(); tm["forward"] = (time.perf_counter() - a) * 1e3
    a = time.perf_counter()
    d = EX.edge_weight_grad(model, hs, sg["rowptr"], sg["col"], sg["ew"], sg["target"].long())
    sync(); tm["backward"] = (time.perf_counter() - a) * 1e3
    a = time.perf_counter()
    _, oa, op, ov = EX.topk(sg["seg"], sg["ew"], d, sg["epos"], EX._edge_event(g, gd.x.device), k)
    sync(); tm["topk"] = (time.perf_counter() - a) * 1e3
    a = time.perf_counter()
    fit = np.nonzero(sg["fit"])[0]
    logits = hs[-1][sg["target"].long()] @ model.node_w.detach() + model.node_b.detach()
    res = EX._results(np.asarray(nodes)[fit], "subgraph", logits, oa, op, ov, gd.rowptr, gd.col)
    EX.attach_events(g, res)
    sync(); tm["event_gather"] = (time.perf_counter() - a) * 1e3
    tm["explain_total"] = sum(tm.values())
    return tm, int(sg["fit"].sum()), int(sg["seg"][-1]), int((~sg["fit"]).sum())


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--procs", type=int, default=10400); ap.add_argument("--attacked", type=int, default=40)
    ap.add_argument("--k", type=int, default=8); ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("explain_timing needs a CUDA device")
    dev = torch.device("cuda")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    torch.manual_seed(0)
    model, scorer = GraphSAGE_T(G.F_IN, 128, 2), LSTMScorer()
    T.train(model, scorer, T.toy_set(range(100, 104)), epochs=25, lr=3e-3, device=dev)
    model.to(dev); scorer.to(dev)
    cols, _ = stream.fleet_columns(a.procs, a.attacked, seed=5)
    sp = stream.StreamingPlanner(model, scorer, window_s=60.0, tick_s=30.0, top_a=4096, n_rollouts=1024, depth=32, iterations=8,
                                 commit_per_search=64, kill_candidates=True)
    ticks = sp.run(cols)
    ds = stream.DeviceStream(cols, "cuda", observable=True)
    t0 = ds.span()[0]
    rows = []
    for t in ticks:
        t_hi = t0 + t.t_hi
        g = ds.window_graph(t_hi - 60.0, t_hi, 60.0)
        kind = np.asarray(g.meta["node_kind"])
        files = np.nonzero(kind == 0)[0]
        seq = lambda cand, g=g: (*ds.sequences_device(g, cand), None)
        res = pipeline.run(g, seq, None, files, model, scorer, top_a=4096, n_rollouts=1024, depth=32, iterations=8,
                           commit_per_search=64, kill_candidates=True)
        nodes = list(dict.fromkeys(res.plan_nodes))
        if not nodes:
            continue
        gd = G.TemporalGraph(g.rowptr, g.col, g.ew, g.x, g.meta)
        stages(gd, g, model, nodes, a.k)                          # warm-up
        runs = [stages(gd, g, model, nodes, a.k) for _ in range(a.reps)]
        med = {key: float(np.median([r[0][key] for r in runs])) for key in runs[0][0]}
        tick_ms = sum(float(res.timings_ms.get(key, 0.0)) for key in ("graphsage_t", "lstm", "mcts_plan"))
        rows.append({"t_hi": t.t_hi, "nodes": g.num_nodes, "edges": g.num_edges, "steps": len(nodes),
                     "explained_subgraph": runs[0][1], "batched_edges": runs[0][2], "over_budget": runs[0][3],
                     "stages_ms": med, "tick_sage_lstm_mcts_ms": tick_ms})
        print(json.dumps(rows[-1]), flush=True)
    tot = {key: sum(r["stages_ms"][key] for r in rows) for key in rows[0]["stages_ms"]} if rows else {}
    out = {"gpu": gpu, "procs": a.procs, "attacked": a.attacked, "k": a.k, "ticks": rows,
           "steps": sum(r["steps"] for r in rows), "explain_ms": tot,
           "tick_sage_lstm_mcts_ms": sum(r["tick_sage_lstm_mcts_ms"] for r in rows)}
    print(json.dumps({k: v for k, v in out.items() if k != "ticks"}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
