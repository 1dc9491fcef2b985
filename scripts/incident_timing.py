"""Time the incident grouping of cfg-5 ticks, stage by stage (DESIGN.md 1.4 / 6).

    python scripts/incident_timing.py [--procs 10400] [--attacked 40] [--reps 5] [--out f.json]

The cfg-5 fleet trace of bench.py (fleet_columns(procs, attacked, seed=5)), toy-trained weights as bench.py trains them.
Every tick's window graph (window 60 s, tick 30 s) is planned once (pipeline.run, kill candidates) and its incidents
computed with the plan's file steps as seeds: flag + owner pass (nerrf_incident_files), group (nerrf_incident_group),
host records (incident.records: names and events).  Each stage ends in a device synchronise; per tick the median of
--reps timed runs after one warm-up.  Printed beside the tick's own graphsage_t + lstm + mcts_plan time, with the
card's name and power limit read in the same run.
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

from nerrf_b200 import graph as G, incident as I, pipeline, stream  # noqa: E402
from nerrf_b200.ai import train as T  # noqa: E402
from nerrf_b200.ai.models import GraphSAGE_T  # noqa: E402
from nerrf_b200.ai.models.lstm import LSTMScorer  # noqa: E402


def stages(g, score, seeds, tau=0.5):
    sync = torch.cuda.synchronize
    dev = g.rowptr.device
    tm = {}
    a = time.perf_counter()
    kind = torch.from_numpy(np.asarray(g.meta["node_kind"]).astype(np.int8)).to(dev)
    et, ev = g.meta["edge_time"](), g.meta["edge_event"]()
    files, fi, fr = I.flag_files(g.rowptr, g.col, kind, score, tau, seeds, None, et, ev)
    sync(); tm["flag_owner"] = (time.perf_counter() - a) * 1e3
    a = time.perf_counter()
    src = torch.from_numpy(np.asarray(g.meta["node_source"], np.int64).astype(np.int32)).to(dev)
    size = torch.from_numpy(np.asarray(g.meta["size_mb"], np.float32)).to(dev)
    ii, ir, grouped, fin = I.group_files(files, fi, fr, src, size, score)
    sync(); tm["group"] = (time.perf_counter() - a) * 1e3
    a = time.perf_counter()
    h = lambda t: t.cpu().numpy()
    recs = I.records(g, h(files), h(fi), h(fr), h(ii), h(ir), h(grouped), h(fin), None, True)[0]
    tm["host_records"] = (time.perf_counter() - a) * 1e3
    tm["incidents_total"] = sum(tm.values())
    return tm, int(files.numel()), len(recs)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--procs", type=int, default=10400); ap.add_argument("--attacked", type=int, default=40)
    ap.add_argument("--reps", type=int, default=5); ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("incident_timing needs a CUDA device")
    dev = torch.device("cuda")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    torch.manual_seed(0)
    model, scorer = GraphSAGE_T(G.F_IN, 128, 2), LSTMScorer()
    T.train(model, scorer, T.toy_set(range(100, 104)), epochs=25, lr=3e-3, device=dev)
    model.to(dev); scorer.to(dev)
    cols, _ = stream.fleet_columns(a.procs, a.attacked, seed=5)
    ds = stream.DeviceStream(cols, "cuda", observable=True)
    t0, t1 = ds.span()
    rows, t_hi = [], t0
    while t_hi < t1:
        t_hi = min(t_hi + 30.0, t1)
        g = ds.window_graph(t_hi - 60.0, t_hi, 60.0)
        if g is None:
            continue
        kind = np.asarray(g.meta["node_kind"])
        files = np.nonzero(kind == 0)[0]
        seq = lambda cand, g=g: (*ds.sequences_device(g, cand), None)
        res = pipeline.run(g, seq, None, files, model, scorer, top_a=4096, n_rollouts=1024, depth=32, iterations=8,
                           commit_per_search=64, kill_candidates=True)
        seeds = np.asarray([n for n in res.plan_nodes if kind[n] == 0], np.int64)
        stages(g, res.node_score, seeds)                           # warm-up
        runs = [stages(g, res.node_score, seeds) for _ in range(a.reps)]
        med = {key: float(np.median([r[0][key] for r in runs])) for key in runs[0][0]}
        tick_ms = sum(float(res.timings_ms.get(key, 0.0)) for key in ("graphsage_t", "lstm", "mcts_plan"))
        rows.append({"t_hi": t_hi - t0, "nodes": g.num_nodes, "edges": g.num_edges, "file_steps": int(seeds.size),
                     "flagged": runs[0][1], "incidents": runs[0][2], "stages_ms": med, "tick_sage_lstm_mcts_ms": tick_ms})
        print(json.dumps(rows[-1]), flush=True)
    tot = {key: sum(r["stages_ms"][key] for r in rows) for key in rows[0]["stages_ms"]} if rows else {}
    out = {"gpu": gpu, "procs": a.procs, "attacked": a.attacked, "ticks": rows, "incident_ms": tot,
           "tick_sage_lstm_mcts_ms": sum(r["tick_sage_lstm_mcts_ms"] for r in rows)}
    print(json.dumps({k: v for k, v in out.items() if k != "ticks"}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
