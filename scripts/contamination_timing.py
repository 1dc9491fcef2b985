"""Time the contamination closure of cfg-5 ticks with bystanders, stage by stage (DESIGN.md 1.5 / 2.9).

    python scripts/contamination_timing.py [--procs 10400] [--attacked 40] [--bystanders 2] [--reps 5] [--out f.json]

The cfg-5 fleet trace of bench.py (fleet_columns(procs, attacked, seed=5)) with `bystanders` benign processes per
attacked process, toy-trained weights as bench.py trains them.  Every tick's window graph (window 60 s, tick 30 s) is
planned once with incidents (pipeline.run(incidents=True), kill candidates), then its contamination is computed from
those incidents (taint.contamination): the flow-class gather, phase 1 (with its rounds), phase 2 (with its levels),
compaction and host records.  Each stage ends in a device synchronise; per tick the median of --reps timed runs after
one warm-up.  Printed beside the tick's own incident stage, with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nerrf_b200 import graph as G, pipeline, stream, taint  # noqa: E402
from nerrf_b200.ai import train as T  # noqa: E402
from nerrf_b200.ai.models import GraphSAGE_T  # noqa: E402
from nerrf_b200.ai.models.lstm import LSTMScorer  # noqa: E402

STAGES = ("flow_gather", "validate", "phase1", "phase2", "compact", "records")


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--procs", type=int, default=10400); ap.add_argument("--attacked", type=int, default=40)
    ap.add_argument("--bystanders", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5); ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("contamination_timing needs a CUDA device")
    dev = torch.device("cuda")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    torch.manual_seed(0)
    model, scorer = GraphSAGE_T(G.F_IN, 128, 2), LSTMScorer()
    T.train(model, scorer, T.toy_set(range(100, 104)), epochs=25, lr=3e-3, device=dev)
    model.to(dev); scorer.to(dev)
    cols, _ = stream.fleet_columns(a.procs, a.attacked, seed=5, bystanders=a.bystanders)
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
                           commit_per_search=64, kill_candidates=True, incidents=True)

        def once():
            tm = {}
            cont = taint.contamination(g, res.incidents, {v: {"onset": r[0]} for v, r in res.file_recovery.items()},
                                       timings=tm)
            return tm, sum(len(v) for v in cont.values())
        once()                                                     # warm-up
        runs = [once() for _ in range(a.reps)]
        med = {k: float(np.median([r[0][k] for r in runs])) for k in STAGES}
        med["total"] = sum(med.values())
        rows.append({"t_hi": t_hi - t0, "nodes": g.num_nodes, "edges": g.num_edges, "incidents": len(res.incidents),
                     "contaminated": runs[0][1], "rounds": runs[0][0]["rounds"], "levels": runs[0][0]["levels"],
                     "stages_ms": med, "tick_incidents_ms": float(res.timings_ms.get("incidents", 0.0))})
        print(json.dumps(rows[-1]), flush=True)
    tot = {k: sum(r["stages_ms"][k] for r in rows) for k in rows[0]["stages_ms"]} if rows else {}
    out = {"gpu": gpu, "procs": a.procs, "attacked": a.attacked, "bystanders": a.bystanders, "ticks": rows,
           "contamination_ms": tot, "rounds": sum(r["rounds"] for r in rows), "levels": sum(r["levels"] for r in rows),
           "max_rounds": max((r["rounds"] for r in rows), default=0), "tick_incidents_ms": sum(r["tick_incidents_ms"] for r in rows)}
    print(json.dumps({k: v for k, v in out.items() if k != "ticks"}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
