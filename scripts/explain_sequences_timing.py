"""Time the BiLSTM sequence explanation of a cfg-5-size plan, stage by stage (DESIGN.md 1.2.1 / 6).

    python scripts/explain_sequences_timing.py [--procs 10400] [--attacked 40] [--k 8] [--reps 5] [--max-batch 512] [--out f.json]

The workload of scripts/explain_timing.py: the cfg-5 fleet trace of bench.py (fleet_columns(procs, attacked, seed=5)),
toy-trained weights as bench.py trains them, a StreamingPlanner run (kill candidates) for the ticks; every tick's window
graph is rebuilt, planned once (pipeline.run, kill candidates) and its planned FILE steps explained: sequences with
events (nerrf_trace_sequences_ex), forward (nerrf_lstm_forward_train), input gradient (nerrf_lstm_input_grad), steps
(nerrf_lstm_explain_steps), records (explain.attach_events), max_batch sequences at a time.  Each stage ends in a device
synchronise; per tick the median of --reps timed runs after one warm-up.  Printed beside the same tick's lstm and
graphsage_t time, with the card's name and power limit.
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


def stages(ds, g, scorer, files, k, max_batch):
    sync = torch.cuda.synchronize
    tm = dict.fromkeys(("sequences_events", "forward_train", "input_grad", "explain_steps", "records"), 0.0)
    a = time.perf_counter()
    seq, ln, ev = ds.sequences_device(g, files, events=True)
    sync(); tm["sequences_events"] = (time.perf_counter() - a) * 1e3
    w = EX._seq_weights(scorer, seq.device)
    out = []
    for s in range(0, len(files), max_batch):
        e = min(s + max_batch, len(files))
        sq, lc = seq[s:e].contiguous(), ln[s:e].contiguous()
        a = time.perf_counter()
        hfin, tape = EX.lstm_forward_tape(scorer, w, sq, lc)
        sync(); tm["forward_train"] += (time.perf_counter() - a) * 1e3
        a = time.perf_counter()
        dseq = EX.lstm_input_grad(scorer, w, sq, lc, tape)
        sync(); tm["input_grad"] += (time.perf_counter() - a) * 1e3
        a = time.perf_counter()
        st, at, ft, vt = EX.explain_steps(sq, dseq, lc, ev[s:e].contiguous(), k)
        sync(); tm["explain_steps"] += (time.perf_counter() - a) * 1e3
        st, vt = st.cpu().numpy(), vt.cpu().numpy()
        out += [{"logit": 0.0, "steps": [{"t": int(st[i, j]), "attr": 0.0, "feature": 0, "event": int(vt[i, j])}
                                         for j in np.nonzero(st[i] >= 0)[0]]} for i in range(e - s)]
    a = time.perf_counter()
    EX.attach_events(g, [], out)
    sync(); tm["records"] = (time.perf_counter() - a) * 1e3
    tm["explain_total"] = sum(tm.values())
    return tm


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--procs", type=int, default=10400); ap.add_argument("--attacked", type=int, default=40)
    ap.add_argument("--k", type=int, default=8); ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--max-batch", type=int, default=512); ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("explain_sequences_timing needs a CUDA device")
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
        steps = np.asarray([n for n in dict.fromkeys(res.plan_nodes) if kind[n] == 0], np.int64)
        if not steps.size:
            continue
        stages(ds, g, scorer, steps, a.k, a.max_batch)                   # warm-up
        runs = [stages(ds, g, scorer, steps, a.k, a.max_batch) for _ in range(a.reps)]
        med = {key: float(np.median([r[key] for r in runs])) for key in runs[0]}
        rows.append({"t_hi": t.t_hi, "nodes": g.num_nodes, "edges": g.num_edges, "file_steps": int(steps.size),
                     "stages_ms": med, "tick_lstm_ms": float(res.timings_ms.get("lstm", 0.0)),
                     "tick_graphsage_t_ms": float(res.timings_ms.get("graphsage_t", 0.0))})
        print(json.dumps(rows[-1]), flush=True)
    tot = {key: sum(r["stages_ms"][key] for r in rows) for key in rows[0]["stages_ms"]} if rows else {}
    out = {"gpu": gpu, "procs": a.procs, "attacked": a.attacked, "k": a.k, "max_batch": a.max_batch, "ticks": rows,
           "file_steps": sum(r["file_steps"] for r in rows), "explain_ms": tot,
           "tick_lstm_ms": sum(r["tick_lstm_ms"] for r in rows),
           "tick_graphsage_t_ms": sum(r["tick_graphsage_t_ms"] for r in rows)}
    print(json.dumps({k: v for k, v in out.items() if k != "ticks"}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
