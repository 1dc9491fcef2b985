"""`nerrf undo` for the hot path: trace in, undo plan out (SURVEY.md 8f rank 4; reference CLI `nerrf undo --id <attack>`,
ROADMAP.md:28,86 -- scheduled, never written).

    python -m nerrf_b200.undo --trace events.pb   --weights weights.pt --out plan.json --shell plan.sh
    python -m nerrf_b200.undo --trace trace.jsonl --train-epochs 25    --out plan.json
    python -m nerrf_b200.undo --trace trace.jsonl --train-epochs 25    --out plan.json --explain 8
    python -m nerrf_b200.undo --trace trace.jsonl --train-epochs 25    --out plan.json --explain-sequences 8
    python -m nerrf_b200.undo --trace nodeA=a.pb --trace nodeB=b.pb --weights weights.pt --out plan.json --shell-dir DIR
    python -m nerrf_b200.undo --trace events.pb   --weights weights.pt --out plan.json --incidents
    python -m nerrf_b200.undo --trace events.pb   --weights weights.pt --out plan.json --incident pid:454
    python -m nerrf_b200.undo --trace events.pb   --weights weights.pt --out plan.json --incidents --contamination

trace: serialized nerrf.trace.EventBatch bytes (*.pb; proto/trace.proto:47-49, e.g. a buffered StreamEvents stream) or
the simulator's TRACE json lines (*.jsonl; benchmarks/m1/scripts/sim_lockbit_m1.py:24-36).  Stages: ingest -> temporal
graph (features + CSR on the GPU for *.pb) -> GraphSAGE_T.forward -> top-A candidates -> lstm.forward -> mcts plan ->
emit.  Everything between the graph and the plan runs in the CUDA kernels; there is no CPU fallback.

Several `--trace HOST=PATH` arguments (*.pb, one per node's tracker) are planned as one graph whose processes and files
are per host (source ids in argument order); every step of the plan names its "host", and --shell-dir writes one
DIR/<host>.sh per host (--shell is refused: one script would hold every host's commands, and the hosts share file
names).  A bare `--trace PATH`, or a single `--trace HOST=PATH`, is one source, as before: no host fields, and
--shell-dir needs the HOST name.

--incidents groups the plan's steps by the process that attacked their files (DESIGN.md 1.4): a top-level "incidents"
table, the "incident" of every step and the "recovery_point" of every file step.  --incident ID plans that incident
alone (ids are "pid:N", "unattributed", or "HOST/pid:N" with several hosts): the full plan is labelled first, then
planned again with every file outside the incident excluded.  --contamination adds to every incident of the table the
nodes its attack spread to (DESIGN.md 1.5: files written and processes that read after the taint arrived, each with
the events that carried it and, for a file, its recovery point); with --incident ID the closure is seeded by that
incident alone.  --contamination-hops H bounds the closure to H hops.  Plan steps are unchanged.
"""
from __future__ import annotations

import argparse
import math
import os
import sys
import time

import numpy as np
import torch

from . import graph as G, ingest, pipeline
from .ai import train as T
from .ai.models import GraphSAGE_T
from .ai.models.lstm import LSTMScorer
from .ai.planner import emit
from .stream import concat_columns, with_source


def parse_traces(specs) -> list:
    """--trace values -> [(host or None, path)]: one bare PATH, or HOST=PATH for every source"""
    out = []
    for sp in specs:
        host, eq, path = sp.partition("=")
        out.append((emit.check_host_name(host), path) if eq and not os.path.exists(sp) else (None, sp))
    if len(out) > 1 and any(h is None for h, _ in out):
        raise SystemExit("several --trace arguments: give every one as HOST=PATH")
    if len({h for h, _ in out}) < len(out):
        raise SystemExit("--trace: a host name appears twice")
    return out


def check_outputs(traces, shell, shell_dir):
    """refuse script outputs that do not fit the traces: --shell with several hosts, --shell-dir without host names"""
    if shell and len(traces) > 1:
        raise SystemExit("--shell with several --trace HOST=PATH: use --shell-dir (one script per host)")
    if shell_dir and traces[0][0] is None:
        raise SystemExit("--shell-dir names its scripts by host: give the trace as --trace HOST=PATH")


def check_incident_args(a):
    """--incident-threshold needs --incidents or --incident, and is a number; --incident takes a non-empty id"""
    if a.incident_threshold is not None:
        if not (a.incidents or a.incident is not None):
            raise SystemExit("--incident-threshold needs --incidents or --incident ID")
        if math.isnan(a.incident_threshold):
            raise SystemExit("--incident-threshold must be a number")
    if a.incident is not None and not a.incident:
        raise SystemExit("--incident needs an incident id (pid:N, unattributed, or HOST/pid:N)")


def check_contamination_args(a):
    """--contamination needs --incidents or --incident; --contamination-hops needs --contamination and is >= -1"""
    if a.contamination and not (a.incidents or a.incident is not None):
        raise SystemExit("--contamination needs --incidents or --incident ID")
    if a.contamination_hops is not None:
        if not a.contamination:
            raise SystemExit("--contamination-hops needs --contamination")
        if a.contamination_hops < -1:
            raise SystemExit("--contamination-hops must be -1 (unbounded) or >= 0")


def load_hosts(paths, device="cuda", events=False):
    """several hosts' EventBatch files as one stream, source id k = the k-th file -> (graph, seq, lengths, seq_nodes, n)
    (events=True: and the event of each sequence step, last)"""
    parts = []
    for k, path in enumerate(paths):
        if not path.endswith(".pb"):
            raise SystemExit("several --trace arguments take EventBatch files (*.pb): %s" % path)
        with open(path, "rb") as f:
            parts.append(with_source(ingest.decode_event_batch(f.read()), k))
    cols = concat_columns(parts)
    g = ingest.graph_from_columns(cols, device=device, observable=True)
    seq, lengths, nodes, *ev = ingest.sequences_from_columns(cols, observable=True, return_events=events)
    return (g, seq, lengths, nodes, cols.n, *ev)


def load_trace(path: str, device="cuda", events=False):
    """-> (graph, seq, lengths, seq_nodes, n_events) (events=True: and the event of each sequence step, last)"""
    if path.endswith(".jsonl") or path.endswith(".json"):
        evs = G.read_trace_jsonl(path)
        g = G.graph_from_events(evs, observable=True)             # the features ai/train.py trains on
        seq, lengths, nodes, *ev = pipeline.file_sequences(evs, g, observable=True, return_events=events)
        return (g, seq, lengths, nodes, len(evs), *ev)
    with open(path, "rb") as f:
        cols = ingest.decode_event_batch(f.read())
    g = ingest.graph_from_columns(cols, device=device, observable=True)
    seq, lengths, nodes, *ev = ingest.sequences_from_columns(cols, observable=True, return_events=events)
    return (g, seq, lengths, nodes, cols.n, *ev)


def load_models(weights: str | None, train_epochs: int, layers: int = 2, log=print):
    model, scorer = GraphSAGE_T(G.F_IN, 128, layers), LSTMScorer()
    if weights:
        ck = torch.load(weights, map_location="cpu")
        model = GraphSAGE_T(G.F_IN, 128, int(ck.get("layers", layers)))
        model.load_state_dict(ck["sage"])
        if ck.get("edge_head_trained"):                             # ai.train --edge-loss: files are attributed by the edge head
            model.edge_head_trained = True
        if ck.get("lstm") is not None:
            scorer.load_state_dict(ck["lstm"])
    elif train_epochs > 0:
        log(f"no --weights: training {train_epochs} epochs on the simulated toy set (ai/train.py)")
        torch.manual_seed(0)
        T.train(model, scorer, T.toy_set(range(100, 104)), epochs=train_epochs)
    else:
        raise SystemExit("no weights: pass --weights FILE (from `python -m nerrf_b200.ai.train --out FILE`) or --train-epochs N")
    return model, scorer


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(prog="python -m nerrf_b200.undo", description=__doc__.split("\n")[0])
    ap.add_argument("--trace", required=True, action="append",
                    help="trace file, or HOST=FILE once per host (*.pb) for a plan over several hosts")
    ap.add_argument("--id", default=None, help="attack id carried into the plan")
    ap.add_argument("--weights", default=None); ap.add_argument("--train-epochs", type=int, default=0)
    ap.add_argument("--out", default=None, help="plan JSON (default: stdout)"); ap.add_argument("--shell", default=None)
    ap.add_argument("--top-a", type=int, default=1024); ap.add_argument("--rollouts", type=int, default=1024)
    ap.add_argument("--depth", type=int, default=50); ap.add_argument("--iterations", type=int, default=16)
    ap.add_argument("--max-steps", type=int, default=None,
                    help="cap on the number of reversions (default: every candidate may be reverted); a capped plan that "
                         "leaves improving candidates is marked truncated and is not auto-approvable")
    ap.add_argument("--shell-dir", default=None, help="write DIR/<host>.sh per --trace HOST=PATH")
    ap.add_argument("--explain", type=int, default=0, metavar="K",
                    help="attach to every node step the K trace events whose edges drove its GraphSAGE-T score most")
    ap.add_argument("--explain-sequences", type=int, default=0, metavar="K",
                    help="attach to every file step the K events of its history that drove its BiLSTM encrypt score most")
    ap.add_argument("--incidents", action="store_true",
                    help="group the steps into incidents (one per attacking process) with per-file recovery points")
    ap.add_argument("--incident-threshold", type=float, default=None, metavar="T",
                    help="anomaly score at or above which a file belongs to an incident (default 0.5)")
    ap.add_argument("--incident", default=None, metavar="ID", help="plan only the incident ID (pid:N, or HOST/pid:N)")
    ap.add_argument("--contamination", action="store_true",
                    help="list under each incident what its attack spread to: derived files and processes that read them")
    ap.add_argument("--contamination-hops", type=int, default=None, metavar="H",
                    help="bound the contamination closure to H hops (default -1: unbounded)")
    ap.add_argument("--device", default="cuda")
    a = ap.parse_args(argv)
    traces = parse_traces(a.trace)
    check_outputs(traces, a.shell, a.shell_dir)
    check_incident_args(a)
    check_contamination_args(a)
    hosts = [h for h, _ in traces] if len(traces) > 1 else None     # host fields only with several sources
    if not torch.cuda.is_available():
        raise SystemExit("nerrf_b200.undo needs a CUDA device (no CPU fallback for the hot path)")
    log = lambda *m: print(*m, file=sys.stderr)
    t0 = time.perf_counter()
    want_ev = a.explain_sequences > 0
    if hosts is None:
        g, seq, lengths, nodes, n_events, *ev = load_trace(traces[0][1], a.device, events=want_ev)
    else:
        g, seq, lengths, nodes, n_events, *ev = load_hosts([p for _, p in traces], a.device, events=want_ev)
    t_ingest = (time.perf_counter() - t0) * 1e3
    model, scorer = load_models(a.weights, a.train_epochs, log=log)
    model.to(a.device); scorer.to(a.device)
    want_inc = a.incidents or a.incident is not None
    tau = 0.5 if a.incident_threshold is None else a.incident_threshold
    run = lambda exclude=None: pipeline.run(g, seq, lengths, nodes, model, scorer, top_a=min(a.top_a, 4096), n_rollouts=a.rollouts,
                                            depth=a.depth, iterations=a.iterations, plan_steps=a.max_steps, device=a.device,
                                            explain=a.explain, explain_sequences=a.explain_sequences,
                                            seq_events=ev[0] if ev else None, exclude=exclude, incidents=want_inc,
                                            incident_tau=tau, host_names=hosts,
                                            contamination=a.contamination and a.incident is None and exclude is None,
                                            contamination_hops=hops)
    hops = -1 if a.contamination_hops is None else a.contamination_hops
    res = run()
    attack_id = a.id
    if a.incident is not None:
        known = {r["id"]: r for r in (res.incidents or [])}            # None: no candidate file had a sequence
        if a.incident not in known:
            raise SystemExit("unknown incident %r; this trace's incidents: %s" % (a.incident, ", ".join(known) or "(none)"))
        mine = np.asarray(known[a.incident]["files"], np.int64)
        full = res
        res = run(exclude=~np.isin(np.asarray(nodes, np.int64), mine))   # every file outside the incident is excluded
        attack_id = a.incident if a.id is None else a.id
        if a.contamination:                                            # seeded by the incident alone, as the full plan found it
            res.contamination = pipeline.contamination_of(g, full, hops, only=a.incident, device=a.device)
    plan = emit.from_pipeline(g, res, attack_id=attack_id, host_names=hosts)
    plan["stats"] = {"events": int(n_events), "nodes": int(g.num_nodes), "edges": int(g.num_edges),
                     "candidates": int(len(res.candidates)), "ingest_ms": t_ingest,
                     "timings_ms": {k: float(v) for k, v in res.timings_ms.items()}}
    text = emit.to_json(plan)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")
    else:
        print(text)
    if a.shell:
        with open(a.shell, "w") as f:
            f.write(emit.to_shell(plan))
    if a.shell_dir:
        os.makedirs(a.shell_dir, exist_ok=True)
        for h, _ in traces:
            with open(os.path.join(a.shell_dir, emit.check_host_name(h) + ".sh"), "w") as f:
                f.write(emit.to_shell(plan, host=h if hosts else None))
    log(f"{n_events} events -> {g.num_nodes} nodes / {g.num_edges} edges -> {len(plan['steps'])} reversions "
        f"(ingest {t_ingest:.1f} ms, hot path {res.timings_ms['total']:.1f} ms)")
    return plan


if __name__ == "__main__":
    main()
