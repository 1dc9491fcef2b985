"""Live ingest of several hosts' streams: 8 hosts (stream.host_streams(8, 1300, 5): 10,400 processes in all, the cfg-5
fleet's count, every other host attacked) fed to DeviceStream.live in 1-s batches per host, interleaved across hosts in
trace time, each append with its host's source id; the same events relabelled as ONE source
(stream.relabel_single_source: one pid per (host, pid), paths prefixed "@<host>/") fed in the same batches, in the same
process, alternately.  The multi-source feed regroups by (source, pid) in 6 radix passes, the single-source one by pid in 4.

Per append (CUDA events): device decode, rebuild (time order + resolution + columns) and compaction; per tick: the window
graph (interning, features, CSR) of the 60-s window, every 30 s of trace time once every host has delivered past it;
median / p99 of the second of two passes over each feed; the GPU and its power limit.

    python scripts/multi_source_timing.py [--hosts 8] [--procs-per-host 1300] [--out file.json]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from nerrf_b200 import ingest, stream  # noqa: E402
from live_stream_timing import gpu_info, pct  # noqa: E402


def pieces_of(cols):
    """-> [(max ts, source, row indices)]: each host's rows in 1-s batches of its trace time, all hosts interleaved"""
    out = []
    ts = cols.timestamp
    for s in np.unique(cols.source).tolist():
        rows = np.nonzero(cols.source == s)[0]
        rows = rows[np.argsort(ts[rows], kind="stable")]
        key = np.floor(ts[rows] - ts.min()).astype(np.int64)
        for part in np.split(rows, np.nonzero(np.diff(key))[0] + 1):
            out.append((float(ts[part].max()), int(s), part))
    out.sort(key=lambda p: (p[0], p[1]))
    return out


def tick_schedule(pieces, k_hosts, tick):
    """after piece j, the tick times that fire: every open host has delivered an event past t_hi (lateness 0); a host
    closes with its last batch (StreamingPlanner.close_source)"""
    last_piece = {s: j for j, (_, s, _) in enumerate(pieces)}
    latest, t_hi, t0, out = {}, None, min(p[0] for p in pieces), []
    for j, (t, s, _) in enumerate(pieces):
        latest[s] = max(latest.get(s, -np.inf), t)
        fire = []
        if len(latest) == k_hosts:
            t_hi = t0 if t_hi is None else t_hi
            mark = min([v for h, v in latest.items() if last_piece[h] > j], default=max(latest.values()))
            while mark > t_hi + tick:
                t_hi += tick
                fire.append(t_hi)
        out.append(fire)
    return out


def run(wires, sources, schedule, window):
    ds = stream.DeviceStream.live("cuda", observable=True)
    dec, reb, comp, graph = [], [], [], []
    for w, s, fire in zip(wires, sources, schedule):
        ds.append(w, source=s)
        dec.append(ds.timings_ms.get("decode_ms", 0.0)); reb.append(ds.timings_ms.get("rebuild_ms", 0.0))
        for t_hi in fire:
            torch.cuda.synchronize()
            a = time.perf_counter()
            g = ds.window_graph(t_hi - window, t_hi, window)
            torch.cuda.synchronize()
            graph.append((time.perf_counter() - a) * 1e3)
            del g
            ds.compact(t_hi - window)
            comp.append(ds.timings_ms["compact_ms"])
    stat = lambda v: {"median": pct(v, 50), "p99": pct(v, 99)}
    return {"decode_ms": stat(dec), "rebuild_ms": stat(reb), "compact_ms": stat(comp), "tick_graph_ms": stat(graph),
            "ticks": len(graph), "key_bits": ds._key_bits}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hosts", type=int, default=8); ap.add_argument("--procs-per-host", type=int, default=1300)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    info = gpu_info()
    hs = stream.host_streams(a.hosts, a.procs_per_host, 5, seed=5)
    cols = stream.concat_columns([c for c, _, _ in hs])
    pieces = pieces_of(cols)
    window, tick = 60.0, 30.0
    schedule = tick_schedule(pieces, a.hosts, tick)
    multi_recs = ingest.encode_columns(cols)
    single_recs = ingest.encode_columns(stream.relabel_single_source(cols))
    multi = [b"".join(multi_recs[i] for i in p.tolist()) for _, _, p in pieces]
    single = [b"".join(single_recs[i] for i in p.tolist()) for _, _, p in pieces]
    sources = [s for _, s, _ in pieces]
    res = {}
    for rep in range(2):                                          # the first pass of each warms allocator and kernels
        for name, wires, src in (("multi_source", multi, sources), ("one_source_relabelled", single, [0] * len(sources))):
            res[name] = run(wires, src, schedule, window)
    out = {"gpu": info, "hosts": a.hosts, "events": int(cols.n), "appends": len(pieces),
           "wire_bytes": {"multi_source": sum(map(len, multi)), "one_source_relabelled": sum(map(len, single))}, **res}
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
