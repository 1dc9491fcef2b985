"""Incidents, restated directly from DESIGN.md 1.4 with per-row Python loops (numpy only): the reference the
nerrf_incident_files / nerrf_incident_group kernels are tested against.

flagged(...)  -> flagged files in ascending node id and, per file, its owner, first / last position, later count,
                 onset / end time and event
incidents(...) -> the incident records, ordered by (onset, source, owner), owner -1 last, NaN onsets after every number
"""
from __future__ import annotations

import math

import numpy as np


def flagged(rowptr, col, node_kind, score, tau=0.5, seeds=None, edge_attack=None, edge_time=None, edge_event=None):
    """-> dict of numpy arrays over the flagged files F (ascending node id): files, owner, first, last, later, onset, end,
    onset_event, end_event.  Raises ValueError on bad input (the ABI's NERRF_ERR_INVALID)."""
    rowptr = np.asarray(rowptr, np.int64)
    col = np.asarray(col, np.int64)
    kind = np.asarray(node_kind, np.int64)
    score = np.asarray(score, np.float32)
    n = rowptr.shape[0] - 1
    if math.isnan(float(tau)):
        raise ValueError("tau is NaN")
    if np.any((kind != 0) & (kind != 1)):
        raise ValueError("node_kind values must be 0 or 1")
    if col.size and (col.min() < 0 or col.max() >= n):
        raise ValueError("col holds node ids outside [0, n)")
    flag = (kind == 0) & (score >= np.float32(tau))
    for s in ([] if seeds is None else np.asarray(seeds, np.int64).reshape(-1).tolist()):
        if not 0 <= s < n:
            raise ValueError("seed node ids must lie in [0, %d)" % n)
        if kind[s] != 0:
            raise ValueError("a seed is not a file node")
        flag[s] = True
    files = np.nonzero(flag)[0].astype(np.int64)
    m = files.shape[0]
    out = {"files": files, "owner": np.full(m, -1, np.int64), "first": np.full(m, -1, np.int64),
           "last": np.full(m, -1, np.int64), "later": np.zeros(m, np.int64), "onset": np.full(m, np.nan),
           "end": np.full(m, np.nan), "onset_event": np.full(m, -1, np.int64), "end_event": np.full(m, -1, np.int64)}
    ea = None if edge_attack is None else np.asarray(edge_attack, np.float32)
    for i, v in enumerate(files.tolist()):
        b, e = int(rowptr[v]), int(rowptr[v + 1])
        if e == b:
            continue
        procs = [p for p in range(b, e) if kind[col[p]] == 1]
        own = -1
        if procs and ea is None:
            own = int(col[procs[-1]])                        # the last process in-edge
        elif procs:
            best = procs[0]
            for p in procs[1:]:                              # highest P(attack), NaN above every number, ties to the later
                a, c = ea[p], ea[best]
                if math.isnan(a) or (not math.isnan(c) and a >= c):
                    best = p
            own = int(col[best])
        if own < 0:
            first, last, later = b, e - 1, 0
        else:
            mine = [p for p in range(b, e) if col[p] == own]
            first, last = mine[0], mine[-1]
            later = sum(1 for p in range(first + 1, e) if kind[col[p]] == 1 and col[p] != own)
        out["owner"][i], out["first"][i], out["last"][i], out["later"][i] = own, first, last, later
        if edge_time is not None:
            out["onset"][i], out["end"][i] = float(edge_time[first]), float(edge_time[last])
        if edge_event is not None:
            out["onset_event"][i], out["end_event"][i] = int(edge_event[first]), int(edge_event[last])
    return out


def incidents(fl: dict, node_source=None, size_mb=None, score=None) -> list:
    """fl = flagged(...) -> incident records {source, owner, files (ascending), n_files, onset, onset_event, end,
    end_event, size_mb, later, max_score}, ordered by (onset, source, owner)."""
    files = fl["files"]
    groups: dict = {}
    for i, v in enumerate(files.tolist()):
        src = 0 if node_source is None else int(node_source[v])
        groups.setdefault((src, int(fl["owner"][i])), []).append(i)
    recs = []
    for (src, own), idx in groups.items():
        r = {"source": src, "owner": own, "files": [int(files[i]) for i in idx], "n_files": len(idx),
             "onset": math.nan, "onset_event": -1, "end": math.nan, "end_event": -1, "size_mb": 0.0, "later": 0,
             "max_score": math.nan}
        for i in idx:                                        # ascending node id: strict comparisons keep the lower id
            t = float(fl["onset"][i])
            if not math.isnan(t) and (math.isnan(r["onset"]) or t < r["onset"]):
                r["onset"], r["onset_event"] = t, int(fl["onset_event"][i])
            t = float(fl["end"][i])
            if not math.isnan(t) and (math.isnan(r["end"]) or t > r["end"]):
                r["end"], r["end_event"] = t, int(fl["end_event"][i])
            v = int(files[i])
            r["size_mb"] += 0.0 if size_mb is None else float(np.float32(size_mb[v]))
            r["later"] += int(fl["later"][i])
            if score is not None and not math.isnan(float(score[v])):
                s = float(np.float32(score[v]))
                r["max_score"] = s if math.isnan(r["max_score"]) else max(r["max_score"], s)
        recs.append(r)
    recs.sort(key=lambda r: (math.isnan(r["onset"]), 0.0 if math.isnan(r["onset"]) else r["onset"], r["source"],
                             r["owner"] < 0, r["owner"]))
    return recs
