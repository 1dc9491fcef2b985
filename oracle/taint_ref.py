"""Contamination, restated directly from DESIGN.md 1.5 with per-row Python loops (numpy only): the reference the
nerrf_taint_closure kernel is tested against, plus an independent earliest-arrival sweep for max_hops = -1.

flow_class(event, flags, ret_val) -> the 2-bit flow class of one event (bit 0 process -> file, bit 1 file -> process)
closure(...)                      -> both phases exactly as stated: T, level, pred, label, rounds, levels
earliest_arrival(...)             -> T by a sweep over the open edges in non-decreasing time (max_hops = -1 only)
"""
from __future__ import annotations

import math

import numpy as np

P2F, F2P = 1, 2
_KINDS = ("file_created", "file_encrypt_start", "file_encrypt_complete", "ransom_note_created", "openat", "write", "rename")
_WRITES = {"write", "rename", "file_encrypt_start", "file_encrypt_complete", "file_created", "ransom_note_created"}


def flow_class(event, flags=0, ret_val=0) -> int:
    """event: a kind name or a raw slot (graph._EVENT_SLOT order, 7 = other).  Integers only."""
    name = _KINDS[event] if isinstance(event, (int, np.integer)) and 0 <= int(event) < len(_KINDS) else event
    if int(ret_val) < 0:
        return 0
    if name in _WRITES:
        return P2F
    if name == "openat":
        return F2P if int(flags) == 0 else P2F if int(flags) == 1 else P2F | F2P
    return 0


def _check(rowptr, col, kind, flow, seeds, seed_time, seed_label, max_hops):
    n = rowptr.shape[0] - 1
    if np.any((kind != 0) & (kind != 1)):
        raise ValueError("node_kind values must be 0 or 1")
    if col.size and (col.min() < 0 or col.max() >= n):
        raise ValueError("col holds node ids outside [0, n)")
    if flow.size and flow.max() > 3:
        raise ValueError("edge_flow bytes must lie in [0, 3]")
    if seeds.size and (seeds.min() < 0 or seeds.max() >= n):
        raise ValueError("seed node ids must lie in [0, %d)" % n)
    if np.unique(seeds).size != seeds.size:
        raise ValueError("seed node ids must be distinct")
    if np.any(np.isnan(seed_time)):
        raise ValueError("a seed time is NaN")
    if np.any(seed_label < 0):
        raise ValueError("seed labels must be >= 0")
    if max_hops < -1:
        raise ValueError("max_hops must be -1 or >= 0")


def _open(kind, flow, et, u, v, p) -> bool:
    if math.isnan(et[p]):
        return False
    if kind[u] == 1 and kind[v] == 0:
        return bool(flow[p] & P2F)
    if kind[u] == 0 and kind[v] == 1:
        return bool(flow[p] & F2P)
    return False


def _arrays(rowptr, col, node_kind, edge_flow, edge_time, seeds, seed_time, seed_label):
    return (np.asarray(rowptr, np.int64), np.asarray(col, np.int64), np.asarray(node_kind, np.int64),
            np.asarray(edge_flow, np.int64), np.asarray(edge_time, np.float64), np.asarray(seeds, np.int64).reshape(-1),
            np.asarray(seed_time, np.float64).reshape(-1),
            np.zeros(0, np.int64) if seed_label is None else np.asarray(seed_label, np.int64).reshape(-1))


def closure(rowptr, col, node_kind, edge_flow, edge_time, seeds, seed_time, seed_label, max_hops=-1) -> dict:
    """-> {"T" float64 [n], "level" int64 [n] (-1 unlevelled), "pred" int64 [n] (-1), "label" int64 [n] (-1),
    "nodes" (levelled, ascending), "rounds", "levels"}.  Raises ValueError on bad input (the ABI's NERRF_ERR_INVALID)."""
    rowptr, col, kind, flow, et, seeds, st, sl = _arrays(rowptr, col, node_kind, edge_flow, edge_time, seeds, seed_time, seed_label)
    _check(rowptr, col, kind, flow, seeds, st, sl, max_hops)
    n = rowptr.shape[0] - 1
    T = np.full(n, np.inf)
    T[seeds] = st
    # phase 1: Jacobi rounds, each reading the previous round's T only
    rounds = 0
    r = 0
    while n and (max_hops < 0 or r < max_hops):
        r += 1
        nxt = T.copy()
        for v in range(n):
            best = None                                          # (t, p): the smallest time, ties to the lower position
            for p in range(int(rowptr[v]), int(rowptr[v + 1])):
                u = int(col[p])
                if _open(kind, flow, et, u, v, p) and T[u] <= et[p] and (best is None or et[p] < best[0]):
                    best = (float(et[p]), p)
            if best is not None and best[0] < T[v]:
                nxt[v] = best[0]
        rounds = r
        changed = bool(np.any(nxt != T))
        T = nxt
        if not changed:
            break
    # phase 2: level-synchronous BFS over the tight edges
    level = np.full(n, -1, np.int64)
    pred = np.full(n, -1, np.int64)
    label = np.full(n, -1, np.int64)
    for s, t, lab in zip(seeds.tolist(), st.tolist(), sl.tolist()):
        if T[s] == t:
            level[s], label[s] = 0, lab
    levels = 1 if np.any(level == 0) else 0
    k = 0
    while levels:
        new = []
        for v in range(n):
            if level[v] != -1 or not T[v] < np.inf:
                continue
            for p in range(int(rowptr[v]), int(rowptr[v + 1])):     # ascending: the first hit is the lowest position
                u = int(col[p])
                if _open(kind, flow, et, u, v, p) and et[p] == T[v] and level[u] == k and T[u] <= et[p]:
                    new.append((v, p))
                    break
        if not new:
            break
        for v, p in new:
            level[v], pred[v], label[v] = k + 1, p, label[col[p]]
        k += 1
        levels = k + 1
    return {"T": T, "level": level, "pred": pred, "label": label, "nodes": np.nonzero(level >= 0)[0].astype(np.int64),
            "rounds": rounds, "levels": levels}


def earliest_arrival(rowptr, col, node_kind, edge_flow, edge_time, seeds, seed_time) -> np.ndarray:
    """T of max_hops = -1 by an independent route: the open edges in non-decreasing time, each group of equal times
    relaxed to a fixed point (an edge u -> v at t lowers T[v] to t when T[u] <= t < T[v])."""
    rowptr, col, kind, flow, et, seeds, st, _ = _arrays(rowptr, col, node_kind, edge_flow, edge_time, seeds, seed_time, None)
    n = rowptr.shape[0] - 1
    T = np.full(n, np.inf)
    T[seeds] = st
    edges = []
    for v in range(n):
        for p in range(int(rowptr[v]), int(rowptr[v + 1])):
            u = int(col[p])
            if _open(kind, flow, et, u, v, p):
                edges.append((float(et[p]), u, v))
    edges.sort(key=lambda e: e[0])
    i = 0
    while i < len(edges):
        j = i
        while j < len(edges) and edges[j][0] == edges[i][0]:
            j += 1
        group = edges[i:j]
        changed = True
        while changed:
            changed = False
            for t, u, v in group:
                if T[u] <= t < T[v]:
                    T[v] = t
                    changed = True
        i = j
    return T
