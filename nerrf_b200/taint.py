"""Contamination: what each incident's attack spread to (DESIGN.md 1.5).

The closure follows information along the direction it flows (a process writes a file, a process reads a file; the
flow class of an event, g.meta["edge_flow"]) and only forward in time: a node is reached by an open edge at t_p when
its source was reached by t_p.  Seeds are the incidents' owners at their onset and their flagged files at their own
recovery points (incident.incidents(return_files=True)).  Every other node the closure reaches is contaminated: files
derived from attacked data (a backup of ciphertext, an index), processes that read it, attacker artefacts written
after the onset.  nerrf_taint_closure runs both phases of the statement on the device.  CUDA only.
"""
from __future__ import annotations

import ctypes as C
import math
import time

import numpy as np
import torch

from . import _lib as L
from .incident import _meta_array


def closure(g, seeds, seed_time, seed_label, max_hops=-1, stage_ms=None) -> dict:
    """nerrf_taint_closure over window graph `g` (CUDA rowptr / col; meta node_kind, edge_flow, edge_time).  seeds: distinct
    node ids; seed_time: float64 each (not NaN; -inf / +inf allowed); seed_label: int >= 0 each; max_hops: -1 = until
    nothing changes.  -> {"nodes" int32, "time" float64 (T), "level" int32, "pred" int64 (CSR position, -1 at level 0),
    "label" int32}: CUDA tensors over the levelled nodes in ascending node id, plus "rounds" and "levels" (ints).
    stage_ms: a dict that receives the milliseconds of validation, phase 1, phase 2 and compaction.  Raises ValueError
    on bad input."""
    rowptr, col = g.rowptr, g.col
    if not (torch.is_tensor(rowptr) and rowptr.is_cuda and torch.is_tensor(col) and col.is_cuda):
        raise L.NerrfError("taint.closure takes a graph of CUDA tensors (no CPU fallback)")
    dev = rowptr.device
    n = rowptr.numel() - 1
    kind = torch.from_numpy(np.asarray(g.meta["node_kind"]).astype(np.int8)).to(dev)
    flow = _meta_array(g, "edge_flow", dev, torch.uint8)
    et = _meta_array(g, "edge_time", dev, torch.float64)
    if flow is None or et is None:
        raise L.NerrfError("taint.closure needs meta['edge_flow'] and meta['edge_time'] (every graph builder sets them)")
    s = torch.as_tensor(np.asarray(seeds, np.int64).reshape(-1)).to(dev)
    st = torch.as_tensor(np.asarray(seed_time, np.float64).reshape(-1)).to(dev)
    sl_h = np.asarray(seed_label, np.int64).reshape(-1)
    if not (s.numel() == st.numel() == sl_h.size):
        raise ValueError("contamination: seeds, seed_time and seed_label must have one entry per seed")
    if sl_h.size and (sl_h.min() < -(1 << 31) or sl_h.max() >= (1 << 31)):
        raise ValueError("contamination: seed labels must fit in int32")
    sl = torch.from_numpy(sl_h.astype(np.int32)).to(dev)
    ns = int(s.numel())
    need = C.c_size_t()
    L.check(L.lib().nerrf_taint_closure_workspace_bytes(n, C.byref(need)), "nerrf_taint_closure_workspace_bytes")
    ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
    m = max(n, 1)
    nodes = torch.empty(m, dtype=torch.int32, device=dev)
    t_out = torch.empty(m, dtype=torch.float64, device=dev)
    level = torch.empty(m, dtype=torch.int32, device=dev)
    pred = torch.empty(m, dtype=torch.int64, device=dev)
    label = torch.empty(m, dtype=torch.int32, device=dev)
    cnt, rounds, levels = C.c_int64(), C.c_int32(), C.c_int32()
    sm = (C.c_double * 4)()
    with torch.cuda.device(dev):
        rc = L.lib().nerrf_taint_closure(L.ptr(rowptr), int(rowptr.dtype == torch.int64), L.ptr(col.contiguous()), n, L.ptr(kind),
                                         L.ptr(flow), L.ptr(et), L.ptr(s) if ns else None, L.ptr(st) if ns else None,
                                         L.ptr(sl) if ns else None, ns, int(max_hops), L.ptr(nodes), L.ptr(t_out), L.ptr(level),
                                         L.ptr(pred), L.ptr(label), C.byref(cnt), C.byref(rounds), C.byref(levels), sm,
                                         L.ptr(ws), ws.numel(), L.current_stream_ptr())
    if rc == -1:
        raise ValueError("contamination: " + L.lib().nerrf_last_error().decode())
    L.check(rc, "nerrf_taint_closure")
    if stage_ms is not None:
        stage_ms.update(zip(("validate", "phase1", "phase2", "compact"), list(sm)))
    k = int(cnt.value)
    return {"nodes": nodes[:k], "time": t_out[:k], "level": level[:k], "pred": pred[:k], "label": label[:k],
            "rounds": int(rounds.value), "levels": int(levels.value)}


def incident_seeds(incident_records, per_file, only=None):
    """-> (seeds, seed_time, seed_label, ids): per incident in list order (label = its index in `ids`), its owner at the
    incident's onset and each of its flagged files at its own onset (per_file[v]["onset"]); entries without a time are
    not seeded.  only=ID: that incident alone."""
    seeds, times, labels, ids, seen = [], [], [], [], set()
    for r in incident_records:
        if only is not None and r["id"] != only:
            continue
        lab = len(ids)
        ids.append(r["id"])
        pts = [(int(r["owner"]), r.get("onset"))] if int(r["owner"]) >= 0 else []
        pts += [(int(v), per_file.get(int(v), {}).get("onset")) for v in r["files"]]
        for v, t in pts:
            if t is None or math.isnan(t) or v in seen:
                continue
            seen.add(v)
            seeds.append(v); times.append(float(t)); labels.append(lab)
    if only is not None and not ids:
        raise ValueError("contamination: unknown incident %r" % (only,))
    return np.asarray(seeds, np.int64), np.asarray(times, np.float64), np.asarray(labels, np.int64), ids


def contamination(g, incident_records, per_file, max_hops=-1, only=None, timings=None) -> dict:
    """The contamination of each incident of `g` (incident.incidents(g, ..., return_files=True) -> records, per_file):
    {incident id: [record]} over the nodes the closure reaches beyond the seeds (level >= 1), each node under the one
    incident its pred chain starts from (the statement's label rule: one closure labels each node once).  A record:
        {"node", "name", "kind" ("file" | "process"), "since" (T: trace-clock seconds), "since_event" (the event of the
         edge that reached it), "hops" (its level), "via" (the events of its pred chain, oldest first)}
    ordered by (since, node).  only=ID: the closure is seeded by that incident alone, so its set is complete.  Events
    are resolved in one g.meta["event_info"] call.  timings: a dict that receives the stage milliseconds (flow_gather,
    validate, phase1 / rounds, phase2 / levels, compact, records)."""
    t0 = time.perf_counter()
    dev = g.rowptr.device
    flow = g.meta.get("edge_flow")
    if callable(flow):                                   # gather the flow class once; the closure reads the tensor
        g = type(g)(g.rowptr, g.col, g.ew, g.x, dict(g.meta, edge_flow=_meta_array(g, "edge_flow", dev, torch.uint8)))
    torch.cuda.synchronize(dev)
    t1 = time.perf_counter()
    seeds, st, sl, ids = incident_seeds(incident_records, per_file, only)
    sm = {}
    res = closure(g, seeds, st, sl, max_hops, stage_ms=sm)
    t2 = time.perf_counter()
    out = {i: [] for i in ids}
    lvl = res["level"]
    nodes = res["nodes"].long()
    has = res["pred"] >= 0
    pos = res["pred"].clamp(min=0)
    src = torch.where(has, g.col.long()[pos], torch.full_like(pos, -1))
    ev_map = _meta_array(g, "edge_event", dev, torch.int64)
    ev = torch.where(has, ev_map[pos], torch.full_like(pos, -1)) if ev_map is not None else torch.full_like(pos, -1)
    nodes_h, t_h, lvl_h, lab_h = (a.cpu().numpy() for a in (nodes, res["time"], lvl, res["label"]))
    src_h, ev_h = src.cpu().numpy(), ev.cpu().numpy()
    row = {int(v): i for i, v in enumerate(nodes_h.tolist())}
    chains = {}
    for i in np.nonzero(lvl_h >= 1)[0].tolist():
        chain, j = [], i
        while lvl_h[j] >= 1:
            chain.append(int(ev_h[j]))
            j = row[int(src_h[j])]
        chains[i] = chain[::-1]
    want = sorted({e for c in chains.values() for e in c if e >= 0})
    info = g.meta.get("event_info")
    rec = dict(zip(want, info(np.asarray(want, np.int64)))) if (info is not None and want) else {}
    names = g.meta.get("names")
    idx = sorted(chains)
    vs = [int(nodes_h[i]) for i in idx]
    nm = (names.take(vs) if hasattr(names, "take") else [names[v] for v in vs]) if names is not None else [None] * len(vs)
    kind = np.asarray(g.meta["node_kind"])
    for i, v, name in zip(idx, vs, nm):
        out[ids[int(lab_h[i])]].append({"node": v, "name": None if name is None else str(name),
                                        "kind": "process" if kind[v] == 1 else "file", "since": float(t_h[i]),
                                        "since_event": rec.get(int(ev_h[i])), "hops": int(lvl_h[i]),
                                        "via": [rec.get(e) for e in chains[i]]})
    for i in out:
        out[i].sort(key=lambda r: (r["since"], r["node"]))
    t3 = time.perf_counter()
    if timings is not None:
        timings.update(flow_gather=(t1 - t0) * 1e3, validate=sm["validate"], phase1=sm["phase1"], rounds=res["rounds"],
                       phase2=sm["phase2"], levels=res["levels"], compact=sm["compact"], records=(t3 - t2) * 1e3)
    return out
