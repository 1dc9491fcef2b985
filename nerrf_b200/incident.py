"""Incidents: the detections of a window grouped by the process that attacked them (DESIGN.md 1.4).

An incident is one attributed process together with the flagged files attributed to it (pipeline.file_owners' rule:
the last writer, or the trained edge head's strongest process edge).  Files with no process source in their row form
their host's single "unattributed" incident.  Per file the incident also gives its recovery point: the first event of
its owner in its row (a restore must go back to before it) and the count of other processes' events after that one
(what such a restore discards).  nerrf_incident_files flags the files and attributes them, one warp per row;
nerrf_incident_group groups them with a radix sort and reduces each incident in a fixed order.  CUDA only.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _lib as L


def _meta_array(g, name, dev, dtype):
    a = g.meta.get(name)
    if callable(a):
        a = a()
    if a is None:
        return None
    return torch.as_tensor(a).to(device=dev, dtype=dtype).contiguous()


def incident_id(owner_name, source, host_names=None, multi=False) -> str:
    """"pid:N" (the owner's node name) or "unattributed", prefixed by "host/" when the graph has several sources"""
    base = "unattributed" if owner_name is None else str(owner_name)
    if not multi:
        return base
    host = host_names[int(source)] if host_names is not None and 0 <= int(source) < len(host_names) else str(int(source))
    return "%s/%s" % (host, base)


def flag_files(rowptr, col, node_kind, score, tau=0.5, seeds=None, edge_attack=None, edge_time=None, edge_event=None):
    """nerrf_incident_files -> (files int32 [m], file_int int64 [m, 6], file_real float64 [m, 2]) CUDA tensors (rows
    as include/nerrf_b200.h documents them).  Raises ValueError on bad input."""
    dev = rowptr.device
    n = rowptr.numel() - 1
    if math.isnan(float(tau)):
        raise ValueError("tau is NaN")
    seeds_t = None if seeds is None else torch.as_tensor(np.asarray(seeds, np.int64).reshape(-1)).to(dev)
    ns = 0 if seeds_t is None else int(seeds_t.numel())
    need = C.c_size_t()
    L.check(L.lib().nerrf_incident_files_workspace_bytes(n, C.byref(need)), "nerrf_incident_files_workspace_bytes")
    ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
    files = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    fi = torch.empty(max(n, 1), 6, dtype=torch.int64, device=dev)
    fr = torch.empty(max(n, 1), 2, dtype=torch.float64, device=dev)
    m = C.c_int64()
    with torch.cuda.device(dev):
        rc = L.lib().nerrf_incident_files(L.ptr(rowptr), int(rowptr.dtype == torch.int64), L.ptr(col), n, L.ptr(node_kind),
                                          L.ptr(score), float(tau), L.ptr(seeds_t) if ns else None, ns, L.ptr(edge_attack),
                                          L.ptr(edge_time), L.ptr(edge_event), L.ptr(files), L.ptr(fi), L.ptr(fr), C.byref(m),
                                          L.ptr(ws), ws.numel(), L.current_stream_ptr())
    if rc == -1:
        raise ValueError("incidents: " + L.lib().nerrf_last_error().decode())
    L.check(rc, "nerrf_incident_files")
    m = m.value
    return files[:m], fi[:m], fr[:m]


def group_files(files, fi, fr, node_source, size_mb, score):
    """nerrf_incident_group -> (inc_int int64 [k, 7], inc_real float64 [k, 4], grouped_files int32 [m],
    file_incident int32 [m]) CUDA tensors"""
    dev = files.device
    m = int(files.numel())
    need = C.c_size_t()
    L.check(L.lib().nerrf_incident_group_workspace_bytes(m, C.byref(need)), "nerrf_incident_group_workspace_bytes")
    ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
    k = torch.zeros(1, dtype=torch.int32, device=dev)
    ii = torch.empty(max(m, 1), 7, dtype=torch.int64, device=dev)
    ir = torch.empty(max(m, 1), 4, dtype=torch.float64, device=dev)
    grouped = torch.empty(max(m, 1), dtype=torch.int32, device=dev)
    fin = torch.empty(max(m, 1), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        L.check(L.lib().nerrf_incident_group(L.ptr(files), L.ptr(fi), L.ptr(fr), m, L.ptr(node_source), L.ptr(size_mb), L.ptr(score),
                                             L.ptr(k), L.ptr(ii), L.ptr(ir), L.ptr(grouped), L.ptr(fin), L.ptr(ws), ws.numel(),
                                             L.current_stream_ptr()), "nerrf_incident_group")
    k = int(k.item())
    return ii[:k], ir[:k], grouped[:m], fin[:m]


def incidents(g, node_score, tau=0.5, seeds=None, edge_attack=None, host_names=None, return_files=False):
    """The incidents of window graph `g` (DESIGN.md 1.4) for node scores `node_score` (fp32 [N]): files with a score
    >= tau, plus the file nodes `seeds`, grouped by (host, owning process).  edge_attack: P(attack) [E] per CSR edge
    (the edge head): owners by the edge rule instead of the last writer.  host_names: source id -> host name; given, or when
    g.meta["node_source"] holds a source other than 0, ids are prefixed "host/" (the decimal source id without names).
    -> a list of records ordered by (onset, host, owner; unattributed last):
        {"id", "host" (None with one source), "process" (owner name or None), "owner" (node id, -1), "files" (node ids,
         ascending), "n_files", "onset" / "end" (trace-clock seconds), "onset_event" / "end_event" (event_info records),
         "size_mb", "later_other_events", "max_score"}
    return_files=True: also {node id: {"incident": id, "onset", "event": record, "later"}} for every flagged file.
    Names and events are resolved in one g.meta["event_info"] call.  CUDA tensors only (g.rowptr, g.col on the device)."""
    rowptr, col = g.rowptr, g.col
    if not (torch.is_tensor(rowptr) and rowptr.is_cuda and torch.is_tensor(col) and col.is_cuda):
        raise L.NerrfError("incidents takes a graph of CUDA tensors (no CPU fallback)")
    dev = rowptr.device
    kind_h = np.asarray(g.meta["node_kind"])
    n = rowptr.numel() - 1
    if seeds is not None:
        s = np.asarray(seeds, np.int64).reshape(-1)
        if s.size and (s.min() < 0 or s.max() >= n):
            raise ValueError("incidents: seed node ids must lie in [0, %d)" % n)
        if s.size and np.any(kind_h[s] != 0):
            raise ValueError("incidents: a seed is not a file node")
    kind = torch.from_numpy(kind_h.astype(np.int8)).to(dev)
    score = torch.as_tensor(node_score).to(device=dev, dtype=torch.float32).contiguous()
    ea = None if edge_attack is None else torch.as_tensor(edge_attack).to(device=dev, dtype=torch.float32).contiguous()
    et = _meta_array(g, "edge_time", dev, torch.float64)
    ev = _meta_array(g, "edge_event", dev, torch.int64)
    files, fi, fr = flag_files(rowptr, col.contiguous(), kind, score, tau, seeds, ea, et, ev)
    src_h = g.meta.get("node_source")
    src = None if src_h is None else torch.from_numpy(np.asarray(src_h, np.int64).astype(np.int32)).to(dev)
    size = torch.as_tensor(np.asarray(g.meta.get("size_mb", np.zeros(n, np.float32)), np.float32)).to(dev)
    ii, ir, grouped, fin = group_files(files, fi, fr, src, size, score)
    return records(g, files.cpu().numpy(), fi.cpu().numpy(), fr.cpu().numpy(), ii.cpu().numpy(), ir.cpu().numpy(),
                   grouped.cpu().numpy(), fin.cpu().numpy(), host_names, return_files)


def _num(x):
    return None if math.isnan(x) else float(x)


def records(g, files, fi, fr, ii, ir, grouped, fin, host_names=None, return_files=False):
    """host records of the kernels' outputs (numpy): names and events in one event_info call"""
    src_h = g.meta.get("node_source")
    multi = host_names is not None or (src_h is not None and len(src_h) > 0 and int(np.max(src_h)) > 0)
    info, names = g.meta.get("event_info"), g.meta.get("names")
    ids = sorted({int(e) for e in np.concatenate([ii[:, 4], ii[:, 5], fi[:, 4]]) if e >= 0})
    rec = dict(zip(ids, info(np.asarray(ids, np.int64)))) if (info is not None and ids) else {}
    owners = sorted({int(o) for o in ii[:, 1] if o >= 0})
    nm = dict(zip(owners, names.take(owners) if hasattr(names, "take") else [names[i] for i in owners])) if names is not None else {}
    out = []
    for r in range(ii.shape[0]):
        src, own, off, cnt = (int(v) for v in ii[r, :4])
        host = None
        if multi:
            host = host_names[src] if host_names is not None and src < len(host_names) else str(src)
        pname = None if own < 0 else nm.get(own, "node:%d" % own)
        out.append({"id": incident_id(pname, src, host_names, multi), "host": host, "process": pname, "owner": own,
                    "files": [int(v) for v in grouped[off:off + cnt]], "n_files": cnt,
                    "onset": _num(ir[r, 0]), "onset_event": rec.get(int(ii[r, 4])), "end": _num(ir[r, 1]),
                    "end_event": rec.get(int(ii[r, 5])), "size_mb": float(ir[r, 2]), "later_other_events": int(ii[r, 6]),
                    "max_score": _num(ir[r, 3])})
    if not return_files:
        return out
    per_file = {int(v): {"incident": out[int(fin[i])]["id"], "onset": _num(fr[i, 0]),
                         "event": rec.get(int(fi[i, 4])), "later": int(fi[i, 3])}
                for i, v in enumerate(files.tolist())}
    return out, per_file
