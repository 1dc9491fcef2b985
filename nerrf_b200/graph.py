"""Host-side temporal dependency graph: synthetic generator, trace -> CSR loader, 1-D sharding.

Reference anchors (prose only -- the reference ships no graph constructor, SURVEY.md 2 row 5):
  * window 30-60 s, merge by path/inode, edge weight = causality confidence
                                                docs/content/docs/architecture.mdx:32-42
  * node JSON schema (type, read/write/rename counts, anomaly_score)
                                                docs/content/docs/architecture.mdx:144-160
  * node / edge kinds, per-node features        docs/content/docs/threat-model.mdx:154-184
  * input event schemas: proto/trace.proto:11-49 (Event), and the simulator's TRACE json
    lines benchmarks/m1/scripts/sim_lockbit_m1.py:24-36 (timestamp,event,path,size,pid,...)

Layout handed to the kernels (CSR by DESTINATION):
    rowptr int32|int64 [N+1]; col int32 [E] = source ids, time-sorted within a row;
    ew fp32 [E] = conf_e * exp(-(t_ref - t_e)/tau)   (the "T" of GraphSAGE-T, host-computed).
"""
from __future__ import annotations

import json
import math
from dataclasses import dataclass
from datetime import datetime

import numpy as np

F_IN = 32          # padded node feature width (SURVEY.md 8a a1)
TAU = 30.0         # seconds
WINDOW = 60.0      # seconds
# Linux's cap on what one read / write can transfer.  An event's byte count is the count ARGUMENT of write(2), traced
# before the call fails, so the traced process can put any uint64 there; every feature clamps it to this first.
MAX_RW_COUNT = 0x7ffff000


def clamp_bytes(size) -> int:
    """An event's byte count as the features see it: the wire's uint64 clamped to MAX_RW_COUNT (a Python int)."""
    return min(int(size or 0), MAX_RW_COUNT)


@dataclass
class TemporalGraph:
    rowptr: np.ndarray      # int32 (int64 when E >= 2**31) [N+1]
    col: np.ndarray         # int32 [E]
    ew: np.ndarray          # fp32 [E]
    x: np.ndarray           # fp32 [N, F_IN]
    meta: dict

    @property
    def num_nodes(self):
        return self.rowptr.shape[0] - 1

    @property
    def num_edges(self):
        return self.col.shape[0]


def csr_from_edges(src, dst, t, conf, N, t_ref=WINDOW, tau=TAU):
    """Sort edges by (dst, t) and build CSR-by-destination with temporal weights."""
    order = np.lexsort((t, dst))
    src = src[order]; dst = dst[order]; t = t[order]; conf = conf[order]
    counts = np.bincount(dst, minlength=N)
    E = src.shape[0]
    rp_dtype = np.int64 if E >= 2 ** 31 else np.int32
    rowptr = np.zeros(N + 1, dtype=rp_dtype)
    np.cumsum(counts, out=rowptr[1:])
    ew = (conf.astype(np.float32) * np.exp(-(np.float32(t_ref) - t.astype(np.float32)) / np.float32(tau))).astype(np.float32)
    return rowptr, src.astype(np.int32), ew


def build_csr_device(src, dst, t, conf, N, t_ref=WINDOW, tau=TAU, rowptr_dtype=None, return_perm=False):
    """Device half of the graph constructor (include/nerrf_b200.h nerrf_graph_build_csr): CUDA int32 src/dst and
    fp32 t/conf tensors -> (rowptr, col, ew) CUDA tensors, same contract as csr_from_edges (rowptr/col bit-exact,
    ew within the exp implementation's 2 ulp).  No CPU fallback."""
    import ctypes as C
    import torch
    from . import _lib
    _lib.require_cuda(src, dst, t, conf)
    E = int(src.shape[0])
    if not (dst.shape[0] == t.shape[0] == conf.shape[0] == E):
        raise ValueError("src, dst, t, conf must have the same length")
    if src.dtype != torch.int32 or dst.dtype != torch.int32 or t.dtype != torch.float32 or conf.dtype != torch.float32:
        raise TypeError("build_csr_device takes int32 src/dst and float32 t/conf")
    src, dst, t, conf = src.contiguous(), dst.contiguous(), t.contiguous(), conf.contiguous()
    dev = src.device
    if rowptr_dtype is None:
        rowptr_dtype = torch.int64 if E >= 2 ** 31 else torch.int32
    h = _lib.lib()
    with torch.cuda.device(dev):
        nbytes = C.c_int64()
        _lib.check(h.nerrf_graph_csr_workspace_bytes(E, int(N), C.byref(nbytes)), "nerrf_graph_csr_workspace_bytes")
        ws = torch.empty(max(nbytes.value, 256), dtype=torch.uint8, device=dev)
        rowptr = torch.empty(int(N) + 1, dtype=rowptr_dtype, device=dev)
        col = torch.empty(E, dtype=torch.int32, device=dev)
        ew = torch.empty(E, dtype=torch.float32, device=dev)
        perm = torch.empty(max(E, 1), dtype=torch.int32, device=dev) if return_perm else None     # uint32 bit patterns
        _lib.check(h.nerrf_graph_build_csr_ex(_lib.ptr(src), _lib.ptr(dst), _lib.ptr(t), _lib.ptr(conf), E, int(N),
                                              float(t_ref), float(tau), _lib.ptr(rowptr), int(rowptr_dtype == torch.int64),
                                              _lib.ptr(col), _lib.ptr(ew), _lib.ptr(perm), _lib.ptr(ws), ws.numel(),
                                              _lib.current_stream_ptr()), "nerrf_graph_build_csr_ex")
    if return_perm:
        return rowptr, col, ew, perm
    return rowptr, col, ew


def edge_labels_device(node_p, node_f, raw_slot, rowptr, col, n_nodes):
    """Device per-pair edge labels (include/nerrf_b200.h nerrf_trace_edge_labels): CUDA int32 node ids per event, uint8
    ANNOTATION event slots, and the graph's CSR -> uint8 [E] in CSR order, the rule of graph_from_events
    meta['edge_label'].  No CPU fallback."""
    import ctypes as C
    import torch
    from . import _lib
    _lib.require_cuda(node_p, node_f, raw_slot, rowptr, col)
    for a, dt in ((node_p, torch.int32), (node_f, torch.int32), (raw_slot, torch.uint8), (col, torch.int32)):
        if a.dtype != dt or not a.is_contiguous():
            raise TypeError(f"edge_labels_device: expected contiguous {dt}, got {a.dtype}")
    if rowptr.dtype not in (torch.int32, torch.int64) or not rowptr.is_contiguous():
        raise TypeError("rowptr must be contiguous int32 / int64")
    n, E, dev = int(node_p.shape[0]), int(col.shape[0]), col.device
    if not (node_f.shape[0] == raw_slot.shape[0] == n and rowptr.shape[0] == int(n_nodes) + 1):
        raise ValueError("node_p / node_f / raw_slot must have one entry per event and rowptr n_nodes + 1")
    h = _lib.lib()
    with torch.cuda.device(dev):
        need = C.c_int64()
        _lib.check(h.nerrf_trace_edge_labels_workspace_bytes(n, C.byref(need)), "nerrf_trace_edge_labels_workspace_bytes")
        ws = torch.empty(need.value + 256, dtype=torch.uint8, device=dev)
        out = torch.empty(E, dtype=torch.uint8, device=dev)
        _lib.check(h.nerrf_trace_edge_labels(_lib.ptr(node_p), _lib.ptr(node_f), _lib.ptr(raw_slot), n, _lib.ptr(rowptr),
                                             int(rowptr.dtype == torch.int64), _lib.ptr(col), E, int(n_nodes), _lib.ptr(out),
                                             C.c_void_p((ws.data_ptr() + 255) & ~255), need.value, _lib.current_stream_ptr()),
                   "nerrf_trace_edge_labels")
    return out


def node_features_device(node_p, node_f, node_g, t, event_slot, nbytes, path_flags, node_kind, window):
    """Device per-node features (include/nerrf_b200.h nerrf_graph_node_features).  CUDA tensors: int32 node ids per
    event (node_g may be None), float64 t (seconds since the first event), uint8 event_slot / path_flags, int64|uint64
    byte counts, int8 node_kind [N].  -> x fp32 [N, 32], label int32 [N], size_mb fp32 [N] (CUDA).  No CPU fallback."""
    import ctypes as C
    import torch
    from . import _lib
    _lib.require_cuda(node_p, node_f, node_g, t, event_slot, nbytes, path_flags, node_kind)
    want = ((node_p, torch.int32), (node_f, torch.int32), (t, torch.float64), (event_slot, torch.uint8),
            (path_flags, torch.uint8), (node_kind, torch.int8))
    for a, dt in want:
        if a.dtype != dt or not a.is_contiguous():
            raise TypeError(f"node_features_device: expected contiguous {dt}, got {a.dtype}")
    if node_g is not None and (node_g.dtype != torch.int32 or not node_g.is_contiguous()):
        raise TypeError("node_g must be contiguous int32")
    if nbytes.dtype not in (torch.int64, torch.uint64) or not nbytes.is_contiguous():
        raise TypeError("nbytes must be contiguous int64 / uint64")
    n, N, dev = int(node_p.shape[0]), int(node_kind.shape[0]), node_p.device
    h = _lib.lib()
    with torch.cuda.device(dev):
        need = C.c_int64()
        _lib.check(h.nerrf_graph_node_features_workspace_bytes(N, C.byref(need)), "nerrf_graph_node_features_workspace_bytes")
        ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
        x = torch.empty(N, F_IN, dtype=torch.float32, device=dev)
        label = torch.empty(N, dtype=torch.int32, device=dev)
        size_mb = torch.empty(N, dtype=torch.float32, device=dev)
        _lib.check(h.nerrf_graph_node_features(_lib.ptr(node_p), _lib.ptr(node_f), _lib.ptr(node_g), _lib.ptr(t),
                                               _lib.ptr(event_slot), _lib.ptr(nbytes), _lib.ptr(path_flags), n,
                                               _lib.ptr(node_kind), N, float(window), _lib.ptr(x), _lib.ptr(label),
                                               _lib.ptr(size_mb), _lib.ptr(ws), ws.numel(), _lib.current_stream_ptr()),
                   "nerrf_graph_node_features")
    return x, label, size_mb


def synthetic_graph(N=1_000_000, E=10_000_000, seed=20250115, hub="src", feat_seed=0, f_in=F_IN) -> TemporalGraph:
    """SURVEY.md 8d cfg 2/4 generator: dst ~ U{0..N-1}, src = floor(N*u^3) (hub sources, one
    ransomware pid touching many files); hub="dst" swaps the roles (long rows)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    uni = rng.integers(0, N, size=E, dtype=np.int64)
    skew = np.minimum((N * rng.random(E) ** 3).astype(np.int64), N - 1)
    src, dst = (skew, uni) if hub == "src" else (uni, skew)
    t = (rng.random(E) * WINDOW).astype(np.float32)
    conf = (0.5 + 0.5 * rng.random(E)).astype(np.float32)
    rowptr, col, ew = csr_from_edges(src, dst, t, conf, N)
    x = np.random.Generator(np.random.PCG64(feat_seed)).standard_normal((N, f_in), dtype=np.float32)
    return TemporalGraph(rowptr, col, ew, x, {"kind": "synthetic", "hub": hub, "seed": seed})


# --------------------------------------------------------------------------- trace -> graph
_EVENT_SLOT = {"file_created": 0, "file_encrypt_start": 1, "file_encrypt_complete": 2,
               "ransom_note_created": 3, "openat": 4, "write": 5, "rename": 6}
_N_EVENT_SLOTS = 8        # slot 7 = any other event kind
ATTACK_EVENTS = ("file_encrypt_start", "file_encrypt_complete", "ransom_note_created")


def _parse_ts(s):
    if isinstance(s, (int, float)):
        return float(s)
    return datetime.fromisoformat(s.replace("Z", "")).timestamp()


def _stem(path: str) -> str:
    """Merge key for a file and its renamed/encrypted twin (x.dat <-> x.lockbit3):
    the graph constructor 'merges by inode' (architecture.mdx:41); traces carry no inode for
    the simulator events, so the extension-less path is the stand-in identity."""
    slash = path.rfind("/")
    dot = path.rfind(".")
    return path[:dot] if dot > slash else path


def read_trace_jsonl(path):
    with open(path) as f:
        return [json.loads(line) for line in f if line.strip()]


def events_from_event_batch(batch) -> list:
    """nerrf.trace.EventBatch (proto/trace.proto:47-49) -> the same dict schema as the JSONL
    traces.  `batch` is any object with .events each having ts/pid/syscall/path/new_path/bytes."""
    out = []
    for e in batch.events:
        ts = e.ts.seconds + e.ts.nanos * 1e-9 if hasattr(e.ts, "seconds") else float(e.ts)
        out.append({"timestamp": ts, "event": e.syscall, "path": e.path, "size": int(e.bytes),
                    "pid": int(e.pid), "new_path": getattr(e, "new_path", "")})
    return out


# Observable-only event kinds: the simulator's annotations (file_created, file_encrypt_*, ransom_note_created) are
# ground truth, not something the tracker can see -- it emits openat / write / rename only
# (tracker/bpf/tracepoints.c:43-81).  `observable=True` folds every simulator kind onto the syscall it stands for,
# so features built from simulator traces equal the features a wire-format trace of the same activity would give;
# labels keep using the annotations.
OBSERVABLE_SLOT = (4, 5, 6, 4, 4, 5, 6, 7)   # created->openat, encrypt_start->write, encrypt_complete->rename, note->openat


def resolve_event_paths(events) -> list:
    """Time-sorted copy of `events` in which every event names a file.  Real tracker traces carry no path on write
    events (tracker/bpf/tracepoints.c:62-64 zeroes it): such an event is attributed to the most recent non-empty path
    of the same pid (the file it has open, as far as the trace can tell); with no such path it identifies no file and is
    dropped.  Without this every path-less event of every process would be interned as ONE file node named ''."""
    evs = sorted(events, key=lambda e: _parse_ts(e["timestamp"]))     # lossy streams may be unordered
    last: dict = {}
    out = []
    for e in evs:
        if e.get("path"):
            last[e["pid"]] = e["path"]
            out.append(e)
        elif e["pid"] in last:
            d = dict(e); d["path"] = last[e["pid"]]; d["path_inferred"] = True
            out.append(d)
    return out


def graph_from_events(events, merge_renames=True, window=None, observable=False) -> TemporalGraph:
    """Events -> temporal graph.  Nodes: one per pid (process) and one per file identity.
    Edges (both directions, so files aggregate from the process that touched them and the
    process from its files): process<->file per event with time t_e and conf_e = 1; rename /
    encrypt pairs are merged into one file node when merge_renames (else linked file<->file).
    meta['edge_label'] (uint8 [E], CSR order): 1 on both edges of a process <-> file pair iff that process emitted an
    ATTACK_EVENTS event on that file; 0 elsewhere (rename links included)."""
    evs = resolve_event_paths(events)
    if not evs:
        raise ValueError("empty trace")
    t0 = _parse_ts(evs[0]["timestamp"]); t1 = _parse_ts(evs[-1]["timestamp"])
    span = max(t1 - t0, 1e-6)
    window = window or max(span, WINDOW)
    node_id: dict = {}
    names: list = []
    kinds: list = []

    def nid(key, kind, name):
        if key not in node_id:
            node_id[key] = len(names); names.append(name); kinds.append(kind)
        return node_id[key]

    src, dst, tt, eid = [], [], [], []
    feats: dict = {}
    labels: dict = {}
    attack_pairs: set = set()          # (process, file) pairs with an ATTACK_EVENTS event of that process on that file
    for i_ev, e in enumerate(evs):
        t = _parse_ts(e["timestamp"]) - t0
        p = nid(("p", e["pid"]), 1, f"pid:{e['pid']}")
        path = e["path"]
        key = ("f", _stem(path) if merge_renames else path)
        f = nid(key, 0, path)
        if path.endswith(".lockbit3"):
            names[f] = path                       # keep the encrypted name: the rollback target
        src += [p, f]; dst += [f, p]; tt += [t, t]; eid += [i_ev, i_ev]
        touched = [p, f]
        new_path = e.get("new_path") or ""
        if new_path and merge_renames:
            # a real rename `a.dat -> a.dat.lockbit3`: the target is the SAME file identity (merge by inode), whatever
            # its stem; later events on the new name land on this node, and the encrypted name is the rollback target
            node_id.setdefault(("f", _stem(new_path)), f)
            if new_path.endswith(".lockbit3"):
                names[f] = new_path
        if new_path and not merge_renames:
            g = nid(("f", new_path), 0, new_path)
            src += [f, g]; dst += [g, f]; tt += [t, t]; eid += [i_ev, i_ev]
            touched.append(g)
        for n in touched:
            fv = feats.setdefault(n, {"cnt": np.zeros(_N_EVENT_SLOTS), "bytes": 0, "first": t, "last": t,
                                       "lockbit": 0.0, "note": 0.0, "tmp": 0.0})
            slot = _EVENT_SLOT.get(e["event"], _N_EVENT_SLOTS - 1)
            fv["cnt"][OBSERVABLE_SLOT[slot] if observable else slot] += 1
            fv["bytes"] += clamp_bytes(e.get("size", 0))      # an exact integer sum, converted to float once below
            fv["last"] = t
        fv = feats[f]
        fv["lockbit"] = max(fv["lockbit"], 1.0 if ".lockbit" in path or (merge_renames and ".lockbit" in new_path) else 0.0)
        fv["note"] = max(fv["note"], 1.0 if "README" in path.upper() or "RANSOM" in path.upper() else 0.0)
        fv["tmp"] = max(fv["tmp"], 1.0 if path.startswith("/tmp") or path.startswith("/proc") else 0.0)
        if e["event"] in ATTACK_EVENTS:
            attack_pairs.add((p, f))
        attacked = e["event"] in ATTACK_EVENTS or e.get("phase") == "attack" and e["event"].startswith("file_encrypt")
        labels[f] = max(labels.get(f, 0), 1 if (attacked and e["event"] != "ransom_note_created"
                                                 and e["event"].startswith("file_encrypt")) else 0)
    N = len(names)
    src = np.asarray(src, np.int64); dst = np.asarray(dst, np.int64)
    tt = np.asarray(tt, np.float32)
    conf = np.ones(src.shape[0], np.float32)
    rowptr, col, ew = csr_from_edges(src, dst, tt, conf, N, t_ref=float(span), tau=TAU)
    # per-pair edge labels in CSR order (the edge head sees only [h_src || h_dst], the same for every event of a pair):
    # 1 in both directions iff the process attacked the file; file <-> file rename links are 0
    pair = src * N + dst
    hit = np.asarray([p_ * N + f_ for p_, f_ in attack_pairs] + [f_ * N + p_ for p_, f_ in attack_pairs], np.int64)
    edge_label = np.isin(pair, hit).astype(np.uint8)[np.lexsort((tt, dst))]
    indeg = np.bincount(dst, minlength=N).astype(np.float32)
    outdeg = np.bincount(src, minlength=N).astype(np.float32)
    x = np.zeros((N, F_IN), np.float32)
    for n in range(N):
        fv = feats[n]
        x[n, 0] = 1.0 if kinds[n] == 0 else 0.0         # file
        x[n, 1] = 1.0 if kinds[n] == 1 else 0.0         # process   (x[:,2] = socket, unused here)
        x[n, 3] = math.log1p(indeg[n]); x[n, 4] = math.log1p(outdeg[n])
        x[n, 5:5 + _N_EVENT_SLOTS] = np.log1p(fv["cnt"])
        x[n, 13] = math.log1p(float(fv["bytes"])) / 20.0
        x[n, 14] = (fv["last"] - fv["first"]) / window   # temporal delta
        x[n, 15] = fv["first"] / window
        x[n, 16] = fv["lockbit"]; x[n, 17] = fv["note"]; x[n, 18] = fv["tmp"]
        wr = fv["cnt"][1] + fv["cnt"][5]
        x[n, 19] = fv["cnt"][2] / wr if wr > 0 else 0.0   # "byte count ratio" proxy: completes / starts
    y = np.zeros(N, np.int64)
    for n, v in labels.items():
        y[n] = v
    size_mb = np.zeros(N, np.float32)
    for n in range(N):
        c = feats[n]["cnt"]
        k = max(c[0] + c[1] + c[2], 1.0)
        size_mb[n] = float(feats[n]["bytes"]) / k / 1e6 if kinds[n] == 0 else 0.0
    file_keys = {k[1]: v for k, v in node_id.items() if k[0] == "f"}      # merge key (or path) -> node, incl. rename aliases
    # edge_event: the event (index into the time-sorted, path-resolved events) that made each CSR edge
    edge_event = np.asarray(eid, np.int64)[np.lexsort((tt, dst))]
    # edge_time: the trace-clock seconds of that event (float64, the time event_info reports), computed when asked for
    edge_time = lambda: np.asarray([_parse_ts(e["timestamp"]) for e in evs], np.float64)[edge_event]
    # edge_flow: the information-flow class of that event (DESIGN.md 1.5; the raw kind, not the observable fold)
    edge_flow = lambda: event_flow([_EVENT_SLOT.get(e["event"], _N_EVENT_SLOTS - 1) for e in evs],
                                   [int(e.get("flags", 0)) for e in evs], [int(e.get("ret_val", 0)) for e in evs])[edge_event]
    return TemporalGraph(rowptr, col, ew, x, {"kind": "trace", "names": names, "node_kind": np.asarray(kinds),
                                              "label": y, "size_mb": size_mb, "t0": t0, "span": span,
                                              "file_keys": file_keys, "merge_renames": bool(merge_renames),
                                              "edge_label": edge_label, "edge_event": edge_event, "edge_time": edge_time,
                                              "edge_flow": edge_flow,
                                              "event_info": lambda ids: [event_record(evs[int(i)]) for i in ids]})


def event_flow(event_slot, flags, ret_val) -> np.ndarray:
    """uint8 flow class of every event (DESIGN.md 1.5: bit 0 process -> file, bit 1 file -> process) from its raw event
    slot, open flags and return value, by the library's one definition of the table (nerrf_trace_flow_class)"""
    slot = np.ascontiguousarray(event_slot, np.uint8)
    fl = np.ascontiguousarray(flags, np.int64)
    rv = np.ascontiguousarray(ret_val, np.int64)
    import ctypes
    from . import _lib
    out = np.zeros(slot.shape[0], np.uint8)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    _lib.check(_lib.lib().nerrf_trace_flow_class(p(slot), p(fl), p(rv), slot.shape[0], p(out)), "nerrf_trace_flow_class")
    return out


def event_record(e) -> dict:
    """The fields of one event an explanation shows: time (seconds), pid, syscall, path (resolved)"""
    return {"time": _parse_ts(e["timestamp"]), "pid": int(e["pid"]), "syscall": str(e["event"]), "path": str(e["path"])}


def graph_from_jsonl(path, **kw) -> TemporalGraph:
    return graph_from_events(read_trace_jsonl(path), **kw)


def replicate_events(events, k, dt=0.0):
    """Amplify a trace k times with pid/path renaming (SURVEY.md 8d cfg 1/5)."""
    out = []
    for i in range(k):
        for e in events:
            d = dict(e)
            d["pid"] = int(e["pid"]) + 100000 * i
            slash = e["path"].rfind("/")
            d["path"] = e["path"][:slash + 1] + (f"r{i}_" if i else "") + e["path"][slash + 1:] if slash >= 0 else e["path"]
            if dt:
                d["timestamp"] = _parse_ts(e["timestamp"]) + dt * i
            out.append(d)
    return out


# --------------------------------------------------------------------------- sharding
def edge_balanced_row_cuts(rowptr, parts):
    """1-D edge-block shards with ROW-ALIGNED cuts (SURVEY.md 8e): returns row boundaries
    [parts+1]; shard g owns destination rows [cuts[g], cuts[g+1]) and hence the contiguous edge
    block [rowptr[cuts[g]], rowptr[cuts[g+1]])."""
    N = rowptr.shape[0] - 1
    E = int(rowptr[-1])
    targets = (np.arange(1, parts, dtype=np.float64) * (E / parts))
    cuts = np.searchsorted(np.asarray(rowptr[1:-1], dtype=np.int64), targets, side="left") + 1 if N > 1 else np.zeros(parts - 1, np.int64)
    cuts = np.concatenate([[0], np.minimum(cuts, N), [N]]).astype(np.int64)
    return np.maximum.accumulate(cuts)
