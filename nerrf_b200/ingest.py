"""EventBatch ingest and the columnar graph constructor (SURVEY.md 8f ranks 2 and 1, host side).

    wire bytes of nerrf.trace.EventBatch  --decode_event_batch-->  EventColumns (numpy, columnar)
    EventColumns  --graph_from_columns-->  TemporalGraph        (same graph as graph.graph_from_events, no per-event
                                                                  Python: interning in C++, everything else vectorised;
                                                                  device=... runs the sort/CSR stage on the GPU)

Reference anchors: proto/trace.proto:11-49 (Event), :47-49 (EventBatch), producer
tracker/cmd/tracker/main.go:229-252; constructor prose docs/content/docs/architecture.mdx:32-42,144-160.
The decoder and the interning live in the C-ABI library (csrc/ingest.cu: nerrf_trace_scan / _decode / _intern).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _lib
from . import graph as G

STRING_COLUMNS = ("comm", "syscall", "path", "new_path")


@dataclass
class EventColumns:
    n: int
    ts_sec: np.ndarray        # int64  [n]   google.protobuf.Timestamp.seconds
    ts_nanos: np.ndarray      # int32  [n]
    pid: np.ndarray           # uint32 [n]
    tid: np.ndarray           # uint32 [n]
    flags: np.ndarray         # int32  [n]   Event.OpenFlags
    ret_val: np.ndarray       # int64  [n]
    bytes: np.ndarray         # uint64 [n]
    event_slot: np.ndarray    # uint8  [n]   feature slot of the syscall / event name (graph._EVENT_SLOT, 7 = other)
    path_flags: np.ndarray    # uint8  [n]   NERRF_PATH_* bits
    strings: dict             # name -> (offsets int64 [n+1], data uint8 [bytes])
    source: np.ndarray = None  # uint16 [n] source id of each event (the host whose tracker sent it); None = all source 0

    def text(self, column: str, i: int) -> str:
        off, data = self.strings[column]
        return bytes(data[off[i]:off[i + 1]]).decode("utf-8", "replace")

    def texts(self, column: str) -> list:
        off, data = self.strings[column]
        raw = data.tobytes()
        return [raw[off[i]:off[i + 1]].decode("utf-8", "replace") for i in range(self.n)]

    @property
    def timestamp(self) -> np.ndarray:
        """seconds as float64, the same arithmetic as graph.events_from_event_batch (seconds + nanos * 1e-9)."""
        return self.ts_sec.astype(np.float64) + self.ts_nanos.astype(np.float64) * 1e-9


def _p(a):
    return C.c_void_p(a.ctypes.data)


def decode_event_batch(buf) -> EventColumns:
    """buf: bytes / bytearray / memoryview / uint8 array holding one serialized EventBatch (or several concatenated)."""
    raw = np.frombuffer(buf, dtype=np.uint8) if not isinstance(buf, np.ndarray) else np.ascontiguousarray(buf, np.uint8)
    h = _lib.lib()
    n = C.c_int64()
    sb = (C.c_int64 * 4)()
    _lib.check(h.nerrf_trace_scan(_p(raw) if raw.size else None, raw.size, C.byref(n), sb), "nerrf_trace_scan")
    n = n.value
    cols = dict(ts_sec=np.empty(n, np.int64), ts_nanos=np.empty(n, np.int32), pid=np.empty(n, np.uint32),
                tid=np.empty(n, np.uint32), flags=np.empty(n, np.int32), ret_val=np.empty(n, np.int64),
                bytes=np.empty(n, np.uint64), event_slot=np.empty(n, np.uint8), path_flags=np.empty(n, np.uint8))
    strings = {name: (np.zeros(n + 1, np.int64), np.empty(max(int(sb[k]), 1), np.uint8)) for k, name in enumerate(STRING_COLUMNS)}   # upper bounds
    args = [_p(cols[k]) for k in ("ts_sec", "ts_nanos", "pid", "tid", "flags", "ret_val", "bytes", "event_slot", "path_flags")]
    for name in STRING_COLUMNS:
        args += [_p(strings[name][0]), _p(strings[name][1])]
    _lib.check(h.nerrf_trace_decode(_p(raw) if raw.size else None, raw.size, n, *args), "nerrf_trace_decode")
    strings = {name: (off, data[:off[-1]].copy()) for name, (off, data) in strings.items()}
    return EventColumns(n=n, strings=strings, **cols)


def _frame(raw: np.ndarray, partial: bool):
    """nerrf_trace_frame -> (error offset or None, rec_at, body_off, body_len, consumed).  On a malformed record the
    arrays still hold the records before it."""
    h = _lib.lib()
    cap = raw.size // 16 + 16
    while True:
        rec = np.empty((3, cap), np.int64)
        n, consumed = C.c_int64(), C.c_int64()
        rc = h.nerrf_trace_frame(_p(raw) if raw.size else None, raw.size, int(bool(partial)), cap, _p(rec[0]), _p(rec[1]),
                                 _p(rec[2]), C.byref(n), C.byref(consumed))
        if n.value <= cap:
            break
        cap = n.value
    if rc != 0 and not h.nerrf_last_error().decode().startswith("malformed"):
        _lib.check(rc, "nerrf_trace_frame")
    m = n.value
    return (consumed.value if rc != 0 else None), rec[0, :m], rec[1, :m], rec[2, :m], consumed.value


def frame_event_batch(buf, partial=False):
    """Top-level framing of EventBatch wire bytes (nerrf_trace_frame): -> (rec_at, body_off, body_len, consumed), one
    entry per Event record.  partial=True: a cut-off trailing record is not an error; `consumed` stops before it."""
    raw = np.frombuffer(buf, dtype=np.uint8) if not isinstance(buf, np.ndarray) else np.ascontiguousarray(buf, np.uint8)
    bad, rec_at, body_off, body_len, consumed = _frame(raw, partial)
    if bad is not None:
        raise _lib.NerrfError(f"nerrf_trace_frame failed: malformed EventBatch at byte offset {bad}")
    return rec_at, body_off, body_len, consumed


def events_from_columns(cols: EventColumns) -> list:
    """The dict schema of graph.events_from_event_batch / the JSONL traces (for the per-event host loader)."""
    ts = cols.timestamp
    sys_, path, new_path = cols.texts("syscall"), cols.texts("path"), cols.texts("new_path")
    return [{"timestamp": float(ts[i]), "event": sys_[i], "path": path[i], "size": int(cols.bytes[i]),
             "pid": int(cols.pid[i]), "new_path": new_path[i]} for i in range(cols.n)]


def column_event_records(cols: EventColumns, ids) -> list:
    """graph.event_record of rows `ids` of `cols`, plus "source" when the columns carry one"""
    ts = cols.timestamp
    out = []
    for i in np.asarray(ids, np.int64).tolist():
        txt = {}
        for name in ("syscall", "path"):
            off, data = cols.strings[name]
            txt[name] = bytes(data[off[i]:off[i + 1]]).decode("utf-8", "replace")
        r = {"time": float(ts[i]), "pid": int(cols.pid[i]), "syscall": txt["syscall"], "path": txt["path"]}
        if cols.source is not None:
            r["source"] = int(cols.source[i])
        out.append(r)
    return out


def _gather_strings(off, data, idx):
    """Packed string column restricted / re-ordered to rows `idx` (vectorised variable-length gather)."""
    ln = (off[idx + 1] - off[idx]).astype(np.int64)
    new_off = np.zeros(idx.shape[0] + 1, np.int64)
    np.cumsum(ln, out=new_off[1:])
    total = int(new_off[-1])
    if total == 0:
        return new_off, np.zeros(0, np.uint8)
    pos = np.arange(total, dtype=np.int64) - np.repeat(new_off[:-1], ln) + np.repeat(off[idx], ln)
    return new_off, data[pos]


def process_keys(cols: EventColumns) -> np.ndarray:
    """uint64 [n] process identity of every event: (source << 32) | pid (the pid alone without a source column)"""
    key = cols.pid.astype(np.uint64)
    if cols.source is not None:
        key |= cols.source.astype(np.uint64) << np.uint64(32)
    return key


def resolve_columns(cols: EventColumns) -> EventColumns:
    """Columnar form of graph.resolve_event_paths: every event must name a file.  The tracker zeroes `path` on write
    events (tracker/bpf/tracepoints.c:62-64); such an event takes the most recent non-empty path of the same process
    -- (source, pid) -- in time order, or is dropped when there is none.  Returns `cols` itself when no path is empty."""
    poff, pdata = cols.strings["path"]
    empty = (poff[1:] - poff[:-1]) == 0
    if cols.n == 0 or not empty.any():
        return cols
    order = np.argsort(cols.timestamp, kind="stable")
    key = process_keys(cols)
    by_pid = order[np.argsort(key[order], kind="stable")]               # grouped by process, time order inside a group
    pid_g = key[by_pid]
    start = np.r_[True, pid_g[1:] != pid_g[:-1]]
    grp_first = np.maximum.accumulate(np.where(start, np.arange(cols.n), 0))
    have = np.where(~empty[by_pid], np.arange(cols.n), -1)
    last = np.maximum.accumulate(have)                                  # position of the last named event so far ...
    ok = last >= grp_first                                              # ... if it belongs to the same pid
    src = np.empty(cols.n, np.int64)                                    # event whose path this event uses, by stored index
    src[by_pid] = np.where(ok, by_pid[np.maximum(last, 0)], -1)
    keep = np.nonzero(src >= 0)[0]                                      # stored order is preserved for the survivors
    strings = {name: _gather_strings(*cols.strings[name], keep) for name in STRING_COLUMNS if name != "path"}
    strings["path"] = _gather_strings(poff, pdata, src[keep])
    sc = {k: getattr(cols, k)[keep] for k in ("ts_sec", "ts_nanos", "pid", "tid", "flags", "ret_val", "bytes", "event_slot")}
    return EventColumns(n=int(keep.shape[0]), path_flags=cols.path_flags[src[keep]], strings=strings,
                        source=None if cols.source is None else cols.source[keep], **sc)


def path_flags_of(off, data) -> np.ndarray:
    """NERRF_PATH_* bits of a packed string column (nerrf_trace_path_flags)."""
    n = off.shape[0] - 1
    out = np.zeros(max(n, 1), np.uint8)
    d = data if data.size else np.zeros(1, np.uint8)
    _lib.check(_lib.lib().nerrf_trace_path_flags(_p(off), _p(d), n, _p(out)), "nerrf_trace_path_flags")
    return out[:n]


def intern_nodes(cols: EventColumns, order=None, merge_renames=True):
    """-> node_p, node_f, node_g (int32 [n], by stored event index; node_g = -1 when absent), kind int8 [N],
    name_event int64 [N], name_which int8 [N]."""
    n = cols.n
    cap = max((2 if merge_renames else 3) * n, 1)
    node_p = np.zeros(n, np.int32); node_f = np.zeros(n, np.int32); node_g = np.zeros(n, np.int32)
    kind = np.zeros(cap, np.int8); name_event = np.zeros(cap, np.int64); name_which = np.zeros(cap, np.int8)
    nn = C.c_int64()
    order_p = None
    if order is not None:
        order = np.ascontiguousarray(order, np.int64)
        order_p = _p(order)
    (poff, pdata), (goff, gdata) = cols.strings["path"], cols.strings["new_path"]
    pdata = pdata if pdata.size else np.zeros(1, np.uint8)
    gdata = gdata if gdata.size else np.zeros(1, np.uint8)
    src = None if cols.source is None else np.ascontiguousarray(cols.source, np.uint16)
    _lib.check(_lib.lib().nerrf_trace_intern_ex(n, order_p, _p(cols.pid), None if src is None else _p(src), _p(poff), _p(pdata),
                                                _p(goff), _p(gdata), int(bool(merge_renames)), _p(node_p), _p(node_f), _p(node_g),
                                                C.byref(nn), _p(kind), _p(name_event), _p(name_which), cap), "nerrf_trace_intern_ex")
    N = nn.value
    return node_p, node_f, node_g, kind[:N].copy(), name_event[:N].copy(), name_which[:N].copy()


def intern_nodes_device(cols: EventColumns, order=None, merge_renames=True, device="cuda", return_device=False):
    """`intern_nodes` on the GPU (nerrf_trace_intern_device, csrc/intern_device.cu: hash table + rename-alias forest +
    creating-mention scan): the same six arrays for the same events in the same processing order.  The pid / path /
    new_path columns are uploaded here; return_device=True leaves node_p / node_f / node_g on the device (torch
    tensors) for the feature / CSR kernels that consume them there."""
    import torch
    dev = torch.device(device)
    n = cols.n
    cap = max((2 if merge_renames else 3) * n, 1)
    up = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)
    (poff, pdata), (goff, gdata) = cols.strings["path"], cols.strings["new_path"]
    d_pid = up(cols.pid.view(np.int32) if cols.pid.dtype == np.uint32 else cols.pid.astype(np.uint32).view(np.int32), np.int32)
    d_poff, d_goff = up(poff, np.int64), up(goff, np.int64)
    d_pdata = up(pdata if pdata.size else np.zeros(1, np.uint8), np.uint8)
    d_gdata = up(gdata if gdata.size else np.zeros(1, np.uint8), np.uint8)
    d_order = None if order is None else up(order, np.int64)
    d_src = None if cols.source is None else up(cols.source.astype(np.uint16).view(np.int16), np.int16)
    node_p = torch.empty(max(n, 1), dtype=torch.int32, device=dev); node_f = torch.empty_like(node_p); node_g = torch.empty_like(node_p)
    kind = torch.zeros(cap, dtype=torch.int8, device=dev); name_event = torch.zeros(cap, dtype=torch.int64, device=dev)
    name_which = torch.zeros(cap, dtype=torch.int8, device=dev)
    need = C.c_int64()
    _lib.check(_lib.lib().nerrf_trace_intern_device_workspace_bytes(n, cap, C.byref(need)), "intern_device_workspace_bytes")
    ws = torch.empty(need.value + 256, dtype=torch.uint8, device=dev)
    ws_ptr = (ws.data_ptr() + 255) & ~255
    nn = C.c_int64()
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().nerrf_trace_intern_device_ex(n, n, _lib.ptr(d_order), _lib.ptr(d_pid), _lib.ptr(d_src), _lib.ptr(d_poff),
                                                           _lib.ptr(d_pdata), _lib.ptr(d_goff), _lib.ptr(d_gdata), int(bool(merge_renames)),
                                                           _lib.ptr(node_p), _lib.ptr(node_f), _lib.ptr(node_g), C.byref(nn),
                                                           _lib.ptr(kind), _lib.ptr(name_event), _lib.ptr(name_which), cap,
                                                           C.c_void_p(ws_ptr), need.value, _lib.current_stream_ptr()),
                   "nerrf_trace_intern_device_ex")
    N = nn.value
    host = lambda t_: t_.cpu().numpy()
    if return_device:
        return node_p[:n], node_f[:n], node_g[:n], host(kind[:N]), host(name_event[:N]), host(name_which[:N])
    return host(node_p[:n]), host(node_f[:n]), host(node_g[:n]), host(kind[:N]), host(name_event[:N]), host(name_which[:N])


def _node_names(cols, name_event, name_which):
    """pid nodes -> "pid:<pid>"; file nodes -> the path (or new_path) of the event that names them."""
    (poff, pdata), (goff, gdata) = cols.strings["path"], cols.strings["new_path"]
    praw, graw = pdata.tobytes(), gdata.tobytes()
    pa, pb = poff[name_event].tolist(), poff[name_event + 1].tolist()
    ga, gb = goff[name_event].tolist(), goff[name_event + 1].tolist()
    pids = cols.pid[name_event].tolist()
    return ["pid:%d" % pids[v] if w == 2 else (praw[pa[v]:pb[v]] if w == 0 else graw[ga[v]:gb[v]]).decode("utf-8", "replace")
            for v, w in enumerate(name_which.tolist())]


def graph_from_columns(cols: EventColumns, merge_renames=True, window=None, device=None, observable=False) -> G.TemporalGraph:
    """Same graph as graph.graph_from_events(events_from_columns(cols)) -- nodes, numbering, CSR, weights, features,
    labels -- without a per-event Python loop.  device=None: arrays are numpy (host stages).  device="cuda[:i]":
    the per-node features (graph.node_features_device) and the edge sort / CSR / temporal weights
    (graph.build_csr_device) run on the GPU; rowptr, col, ew, x are CUDA tensors ready for GraphSAGE_T.forward
    (rowptr / col / labels identical to the host path, ew and x within the rounding of exp / log1p)."""
    cols = resolve_columns(cols)                              # path-less (write) events follow the pid's open file
    n = cols.n
    if n == 0:
        raise ValueError("empty trace")
    ts = cols.timestamp
    order = np.argsort(ts, kind="stable")                     # lossy streams may be unordered (main.go:257-263)
    t0 = float(ts[order[0]]); t1 = float(ts[order[-1]])
    span = max(t1 - t0, 1e-6)
    window = window or max(span, G.WINDOW)
    node_p, node_f, node_g, kind, name_event, name_which = intern_nodes(cols, order, merge_renames)
    N = kind.shape[0]
    P = node_p[order].astype(np.int64); F = node_f[order].astype(np.int64); Gn = node_g[order].astype(np.int64)
    t = ts[order] - t0
    raw_slot = cols.event_slot[order].astype(np.int64)
    slot = np.asarray(G.OBSERVABLE_SLOT, np.int64)[raw_slot] if observable else raw_slot
    size = np.minimum(cols.bytes[order], np.uint64(G.MAX_RW_COUNT)).astype(np.int64)
    pf = cols.path_flags[order]
    if merge_renames:                                         # the renamed twin is this node: its .lockbit bit counts
        pf = pf | (path_flags_of(*cols.strings["new_path"])[order] & np.uint8(1))
    has_g = Gn >= 0

    # edges, in the per-event order of the host loader: p->f, f->p [, f->g, g->f]
    src4 = np.stack([P, F, F, Gn], 1); dst4 = np.stack([F, P, Gn, F], 1)
    keep = np.stack([np.ones(n, bool), np.ones(n, bool), has_g, has_g], 1).ravel()
    src = src4.ravel()[keep]; dst = dst4.ravel()[keep]
    tt = np.repeat(t, 4)[keep].astype(np.float32)
    conf = np.ones(src.shape[0], np.float32)

    names = _node_names(cols, name_event, name_which)
    meta = {"kind": "trace", "names": names, "node_kind": kind.astype(np.int64), "t0": t0, "span": span,
            "merge_renames": bool(merge_renames),
            "node_source": np.zeros(N, np.int64) if cols.source is None else cols.source[name_event].astype(np.int64)}
    if device is not None:
        # device path: features by integer atomics + one node pass, edges sorted into CSR by the radix-sort stage
        import torch
        dev = torch.device(device)
        up = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a.astype(dt, copy=False))).to(dev)
        x, label, size_mb = G.node_features_device(up(P, np.int32), up(F, np.int32), up(Gn, np.int32) if has_g.any() else None,
                                                   up(t, np.float64), up(slot, np.uint8), up(cols.bytes[order], np.int64),
                                                   up(pf, np.uint8), up(kind, np.int8), window)
        rowptr, col, ew, perm = G.build_csr_device(up(src, np.int32), up(dst, np.int32), up(tt, np.float32), up(conf, np.float32),
                                                   N, t_ref=float(span), tau=G.TAU, return_perm=True)

        def edge_event(perm=perm, keep=keep, order=order, E=int(src.shape[0])):
            """the event (row of the path-resolved columns) that made each CSR edge"""
            if E == 0:                                                        # perm holds one spare entry
                return torch.zeros(0, dtype=torch.int64, device=perm.device)
            ev = up(np.repeat(order, 4)[keep], np.int64)                      # edge in constructor order -> event row
            return ev[perm.long() & 0xffffffff]

        def edge_time(ts=ts):
            """the trace-clock seconds (float64) of the event that made each CSR edge"""
            return up(ts, np.float64)[edge_event()]

        def edge_flow():
            """the information-flow class (uint8, DESIGN.md 1.5) of the event that made each CSR edge"""
            return up(column_flow(cols), np.uint8)[edge_event()]
        meta.update(edge_event=edge_event, edge_time=edge_time, edge_flow=edge_flow,
                    event_info=lambda ids, cols=cols: column_event_records(cols, ids))
        lab = label.cpu().numpy().astype(np.int64)
        if observable:                                        # the kernel saw the folded slots: labels come from the annotations
            lab = (np.bincount(F[(raw_slot == 1) | (raw_slot == 2)], minlength=N) > 0).astype(np.int64)
        meta.update(label=lab, size_mb=size_mb.cpu().numpy(), device=str(dev))
        return G.TemporalGraph(rowptr, col, ew, x, meta)

    # per-node features over the touched nodes (p, f [, g]) of every event
    tn = np.concatenate([P, F, Gn[has_g]]); tslot = np.concatenate([slot, slot, slot[has_g]])
    tsize = np.concatenate([size, size, size[has_g]]); ttime = np.concatenate([t, t, t[has_g]])
    cnt = np.bincount(tn * G._N_EVENT_SLOTS + tslot, minlength=N * G._N_EVENT_SLOTS).reshape(N, G._N_EVENT_SLOTS).astype(np.float64)
    nbytes = np.zeros(N, np.int64)
    np.add.at(nbytes, tn, tsize)                              # exact: < 2^29 events of < 2^31 bytes each
    nbytes = nbytes.astype(np.float64)
    first = np.full(N, np.inf); last = np.full(N, -np.inf)
    np.minimum.at(first, tn, ttime); np.maximum.at(last, tn, ttime)
    flag = lambda bit: (np.bincount(F[(pf & bit) != 0], minlength=N) > 0).astype(np.float64)
    lockbit, note, tmp = flag(1), flag(2), flag(4)
    label = (np.bincount(F[(raw_slot == 1) | (raw_slot == 2)], minlength=N) > 0).astype(np.int64)

    indeg = np.bincount(dst, minlength=N).astype(np.float32)
    outdeg = np.bincount(src, minlength=N).astype(np.float32)
    x = np.zeros((N, G.F_IN), np.float32)
    x[:, 0] = kind == 0; x[:, 1] = kind == 1
    x[:, 3] = np.log1p(indeg.astype(np.float64)); x[:, 4] = np.log1p(outdeg.astype(np.float64))
    x[:, 5:5 + G._N_EVENT_SLOTS] = np.log1p(cnt)
    x[:, 13] = np.log1p(nbytes) / 20.0
    x[:, 14] = (last - first) / window
    x[:, 15] = first / window
    x[:, 16] = lockbit; x[:, 17] = note; x[:, 18] = tmp
    wr = cnt[:, 1] + cnt[:, 5]
    x[:, 19] = np.divide(cnt[:, 2], wr, out=np.zeros(N), where=wr > 0)
    k = np.maximum(cnt[:, 0] + cnt[:, 1] + cnt[:, 2], 1.0)
    size_mb = np.where(kind == 0, nbytes / k / 1e6, 0.0).astype(np.float32)

    meta.update(label=label, size_mb=size_mb)
    rowptr, col, ew = G.csr_from_edges(src, dst, tt, conf, N, t_ref=float(span), tau=G.TAU)
    # the event (row of the path-resolved columns) that made each CSR edge, its time and its flow class, as on the device
    edge_event = np.repeat(order, 4)[keep].astype(np.int64)[np.lexsort((tt, dst))]
    meta.update(edge_event=edge_event, edge_time=lambda: ts[edge_event].astype(np.float64),
                edge_flow=lambda: column_flow(cols)[edge_event], event_info=lambda ids, cols=cols: column_event_records(cols, ids))
    return G.TemporalGraph(rowptr, col, ew, x, meta)


def column_flow(cols: EventColumns) -> np.ndarray:
    """uint8 flow class of every row (graph.event_flow of its raw slot, flags and ret_val)"""
    return G.event_flow(cols.event_slot, cols.flags.astype(np.int64), cols.ret_val)


def sequences_from_columns(cols: EventColumns, merge_renames=True, t_max=None, observable=False, only_nodes=None,
                           return_events=False):
    """Per-file event sequences for the LSTM without per-event Python: the same arrays as
    pipeline.file_sequences(events_from_columns(cols), graph) -- seq fp32 [n_files, t_max, 16], lengths int32, node ids --
    (the last t_max events of every file node, oldest first; feature layout: pipeline.file_sequences).
    return_events: also the event of each step (sequences_core), a row of the path-resolved columns -- the ids
    graph_from_columns' meta["edge_event"] / meta["event_info"] use."""
    cols = resolve_columns(cols)
    n = cols.n
    ts = cols.timestamp
    order = np.argsort(ts, kind="stable")
    t0 = float(ts[order[0]]) if n else 0.0
    span = max(float(ts[order[-1]]) - t0, 1e-6) if n else 1.0
    _, node_f, _, kind, _, _ = intern_nodes(cols, order, merge_renames)
    return sequences_core(cols, order, node_f[order].astype(np.int64), ts[order], t0, span, kind.shape[0], t_max, observable, only_nodes,
                          return_events)


def sequences_core(cols: EventColumns, order, F, tt, t0, span, n_nodes, t_max=None, observable=False, only_nodes=None,
                   return_events=False):
    """The sequence builder proper, on already interned events: `order` = stored indices of the events in time order,
    F = their file node ids, tt = their absolute timestamps (both in that order).  Used by sequences_from_columns and by the
    device stream (stream.DeviceStream), whose interning ran on the GPU.
    return_events: a fourth array, int64 [n_files, t_max], the stored index (`order` entry) of the event of each step,
    -1 at padded steps."""
    from .ai.models import lstm
    t_max = t_max or lstm.T_MAX
    n = int(F.shape[0])
    if only_nodes is not None:
        # sequences for a subset of the file nodes only (the top-A candidates of a large window): drop every other event
        # up front -- node ids, time order and the per-file histories of the kept nodes are unchanged
        keep_node = np.zeros(n_nodes, bool); keep_node[np.asarray(only_nodes, np.int64)] = True
        sel_ev = keep_node[F]
        order, F, tt = order[sel_ev], F[sel_ev], tt[sel_ev]
        n = int(F.shape[0])
    if n == 0:
        empty = (np.zeros((0, t_max, lstm.D_IN), np.float32), np.zeros(0, np.int32), np.zeros(0, np.int64))
        return empty + (np.zeros((0, t_max), np.int64),) if return_events else empty
    # group by file node, keeping time order inside a group
    by_file = np.argsort(F, kind="stable")
    Fg = F[by_file]
    nodes, start, count = np.unique(Fg, return_index=True, return_counts=True)
    pos = np.arange(n) - np.repeat(start, count)          # rank of the event inside its file's history
    keep_from = np.repeat(np.maximum(count - t_max, 0), count)
    sel = pos >= keep_from                                # the last t_max events
    row = np.repeat(np.arange(nodes.size), count)[sel]
    k = (pos - keep_from)[sel]
    ev = by_file[sel]                                     # index into the time-sorted arrays
    seq = np.zeros((nodes.size, t_max, lstm.D_IN), np.float32)
    lengths = np.minimum(count, t_max).astype(np.int32)
    slot = cols.event_slot[order][ev].astype(np.int64)
    if observable:
        slot = np.asarray(G.OBSERVABLE_SLOT, np.int64)[slot]
    seq[row, k, slot] = 1.0
    seq[row, k, 8] = np.log1p(np.minimum(cols.bytes[order][ev], np.uint64(G.MAX_RW_COUNT)).astype(np.float64)) / 20.0
    prev_t = np.empty(n); prev_t[1:] = tt[by_file][:-1]; prev_t[0] = 0.0
    dt = np.minimum(tt[by_file] - prev_t, 10.0)
    dt[(pos == keep_from)] = 0.0                          # first kept event of a file has no predecessor in the window
    seq[row, k, 9] = dt[sel]
    seq[row, k, 10] = (tt[ev] - t0) / span
    pf = cols.path_flags[order][ev]
    seq[row, k, 11] = (pf & 1) != 0
    seq[row, k, 12] = (pf & 4) != 0
    if return_events:
        events = np.full((nodes.size, t_max), -1, np.int64)
        events[row, k] = np.asarray(order, np.int64)[ev]
        return seq, lengths, nodes.astype(np.int64), events
    return seq, lengths, nodes.astype(np.int64)


# ------------------------------------------------------------------ test / tooling helper (not on the product path)
def encode_event_batch(events) -> bytes:
    """Minimal protobuf WRITER for nerrf.trace.EventBatch (proto3 canonical form: default-valued fields omitted),
    so traces in the dict schema can be replayed through the ingest path without protoc.  events: dicts with
    ts=(seconds, nanos) | None or timestamp=float seconds, pid, tid, comm, syscall|event, path, new_path, flags, ret_val,
    bytes|size."""
    def varint(v):
        v &= (1 << 64) - 1
        out = bytearray()
        while True:
            b = v & 0x7f
            v >>= 7
            out.append(b | (0x80 if v else 0))
            if not v:
                return bytes(out)

    def field_varint(num, v):
        return b"" if v == 0 else varint(num << 3) + varint(v)

    def field_bytes(num, s, keep_empty=False):
        s = s.encode("utf-8") if isinstance(s, str) else bytes(s)
        return b"" if (not s and not keep_empty) else varint(num << 3 | 2) + varint(len(s)) + s

    out = bytearray()
    for e in events:
        if "ts" in e and e["ts"] is None:
            sec = nanos = None                       # field absent (presence matters for sub-messages)
        elif "ts" in e:
            sec, nanos = e["ts"]
        else:
            tsf = float(e["timestamp"]) if not isinstance(e["timestamp"], str) else G._parse_ts(e["timestamp"])
            sec = int(np.floor(tsf)); nanos = int(round((tsf - sec) * 1e9))
            if nanos >= 1_000_000_000:
                sec += 1; nanos -= 1_000_000_000
        ts = b"" if sec is None else field_bytes(1, field_varint(1, sec) + field_varint(2, nanos), keep_empty=True)
        rv = int(e.get("ret_val", 0))
        body = (ts + field_varint(2, int(e.get("pid", 0))) + field_varint(3, int(e.get("tid", 0)))
                + field_bytes(4, e.get("comm", "")) + field_bytes(5, e.get("syscall", e.get("event", "")))
                + field_bytes(6, e.get("path", "")) + field_bytes(7, e.get("new_path", "") or "")
                + field_varint(8, int(e.get("flags", 0))) + field_varint(9, (rv << 1) ^ (rv >> 63))
                + field_varint(10, int(e.get("bytes", e.get("size", 0)) or 0)))
        out += varint(1 << 3 | 2) + varint(len(body)) + body
    return bytes(out)


def encode_columns(cols: EventColumns) -> list:
    """One serialized EventBatch record (field 1 = an Event) per row of `cols`, in stored order: the stream a tracker
    would send, for replaying column traces through the live path (test / tooling helper)."""
    from functools import lru_cache

    @lru_cache(maxsize=1 << 16)
    def varint(v):
        v &= (1 << 64) - 1
        out = bytearray()
        while True:
            b = v & 0x7f
            v >>= 7
            out.append(b | (0x80 if v else 0))
            if not v:
                return bytes(out)

    raw = {k: (off.tolist(), data.tobytes()) for k, (off, data) in cols.strings.items()}
    sec, nan, pid, tid = cols.ts_sec.tolist(), cols.ts_nanos.tolist(), cols.pid.tolist(), cols.tid.tolist()
    flg, rv, by = cols.flags.tolist(), cols.ret_val.tolist(), cols.bytes.tolist()
    fields = ((4, "comm"), (5, "syscall"), (6, "path"), (7, "new_path"))
    recs = []
    for i in range(cols.n):
        ts = (varint(8) + varint(sec[i]) if sec[i] else b"") + (varint(16) + varint(nan[i]) if nan[i] else b"")
        body = [b"\x0a", varint(len(ts)), ts]
        if pid[i]:
            body += [b"\x10", varint(pid[i])]
        if tid[i]:
            body += [b"\x18", varint(tid[i])]
        for num, name in fields:
            off, data = raw[name]
            if off[i + 1] > off[i]:
                body += [varint(num << 3 | 2), varint(off[i + 1] - off[i]), data[off[i]:off[i + 1]]]
        if flg[i]:
            body += [b"\x40", varint(flg[i])]
        if rv[i]:
            body += [b"\x48", varint((rv[i] << 1) ^ (rv[i] >> 63))]
        if by[i]:
            body += [b"\x50", varint(by[i])]
        b = b"".join(body)
        recs.append(b"\x0a" + varint(len(b)) + b)
    return recs
