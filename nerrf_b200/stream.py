"""Streamed traces at fleet scale (BASELINE config 5: "End-to-end LockBit trace: streamed graph -> GNN anomaly score ->
MCTS rollback plan"): a columnar fleet-trace generator, the sliding window, and the tick loop around pipeline.run.

Reference anchors (prose + fixtures; the reference ships no graph constructor or planner):
  * "Sliding window (30-60 sec)", "Node merging (inode deduplication)"      docs/content/docs/architecture.mdx:39-41
  * pipeline order tracker -> graph -> AI models -> planner -> sandbox       docs/content/docs/architecture.mdx:12-86
  * one process's trace = the simulator's schema and phases                  benchmarks/m1/scripts/sim_lockbit_m1.py:24-36,
    benchmarks/m1/results/m1_trace.jsonl (149 events, 45 encrypted files)
  * SURVEY.md 8d cfg 5: "m1 trace replicated xK with pid/path renaming to a >= 1M-node stream"

Host code (numpy, no per-event Python): replicas are produced by tiling the columns of ONE decoded base trace and
patching a fixed-width placeholder in the path bytes."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from . import graph as G, ingest, trace_sim

_PLACEHOLDER = b"p0000000_"          # fixed width: 7 decimal digits patched per replica
_DIGITS = 7


def _base_columns(attacked: bool, n_files: int, benign_files: int, seed: int, bystanders: int = 0,
                  pid_stride: int = 0) -> ingest.EventColumns:
    ev = trace_sim.lockbit_trace(n_files=n_files if attacked else 0, seed=seed, benign_files=benign_files + (0 if attacked else n_files),
                                 bystanders=bystanders)
    if not attacked:                      # a benign process: no encryption phase, no ransom note
        ev = [e for e in ev if e["phase"] not in ("attack",) and e["event"] not in ("encryption_start", "encryption_complete")]
    if bystanders:                        # bystander k: pid + (k + 1) * pid_stride, clear of every replica's attacker pid
        pid0 = ev[0]["pid"]
        for e in ev:
            if e["pid"] != pid0:
                e["pid"] = pid0 + (e["pid"] - pid0) * pid_stride
    for e in ev:
        slash = e["path"].rfind("/")
        if e["path"].startswith("/app/uploads/") and slash >= 0 and "." in e["path"][slash:]:
            e["path"] = e["path"][:slash + 1] + _PLACEHOLDER.decode() + e["path"][slash + 1:]   # per-process files; dirs stay shared
    return ingest.decode_event_batch(ingest.encode_event_batch(ev))


def _replicate(cols: ingest.EventColumns, ids: np.ndarray, t_shift: np.ndarray) -> ingest.EventColumns:
    """K copies of `cols`: replica j gets pid + ids[j], its placeholder digits = ids[j], its clock shifted by t_shift[j] s."""
    K, n = ids.shape[0], cols.n
    strings = {}
    for name, (off, data) in cols.strings.items():
        L = int(off[-1])
        d = np.tile(data, K).reshape(K, L) if L else np.zeros((K, 0), np.uint8)
        if L:
            raw = data.tobytes()
            pos, start = [], 0
            while True:
                k = raw.find(_PLACEHOLDER, start)
                if k < 0:
                    break
                pos.append(k + 1); start = k + 1
            if pos:
                pos = np.asarray(pos, np.int64)
                for dgt in range(_DIGITS):
                    digit = ((ids // 10 ** (_DIGITS - 1 - dgt)) % 10).astype(np.uint8) + np.uint8(ord("0"))
                    d[:, pos + dgt] = digit[:, None]
        new_off = np.empty(K * n + 1, np.int64)
        new_off[:-1] = (off[None, :-1] + (np.arange(K, dtype=np.int64) * L)[:, None]).ravel()
        new_off[-1] = K * L
        strings[name] = (new_off, d.reshape(-1))
    ts = cols.timestamp[None, :] + t_shift[:, None]
    sec = np.floor(ts)
    out = ingest.EventColumns(
        n=K * n, ts_sec=sec.astype(np.int64).ravel(), ts_nanos=np.round((ts - sec) * 1e9).astype(np.int32).clip(0, 999_999_999).ravel(),
        pid=(cols.pid[None, :].astype(np.int64) + ids[:, None]).astype(np.uint32).ravel(), tid=np.tile(cols.tid, K),
        flags=np.tile(cols.flags, K), ret_val=np.tile(cols.ret_val, K), bytes=np.tile(cols.bytes, K),
        event_slot=np.tile(cols.event_slot, K), path_flags=np.tile(cols.path_flags, K), strings=strings)
    return out


def concat_columns(parts) -> ingest.EventColumns:
    strings = {}
    for name in ingest.STRING_COLUMNS:
        offs, datas, base = [], [], 0
        for c in parts:
            off, data = c.strings[name]
            offs.append(off[:-1] + base); datas.append(data); base += int(off[-1])
        strings[name] = (np.concatenate(offs + [np.asarray([base], np.int64)]), np.concatenate(datas) if datas else np.zeros(0, np.uint8))
    cat = lambda k: np.concatenate([getattr(c, k) for c in parts])
    source = None
    if any(c.source is not None for c in parts):
        source = np.concatenate([c.source if c.source is not None else np.zeros(c.n, np.uint16) for c in parts]).astype(np.uint16)
    return ingest.EventColumns(n=sum(c.n for c in parts), strings=strings, source=source,
                               **{k: cat(k) for k in ("ts_sec", "ts_nanos", "pid", "tid", "flags", "ret_val", "bytes", "event_slot", "path_flags")})


def fleet_columns(n_procs: int, n_attacked: int, seed: int = 0, n_files: int = 45, benign_files: int = 50, jitter_s: float = 5.0,
                  return_pids: bool = False, bystanders: int = 0):
    """A fleet of `n_procs` processes, each with its own n_files + benign_files files under /app/uploads (the m1
    simulator's layout); `n_attacked` of them run the LockBit encryption phase on n_files of their files.
    bystanders: k benign processes per attacked process that open and write its files, some of the encrypted ones after
    the attacker under their .lockbit3 name (trace_sim.lockbit_trace), each with a pid of its own; without them the
    per-pair edge labels of a window only repeat its file labels.  bystanders=0 emits exactly the events it always did.
    -> (EventColumns, encrypted_paths: set of the .lockbit3 names a correct plan must rename back)."""
    rng = np.random.default_rng(seed)
    att = _base_columns(True, n_files, benign_files, seed, bystanders, pid_stride=n_procs + 1000)
    ben = _base_columns(False, n_files, benign_files, seed + 1)
    ids = rng.permutation(n_procs).astype(np.int64) + 1000
    shift = rng.random(n_procs) * jitter_s
    parts = []
    if n_attacked:
        parts.append(_replicate(att, ids[:n_attacked], shift[:n_attacked]))
    if n_procs > n_attacked:
        parts.append(_replicate(ben, ids[n_attacked:], shift[n_attacked:]))
    cols = concat_columns(parts)
    enc = set()
    if n_attacked:
        a = parts[0]
        off, data = a.strings["path"]
        idx = np.nonzero((a.path_flags & 8) != 0)[0]
        raw = data.tobytes()
        enc = {raw[off[i]:off[i + 1]].decode() for i in idx.tolist()}
    if return_pids:                       # the ransomware processes, by the node name the graph constructor gives them
        return cols, enc, {"pid:%d" % (int(att.pid[0]) + int(i)) for i in ids[:n_attacked].tolist()}
    return cols, enc


def window(cols: ingest.EventColumns, t_lo: float, t_hi: float) -> ingest.EventColumns:
    """The events with t_lo < t <= t_hi (the sliding window of architecture.mdx:39-41), stored order preserved."""
    ts = cols.timestamp
    keep = np.nonzero((ts > t_lo) & (ts <= t_hi))[0]
    strings = {name: ingest._gather_strings(*cols.strings[name], keep) for name in ingest.STRING_COLUMNS}
    sc = {k: getattr(cols, k)[keep] for k in ("ts_sec", "ts_nanos", "pid", "tid", "flags", "ret_val", "bytes", "event_slot", "path_flags")}
    return ingest.EventColumns(n=int(keep.shape[0]), strings=strings, source=None if cols.source is None else cols.source[keep], **sc)


def with_source(cols: ingest.EventColumns, source: int) -> ingest.EventColumns:
    """`cols` with every event from source id `source`"""
    check_source_id(source)
    return ingest.EventColumns(**{**cols.__dict__, "source": np.full(cols.n, source, np.uint16)})


def host_streams(k_hosts: int, n_procs: int, n_attacked: int, attacked_hosts=None, seed: int = 0, bystanders: int = 0):
    """K hosts' traces whose processes and files collide on purpose: every host runs fleet_columns(n_procs, ...) with the
    same seed, so all hosts reuse the same pids and /app/uploads file names and the same clock; the hosts in
    `attacked_hosts` (default: every other host, starting with host 0) run `n_attacked` LockBit processes, the others only
    benign ones -- whose pids equal the attackers' pids on the attacked hosts.
    -> list of (EventColumns of source h, encrypted paths, attacker node names "pid:<n>"), one per host h."""
    attacked = set(range(0, k_hosts, 2)) if attacked_hosts is None else set(attacked_hosts)
    out = []
    for h in range(k_hosts):
        cols, enc, pids = fleet_columns(n_procs, n_attacked if h in attacked else 0, seed=seed, return_pids=True,
                                        bystanders=bystanders if h in attacked else 0)
        out.append((with_source(cols, h), enc, pids))
    return out


def relabel_single_source(cols: ingest.EventColumns) -> ingest.EventColumns:
    """The multi-source stream `cols` as ONE source, the identity the source column stands for: every (source, pid)
    becomes a pid of its own (numbered in (source, pid) order), every non-empty path / new_path gets the prefix
    "@<source>/", empty paths stay empty (so path-less writes resolve as before).  path_flags are kept as they were (the
    prefix would hide the /tmp rule).  Feeding the result to the single-source path gives the multi-source graph."""
    if cols.source is None:
        return cols
    uniq, inv = np.unique(ingest.process_keys(cols), return_inverse=True)
    if uniq.size >= (1 << 32):
        raise ValueError("more than 2^32 processes")
    strings = dict(cols.strings)
    for name in ("path", "new_path"):
        off, data = cols.strings[name]
        ln = off[1:] - off[:-1]
        pre = [("@%d/" % s).encode() for s in range(int(cols.source.max()) + 1)]
        plen = np.asarray([len(p) for p in pre], np.int64)[cols.source.astype(np.int64)] * (ln > 0)
        new_off = np.zeros(cols.n + 1, np.int64); np.cumsum(ln + plen, out=new_off[1:])
        raw, parts = data.tobytes(), []
        src = cols.source.tolist()
        for i, (a, b) in enumerate(zip(off[:-1].tolist(), off[1:].tolist())):
            if b > a:
                parts.append(pre[src[i]]); parts.append(raw[a:b])
        strings[name] = (new_off, np.frombuffer(b"".join(parts), np.uint8).copy())
    return ingest.EventColumns(**{**cols.__dict__, "pid": inv.astype(np.uint32).reshape(-1), "strings": strings, "source": None})


# ---------------------------------------------------------------------------------------------- device-resident stream
_M64 = (1 << 64) - 1


def _mix64(h: int) -> int:
    h ^= h >> 33; h = (h * 0xff51afd7ed558ccd) & _M64; h ^= h >> 33; h = (h * 0xc4ceb9fe1a85ec53) & _M64; h ^= h >> 33
    return h or 1


def check_source_id(source: int) -> int:
    from . import _lib
    if not isinstance(source, (int, np.integer)) or not 0 <= int(source) < (1 << 16):
        raise _lib.NerrfError("source id %r out of range [0, 65536)" % (source,))
    return int(source)


def name_hash(name, source: int = 0) -> int:
    """The 64-bit name hash of csrc/intern_device.cu (nerrf_trace_name_hash_ex) on the host, as a SIGNED int64: FNV-1a
    over the bytes seeded with the length, murmur3 finaliser; "pid:<n>" names hash (source << 32) | pid; a file name of
    a nonzero source is qualified by it (source 0: the unqualified hash)."""
    source = check_source_id(source)
    if isinstance(name, str) and name.startswith("pid:") and name[4:].isdigit():
        h = _mix64((((source << 32) | int(name[4:])) + 0x9E3779B97F4A7C15) & _M64)
    else:
        b = name.encode("utf-8") if isinstance(name, str) else bytes(name)
        h = (0xcbf29ce484222325 ^ len(b)) & _M64
        for c in b:
            h = ((h ^ c) * 0x100000001b3) & _M64
        h = _mix64(h)
        if source:
            h = _mix64((h + source * 0x9E3779B97F4A7C15) & _M64)
    return h - (1 << 64) if h >= (1 << 63) else h


def dir_hash(name, source: int = 0) -> int:
    """The 64-bit hash of a node's parent directory (csrc/intern_device.cu nerrf_trace_dir_hash_ex) on the host, as a
    SIGNED int64: name_hash of the bytes up to (not including) the last '/' -- the empty string when there is none;
    "pid:<n>" names hash as in name_hash.  Qualified by `source` like name_hash."""
    if isinstance(name, str) and name.startswith("pid:") and name[4:].isdigit():
        return name_hash(name, source)
    b = name.encode("utf-8") if isinstance(name, str) else bytes(name)
    k = b.rfind(b"/")
    return name_hash(b[:k] if k >= 0 else b"", source)


def parent_dir(name) -> str:
    """The directory dir_hash hashes (the name up to its last '/')."""
    k = name.rfind("/")
    return name[:k] if k >= 0 else ""


class LazyNames:
    """Node names of a window graph, decoded on demand (a window holds ~10^6 nodes, a plan names a few thousand)."""

    def __init__(self, cols: ingest.EventColumns, name_event: np.ndarray, name_which: np.ndarray):
        self.cols, self.name_event, self.name_which = cols, name_event, name_which

    def __len__(self):
        return int(self.name_event.shape[0])

    def __getitem__(self, v):
        e, w = int(self.name_event[v]), int(self.name_which[v])
        return "pid:%d" % int(self.cols.pid[e]) if w == 2 else self.cols.text("path" if w == 0 else "new_path", e)

    def take(self, nodes):
        return [self[v] for v in nodes]


class DeviceNames:
    """Node names of a live window graph, read from the device string columns: `take` fetches the names of many nodes
    with two device-to-host copies, whatever their number."""

    def __init__(self, pid, poff, pdata, goff, gdata, name_event: np.ndarray, name_which: np.ndarray):
        self.pid, self.poff, self.pdata, self.goff, self.gdata = pid, poff, pdata, goff, gdata
        self.name_event, self.name_which = name_event, name_which

    def __len__(self):
        return int(self.name_event.shape[0])

    def __getitem__(self, v):
        return self.take([v])[0]

    def take(self, nodes):
        import torch
        nodes = np.asarray(nodes, np.int64).reshape(-1)
        if nodes.size == 0:
            return []
        ev, which = self.name_event[nodes], self.name_which[nodes]
        e = torch.from_numpy(ev).to(self.pid.device)
        meta = torch.stack([self.poff[e], self.poff[e + 1], self.goff[e], self.goff[e + 1],
                            self.pid[e].to(torch.int64) & 0xffffffff]).cpu().numpy()
        lo = np.where(which == 1, meta[2], meta[0]); hi = np.where(which == 1, meta[3], meta[1])
        ln = np.where(which == 2, 0, hi - lo)
        starts = np.zeros(nodes.size + 1, np.int64); np.cumsum(ln, out=starts[1:])
        raw = b""
        if starts[-1]:
            pos = np.arange(starts[-1], dtype=np.int64) - np.repeat(starts[:-1], ln) + np.repeat(lo, ln)
            from_g = np.repeat(which == 1, ln)
            p = torch.from_numpy(pos).to(self.pid.device); g = torch.from_numpy(from_g).to(self.pid.device)
            pick = torch.where(g, self.gdata[p.clamp(max=self.gdata.numel() - 1)], self.pdata[p.clamp(max=self.pdata.numel() - 1)])
            raw = pick.cpu().numpy().tobytes()
        return ["pid:%d" % int(meta[4][k]) if which[k] == 2 else raw[starts[k]:starts[k + 1]].decode("utf-8", "replace")
                for k in range(nodes.size)]


_SCALARS = (("ts_sec", "int64"), ("ts_nanos", "int32"), ("pid", "int32"), ("tid", "int32"), ("flags", "int32"),
            ("ret_val", "int64"), ("bytes", "int64"), ("event_slot", "uint8"), ("path_flags", "uint8"))


class _DeviceColumns:
    """EventColumns in HBM with room to grow: scalars [rows], string offsets [rows + 1], string bytes; ptrs() = the 17
    column pointers of the C entry points (nerrf_trace_decode's argument order)."""

    def __init__(self, dev, rows: int, nbytes):
        import torch
        self.dev = dev
        self.s = {k: torch.zeros(max(rows, 1), dtype=getattr(torch, dt), device=dev) for k, dt in _SCALARS}
        self.off = [torch.zeros(max(rows, 1) + 1, dtype=torch.int64, device=dev) for _ in range(4)]
        self.data = [torch.zeros(max(int(b), 1), dtype=torch.uint8, device=dev) for b in nbytes]
        self.source = torch.zeros(max(rows, 1), dtype=torch.int16, device=dev)   # uint16 source ids, stored as int16

    @property
    def rows(self):
        return int(self.s["ts_sec"].shape[0])

    def ptrs(self):
        t = [self.s[k] for k, _ in _SCALARS]
        for q in range(4):
            t += [self.off[q], self.data[q]]
        return _lib_ptr_array(t)

    def reserve(self, n_used: int, used_bytes, rows: int, nbytes):
        """room for `rows` rows and nbytes[q] bytes per string column, keeping the first n_used rows"""
        import torch
        if rows > self.rows:
            new = max(rows, 2 * self.rows)
            for k, _ in _SCALARS:
                t = torch.zeros(new, dtype=self.s[k].dtype, device=self.dev); t[:n_used] = self.s[k][:n_used]; self.s[k] = t
            for q in range(4):
                t = torch.zeros(new + 1, dtype=torch.int64, device=self.dev); t[:n_used + 1] = self.off[q][:n_used + 1]; self.off[q] = t
            t = torch.zeros(new, dtype=torch.int16, device=self.dev); t[:n_used] = self.source[:n_used]; self.source = t
        for q in range(4):
            if nbytes[q] > self.data[q].numel():
                t = torch.zeros(max(int(nbytes[q]), 2 * self.data[q].numel()), dtype=torch.uint8, device=self.dev)
                t[:used_bytes[q]] = self.data[q][:used_bytes[q]]
                self.data[q] = t

    def host(self, n: int) -> ingest.EventColumns:
        """the first n rows as host EventColumns"""
        sc = {k: self.s[k][:n].cpu().numpy() for k, _ in _SCALARS}
        sc["pid"] = sc["pid"].view(np.uint32); sc["tid"] = sc["tid"].view(np.uint32); sc["bytes"] = sc["bytes"].view(np.uint64)
        strings = {}
        for q, name in enumerate(ingest.STRING_COLUMNS):
            off = self.off[q][:n + 1].cpu().numpy()
            strings[name] = (off, self.data[q][:int(off[-1])].cpu().numpy())
        source = self.source[:n].cpu().numpy().view(np.uint16)
        return ingest.EventColumns(n=n, strings=strings, source=source if source.any() else None, **sc)


def _lib_ptr_array(tensors):
    from . import _lib
    return _lib.ptr_array(tensors)


def _decode_into(dc: _DeviceColumns, n: int, used_bytes, raw: np.ndarray, partial: bool, timings=None, source: int = 0):
    """Frame `raw` on the host, decode its Event records on the device into rows n.. of `dc`, all from source id `source`.
    -> (rows added, bytes consumed, new used_bytes).  Raises (and adds nothing) when a record is malformed: same message and byte offset as
    ingest.decode_event_batch."""
    import ctypes as C
    import time
    import torch
    from . import _lib
    a = time.perf_counter()
    bad, rec_at, body_off, body_len, consumed = ingest._frame(raw, partial)
    m = int(rec_at.shape[0])
    if timings is not None:
        timings["frame_ms"] = (time.perf_counter() - a) * 1e3
    dev_bad = None
    used = list(used_bytes)
    if m:
        payload = int(body_len.sum())
        if payload >= (1 << 31):
            raise _lib.NerrfError("append of %d event bytes: split it (at most 2^31 - 1 per append)" % payload)
        end = int(body_off[-1] + body_len[-1])
        wire_d = torch.from_numpy(raw[:end] if raw.flags.writeable else raw[:end].copy()).to(dc.dev)
        rec_d = torch.from_numpy(np.stack([rec_at, body_off, body_len])).to(dc.dev)
        dc.reserve(n, used, n + m, [u + payload for u in used])
        need = C.c_int64()
        _lib.check(_lib.lib().nerrf_trace_decode_device_workspace_bytes(m, C.byref(need)), "decode_device_workspace_bytes")
        ws = torch.empty(need.value + 256, dtype=torch.uint8, device=dc.dev)
        status = torch.empty(1, dtype=torch.int64, device=dc.dev)
        ev0 = torch.cuda.Event(enable_timing=True); ev1 = torch.cuda.Event(enable_timing=True)
        with torch.cuda.device(dc.dev):
            ev0.record()
            _lib.check(_lib.lib().nerrf_trace_decode_device_ex(
                _lib.ptr(wire_d), _lib.ptr(rec_d[0]), _lib.ptr(rec_d[1]), _lib.ptr(rec_d[2]), m, n, dc.ptrs(), _lib.ptr(dc.source),
                int(source), _lib.ptr(status), C.c_void_p((ws.data_ptr() + 255) & ~255), need.value, _lib.current_stream_ptr()),
                "nerrf_trace_decode_device_ex")
            ev1.record()
        back = torch.cat([status] + [o[n + m:n + m + 1] for o in dc.off]).cpu().numpy()
        if timings is not None:
            timings["decode_ms"] = ev0.elapsed_time(ev1)
        if back[0] != -1:
            dev_bad = int(back[0])
        used = [int(v) for v in back[1:]]
    worst = min([b for b in (bad, dev_bad) if b is not None], default=None)
    if worst is not None:
        raise _lib.NerrfError(f"nerrf_trace_decode_device failed: malformed EventBatch at byte offset {worst}")
    return m, consumed, used


def _rows_string_bytes(dc: _DeviceColumns, rows) -> list:
    """bytes of each of the four string columns held by `rows` (device int64 indices) of `dc`"""
    import torch
    if rows.numel() == 0:
        return [0, 0, 0, 0]
    return [int(v) for v in torch.stack([(o[rows + 1] - o[rows]).sum() for o in dc.off]).cpu().numpy()]


def _require_gather_fits(nbytes):
    """nerrf_trace_gather_rows turns the lengths of all four string columns into offsets with ONE int32 scan: the bytes
    it moves must sum to less than 2^31 (the per-append limit of _decode_into, for the rows a compaction keeps)."""
    from . import _lib
    total = sum(int(b) for b in nbytes)
    if total >= (1 << 31):
        raise _lib.NerrfError("compaction keeps %d string bytes: at most 2^31 - 1 (advance the horizon, or compact more often)" % total)


def decode_event_batch_device(buf, device="cuda") -> ingest.EventColumns:
    """ingest.decode_event_batch with the Event bodies parsed ON THE DEVICE (nerrf_trace_decode_device): the same
    columns, brought back to the host."""
    import torch
    raw = np.frombuffer(buf, dtype=np.uint8) if not isinstance(buf, np.ndarray) else np.ascontiguousarray(buf, np.uint8)
    dc = _DeviceColumns(torch.device(device), 1, [1, 1, 1, 1])
    m, _, _ = _decode_into(dc, 0, [0, 0, 0, 0], raw, False)
    return dc.host(m)


class DeviceStream:
    """The event stream resident in HBM (SURVEY.md 8f rank 1: "window, inode/path dedup via hash, sort-by-dst -> CSR,
    feature counts" on the GPU; docs/content/docs/architecture.mdx:39-41).  Columns are uploaded ONCE; a sliding window
    is a slice of the time-sorted index array, and everything per tick -- node interning (hash table), per-node features,
    edge assembly, CSR -- runs on the device.  The host keeps the strings only to NAME the few nodes a plan touches."""

    def __init__(self, cols: ingest.EventColumns, device="cuda", observable=True, merge_renames=True):
        import torch
        self.torch = torch
        cols = ingest.resolve_columns(cols)                   # path-less (write) events follow the pid's open file
        self.cols, self.observable, self.merge = cols, observable, bool(merge_renames)
        self.dev = dev = torch.device(device)
        ts = cols.timestamp
        self.order = np.argsort(ts, kind="stable")
        self.ts_sorted = ts[self.order]
        up = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)
        n = cols.n
        self.n = n
        (poff, pdata), (goff, gdata) = cols.strings["path"], cols.strings["new_path"]
        self.d_order = up(self.order, np.int64)
        self.d_ts = up(ts, np.float64)
        self.d_pid = up(cols.pid.astype(np.uint32).view(np.int32), np.int32)
        self.d_source = None if cols.source is None else up(cols.source.astype(np.uint16).view(np.int16), np.int16)
        self.d_poff, self.d_goff = up(poff, np.int64), up(goff, np.int64)
        self.d_pdata = up(pdata if pdata.size else np.zeros(1, np.uint8), np.uint8)
        self.d_gdata = up(gdata if gdata.size else np.zeros(1, np.uint8), np.uint8)
        raw = cols.event_slot
        self.d_raw_slot = up(raw, np.uint8)
        self.d_slot = up(np.asarray(G.OBSERVABLE_SLOT, np.uint8)[raw] if observable else raw, np.uint8)
        self.d_bytes = up(cols.bytes.astype(np.int64), np.int64)
        pf = cols.path_flags
        if self.merge:                                        # the renamed twin is the same node: its .lockbit bit counts
            pf = pf | (ingest.path_flags_of(goff, gdata) & np.uint8(1))
        self.d_pf = up(pf, np.uint8)
        self.d_pf_raw = up(cols.path_flags, np.uint8)         # the sequences use the event's own path flags
        self._flow = None                                     # the flow class of every event, on first use (flow())
        self.cap = max((2 if self.merge else 3) * n, 1)
        self.node_p = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        self.node_f = torch.empty_like(self.node_p); self.node_g = torch.empty_like(self.node_p)
        self.kind = torch.zeros(self.cap, dtype=torch.int8, device=dev)
        self.name_event = torch.zeros(self.cap, dtype=torch.int64, device=dev)
        self.name_which = torch.zeros(self.cap, dtype=torch.int8, device=dev)
        import ctypes as C
        from . import _lib
        need = C.c_int64()
        _lib.check(_lib.lib().nerrf_trace_intern_device_workspace_bytes(max(n, 1), self.cap, C.byref(need)), "intern_device_workspace_bytes")
        self._ws = torch.empty(need.value + 256, dtype=torch.uint8, device=dev)
        self._ws_bytes = need.value

    @classmethod
    def live(cls, device="cuda", observable=True, merge_renames=True):
        """An empty stream that grows as the tracker delivers EventBatch bytes (append) and sheds what no future window
        can reach (compact).  Decoding, time order, path resolution and retention run on the device."""
        import torch
        self = cls.__new__(cls)
        self.torch = torch
        self.dev = torch.device(device)
        self.observable, self.merge = observable, bool(merge_renames)
        self.cols = None
        self._dc = _DeviceColumns(self.dev, 1024, [1 << 16] * 4)
        self._used = [0, 0, 0, 0]
        self._key_bits = 32                                    # 48 once a nonzero source has appended: (source, pid) regroup
        self._horizon = -np.inf
        self._slot_map = torch.tensor(G.OBSERVABLE_SLOT, dtype=torch.uint8, device=self.dev) if observable else None
        self.n = 0
        self.n_keep = 0
        self.timings_ms = {}
        self._rebuild()
        return self

    @property
    def multi_source(self) -> bool:
        """some event comes from a nonzero source (the live stream: since the first such append)"""
        if self.cols is None:
            return self._key_bits == 48
        return self.cols.source is not None and bool(self.cols.source.any())

    @property
    def resident_events(self) -> int:
        """events held in HBM (live stream)"""
        return self.n

    def append(self, wire_bytes, partial=False, source: int = 0) -> int:
        """Decode whole EventBatch records on the device and append them, every one from source id `source` (the host
        whose tracker sent them; processes and files of different sources never merge).  partial=True: a cut-off trailing
        record is left for the caller to resend with the rest of its bytes.  -> bytes consumed.  A malformed record
        raises and leaves the stream as it was."""
        source = check_source_id(source)
        raw = np.frombuffer(wire_bytes, dtype=np.uint8) if not isinstance(wire_bytes, np.ndarray) else np.ascontiguousarray(wire_bytes, np.uint8)
        self.timings_ms = {}
        m, consumed, used = _decode_into(self._dc, self.n, self._used, raw, partial, self.timings_ms, source)
        self.appended = (self.n, self.n + m)
        if m:
            before = self.n, self._used, self._key_bits
            self.n += m
            self._used = used
            if source:
                self._key_bits = 48
            try:
                self._rebuild()
            except Exception:                                  # e.g. 2^31 resolved path bytes: the rows stay unused past n
                self.n, self._used, self._key_bits = before
                self.appended = (self.n, self.n)
                raise
        return consumed

    def compact(self, horizon: float):
        """Drop the events no window ending after `horizon + window` can hold (ts <= horizon), except each (source, pid)'s
        latest event with a path, which a later path-less write of that process still resolves to.  Stored order is kept."""
        import ctypes as C
        from . import _lib
        torch = self.torch
        self._horizon = max(self._horizon, float(horizon))
        ev0 = torch.cuda.Event(enable_timing=True); ev1 = torch.cuda.Event(enable_timing=True)
        with torch.cuda.device(self.dev):
            ev0.record()
        self._rebuild()
        if self._n_retain < self.n:
            m = self._n_retain
            nbytes = self._used                                # distinct rows: at most the stored bytes of each column
            if sum(nbytes) >= 1 << 31:
                nbytes = _rows_string_bytes(self._dc, self._retain)
            _require_gather_fits(nbytes)
            out = _DeviceColumns(self.dev, self._dc.rows, [d.numel() for d in self._dc.data])
            need = C.c_int64()
            _lib.check(_lib.lib().nerrf_trace_gather_rows_workspace_bytes(m, C.byref(need)), "gather_rows_workspace_bytes")
            ws = torch.empty(need.value + 256, dtype=torch.uint8, device=self.dev)
            with torch.cuda.device(self.dev):
                _lib.check(_lib.lib().nerrf_trace_gather_rows_ex(self._dc.ptrs(), _lib.ptr(self._dc.source), _lib.ptr(self._retain), m,
                                                                 out.ptrs(), _lib.ptr(out.source), C.c_void_p((ws.data_ptr() + 255) & ~255),
                                                                 need.value, _lib.current_stream_ptr()), "nerrf_trace_gather_rows_ex")
            self._dc, self.n = out, m
            self._used = [int(v) for v in torch.cat([o[m:m + 1] for o in out.off]).cpu().numpy()]
            self._rebuild()
        with torch.cuda.device(self.dev):
            ev1.record()
        ev1.synchronize()
        self.timings_ms["compact_ms"] = ev0.elapsed_time(ev1)

    def _rebuild(self):
        """time order, path resolution and the per-event columns of the window graph over the resident events"""
        import ctypes as C
        from . import _lib
        torch = self.torch
        dev, n, dc = self.dev, self.n, self._dc
        ev0 = torch.cuda.Event(enable_timing=True); ev1 = torch.cuda.Event(enable_timing=True)
        with torch.cuda.device(dev):
            ev0.record()
        need = C.c_int64()
        _lib.check(_lib.lib().nerrf_trace_stream_order_workspace_bytes(n, C.byref(need)), "stream_order_workspace_bytes")
        ws = torch.empty(need.value + 256, dtype=torch.uint8, device=dev)
        e = lambda dt, k=n: torch.empty(max(k, 1), dtype=dt, device=dev)
        ts, order, ts_sorted, src, retain = e(torch.float64), e(torch.int64), e(torch.float64), e(torch.int64), e(torch.int64)
        res_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        counts = (C.c_int64 * 3)()
        poff, pdata, goff, gdata = dc.off[2], dc.data[2], dc.off[3], dc.data[3]
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().nerrf_trace_stream_order_ex(
                n, _lib.ptr(dc.s["ts_sec"]), _lib.ptr(dc.s["ts_nanos"]), _lib.ptr(dc.s["pid"]), _lib.ptr(dc.source), self._key_bits,
                _lib.ptr(poff), float(self._horizon), _lib.ptr(ts), _lib.ptr(order), _lib.ptr(ts_sorted), _lib.ptr(src),
                _lib.ptr(res_off), _lib.ptr(retain), counts, C.c_void_p((ws.data_ptr() + 255) & ~255), need.value,
                _lib.current_stream_ptr()), "nerrf_trace_stream_order_ex")
        n_keep, n_retain, pbytes = int(counts[0]), int(counts[1]), int(counts[2])
        res_data = torch.zeros(max(pbytes, 1), dtype=torch.uint8, device=dev)
        pf, pf_raw, slot = e(torch.uint8), e(torch.uint8), e(torch.uint8)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().nerrf_trace_stream_columns(
                n, _lib.ptr(src), _lib.ptr(poff), _lib.ptr(pdata), _lib.ptr(dc.s["path_flags"]), _lib.ptr(goff), _lib.ptr(gdata),
                _lib.ptr(dc.s["event_slot"]), _lib.ptr(self._slot_map), _lib.ptr(res_off), int(self.merge), _lib.ptr(res_data),
                _lib.ptr(pf), _lib.ptr(pf_raw), _lib.ptr(slot), _lib.current_stream_ptr()), "nerrf_trace_stream_columns")
            ev1.record()
        self.n_keep, self._n_retain, self._retain = n_keep, n_retain, retain[:n_retain]
        self.d_order, self.d_ts_sorted, self.d_ts = order[:n_keep], ts_sorted[:n_keep], ts
        self.d_pid, self.d_poff, self.d_pdata, self.d_goff, self.d_gdata = dc.s["pid"], res_off, res_data, goff, gdata
        self.d_source = dc.source
        self.d_raw_slot, self.d_slot, self.d_bytes, self.d_pf, self.d_pf_raw = dc.s["event_slot"], slot, dc.s["bytes"], pf, pf_raw
        self._flow = None                                      # rows changed: flow() recomputes on first use
        if n_keep:
            lohi = torch.stack([ts_sorted[0], ts_sorted[n_keep - 1]]).cpu().numpy()
            self._span = (float(lohi[0]), float(lohi[1]))
        else:
            self._span = (0.0, 0.0)
        self._alloc_intern(max(n, 1))
        ev1.synchronize()
        self.timings_ms["rebuild_ms"] = self.timings_ms.get("rebuild_ms", 0.0) + ev0.elapsed_time(ev1)

    def flow(self):
        """uint8 [rows] the information-flow class of every stored event (DESIGN.md 1.5), kept resident once asked for:
        uploaded from the host columns of a whole-trace stream, computed on the device from the live decoder's
        event_slot / flags / ret_val columns (nerrf_trace_flow_class_device) until the stream changes"""
        if self._flow is None:
            torch = self.torch
            if self.cols is not None:
                self._flow = torch.from_numpy(ingest.column_flow(self.cols)).to(self.dev)
            else:
                from . import _lib
                dc, n = self._dc, self.n
                flow = torch.empty(max(n, 1), dtype=torch.uint8, device=self.dev)
                with torch.cuda.device(self.dev):
                    _lib.check(_lib.lib().nerrf_trace_flow_class_device(_lib.ptr(dc.s["event_slot"]), _lib.ptr(dc.s["flags"]),
                                                                        _lib.ptr(dc.s["ret_val"]), n, _lib.ptr(flow),
                                                                        _lib.current_stream_ptr()), "nerrf_trace_flow_class_device")
                self._flow = flow
        return self._flow

    def _alloc_intern(self, n):
        """node tables and interning workspace for windows of up to n events"""
        import ctypes as C
        from . import _lib
        torch = self.torch
        if getattr(self, "node_p", None) is not None and self.node_p.shape[0] >= n:
            return
        n = max(n, 2 * getattr(self, "node_p", torch.empty(0)).shape[0])
        self.cap = max((2 if self.merge else 3) * n, 1)
        self.node_p = torch.empty(n, dtype=torch.int32, device=self.dev)
        self.node_f = torch.empty_like(self.node_p); self.node_g = torch.empty_like(self.node_p)
        self.kind = torch.zeros(self.cap, dtype=torch.int8, device=self.dev)
        self.name_event = torch.zeros(self.cap, dtype=torch.int64, device=self.dev)
        self.name_which = torch.zeros(self.cap, dtype=torch.int8, device=self.dev)
        need = C.c_int64()
        _lib.check(_lib.lib().nerrf_trace_intern_device_workspace_bytes(n, self.cap, C.byref(need)), "intern_device_workspace_bytes")
        self._ws = torch.empty(need.value + 256, dtype=torch.uint8, device=self.dev)
        self._ws_bytes = need.value

    def span(self):
        if self.cols is None:                                  # live stream: first and last surviving event
            return self._span
        if self.n == 0:
            return 0.0, 0.0
        return float(self.ts_sorted[0]), float(self.ts_sorted[-1])

    def _window_ranks(self, t_lo: float, t_hi: float):
        """-> (lo, hi, ts of rank lo, ts of rank hi - 1): the window's slice of the time-sorted survivors"""
        if self.cols is not None:
            lo = int(np.searchsorted(self.ts_sorted, t_lo, "right")); hi = int(np.searchsorted(self.ts_sorted, t_hi, "right"))
            if hi <= lo:
                return lo, hi, None, None
            return lo, hi, float(self.ts_sorted[lo]), float(self.ts_sorted[hi - 1])
        torch = self.torch
        if self.n_keep == 0:
            return 0, 0, None, None
        b = torch.searchsorted(self.d_ts_sorted, torch.tensor([t_lo, t_hi], dtype=torch.float64, device=self.dev), right=True)
        lo, hi = (int(v) for v in b.cpu().numpy())
        if hi <= lo:
            return lo, hi, None, None
        v = self.d_ts_sorted[torch.tensor([lo, hi - 1], device=self.dev)].cpu().numpy()
        return lo, hi, float(v[0]), float(v[1])

    def window_graph(self, t_lo: float, t_hi: float, window_s: float, edge_labels: bool = False):
        """The temporal graph of the events with t_lo < t <= t_hi (device tensors), or None when there are none.
        Same construction as ingest.graph_from_columns(stream.window(cols, t_lo, t_hi), device=...).
        edge_labels=True also attaches meta['edge_label'] (uint8 [E] CUDA tensor, CSR order: graph_from_events' per-pair
        rule, from the annotation slots; graph.edge_labels_device) -- the edge head's training target."""
        import ctypes as C
        from . import _lib
        torch = self.torch
        lo, hi, t_first, t_last = self._window_ranks(t_lo, t_hi)
        nw = hi - lo
        if nw <= 0:
            return None
        sel = self.d_order[lo:hi]                                   # the window = a slice of the time-sorted index array
        nn = C.c_int64()
        ws_ptr = (self._ws.data_ptr() + 255) & ~255
        with torch.cuda.device(self.dev):
            _lib.check(_lib.lib().nerrf_trace_intern_device_ex(
                nw, self.n, _lib.ptr(sel), _lib.ptr(self.d_pid), _lib.ptr(self.d_source), _lib.ptr(self.d_poff), _lib.ptr(self.d_pdata),
                _lib.ptr(self.d_goff), _lib.ptr(self.d_gdata), int(self.merge), _lib.ptr(self.node_p), _lib.ptr(self.node_f),
                _lib.ptr(self.node_g), C.byref(nn), _lib.ptr(self.kind), _lib.ptr(self.name_event), _lib.ptr(self.name_which),
                self.cap, C.c_void_p(ws_ptr), self._ws_bytes, _lib.current_stream_ptr()), "nerrf_trace_intern_device_ex")
        N = int(nn.value)
        t0 = t_first; span = max(t_last - t0, 1e-6)
        window = window_s or max(span, G.WINDOW)
        P, F = self.node_p[sel], self.node_f[sel]                   # by rank: the window's events in time order
        t = self.d_ts[sel] - t0
        kind_d = self.kind[:N].contiguous()
        Gn = None
        if not self.merge:
            Gn = self.node_g[sel]
            if not bool((Gn >= 0).any()):
                Gn = None
        x, label, size_mb = G.node_features_device(P, F, Gn, t, self.d_slot[sel], self.d_bytes[sel], self.d_pf[sel], kind_d, window)
        tt = t.to(torch.float32)
        if Gn is None:                                              # edges in the host loader's per-event order: p->f, f->p
            src = torch.stack([P, F], 1).reshape(-1); dst = torch.stack([F, P], 1).reshape(-1)
            te = tt.repeat_interleave(2)
        else:                                                       # [, f->g, g->f]
            keep = torch.stack([torch.ones_like(P, dtype=torch.bool)] * 2 + [Gn >= 0] * 2, 1).reshape(-1)
            src = torch.stack([P, F, F, Gn], 1).reshape(-1)[keep]; dst = torch.stack([F, P, Gn, F], 1).reshape(-1)[keep]
            te = tt.repeat_interleave(4)[keep]
        rowptr, col, ew, perm = G.build_csr_device(src.contiguous(), dst.contiguous(), te.contiguous(), torch.ones_like(te), N,
                                                   t_ref=float(span), tau=G.TAU, return_perm=True)
        lab = label
        if self.observable:                                         # the kernel saw the folded slots: labels come from the annotations
            raw = self.d_raw_slot[sel]
            lab = (torch.bincount(F[(raw == 1) | (raw == 2)].long(), minlength=N) > 0)
        nh = torch.empty(N, dtype=torch.int64, device=self.dev)
        with torch.cuda.device(self.dev):
            _lib.check(_lib.lib().nerrf_trace_name_hash_ex(N, _lib.ptr(self.name_event), _lib.ptr(self.name_which), _lib.ptr(self.d_pid),
                                                           _lib.ptr(self.d_source), _lib.ptr(self.d_poff), _lib.ptr(self.d_pdata),
                                                           _lib.ptr(self.d_goff), _lib.ptr(self.d_gdata), _lib.ptr(nh),
                                                           _lib.current_stream_ptr()), "nerrf_trace_name_hash_ex")
        bufs = (self.name_event, self.name_which, self.d_pid, self.d_source, self.d_poff, self.d_pdata, self.d_goff, self.d_gdata)

        def dir_hash_device(bufs=bufs):
            """int64 [N] parent-directory hash of every node (nerrf_trace_dir_hash); valid until the stream changes."""
            dh = torch.empty(N, dtype=torch.int64, device=self.dev)
            with torch.cuda.device(self.dev):
                _lib.check(_lib.lib().nerrf_trace_dir_hash_ex(N, *(_lib.ptr(b) for b in bufs), _lib.ptr(dh), _lib.current_stream_ptr()),
                           "nerrf_trace_dir_hash_ex")
            return dh
        ne, nwh = self.name_event[:N].cpu().numpy(), self.name_which[:N].cpu().numpy()
        node_source = np.zeros(N, np.int64) if self.d_source is None else \
            (self.d_source[self.name_event[:N]].to(torch.int64) & 0xffff).cpu().numpy()
        names = LazyNames(self.cols, ne, nwh) if self.cols is not None else \
            DeviceNames(self.d_pid, self.d_poff, self.d_pdata, self.d_goff, self.d_gdata, ne, nwh)
        meta = {"kind": "trace", "names": names,
                "node_kind": kind_d.cpu().numpy().astype(np.int64), "t0": t0, "span": span, "merge_renames": self.merge,
                "label": lab.cpu().numpy().astype(np.int64), "size_mb": size_mb.cpu().numpy(), "device": str(self.dev),
                "name_hash": nh, "dir_hash": dir_hash_device, "events": nw, "node_source": node_source, "window_ranks": (lo, hi), "perm": perm if Gn is None else None}
        per_event = 2 if Gn is None else 4

        def edge_event(perm=perm, sel=sel, keep=None if Gn is None else keep):
            """the event (stream row) that made each CSR edge"""
            if perm.numel() != col.numel():                                 # E = 0: perm holds one spare entry
                return torch.zeros(0, dtype=torch.int64, device=self.dev)
            rank = torch.arange(nw, device=self.dev).repeat_interleave(per_event)
            return sel[(rank if keep is None else rank[keep])[perm.long() & 0xffffffff]]

        def edge_time():
            """the trace-clock seconds (float64) of the event that made each CSR edge, gathered on the device"""
            return self.d_ts[edge_event()]

        def edge_flow():
            """the information-flow class (uint8, DESIGN.md 1.5) of the event that made each CSR edge, gathered on the device"""
            return self.flow()[edge_event()]
        meta.update(edge_event=edge_event, edge_time=edge_time, edge_flow=edge_flow, event_info=self.event_records)
        if edge_labels:
            meta["edge_label"] = G.edge_labels_device(P, F, self.d_raw_slot[sel], rowptr, col, N)
        return G.TemporalGraph(rowptr, col, ew, x, meta)

    def event_records(self, rows) -> list:
        """graph.event_record of stream rows `rows` (valid until the stream is compacted), plus "source" for a stream of
        several sources.  A live stream holds no syscall strings: its records name the event kind of the row's slot."""
        rows = np.asarray(rows, np.int64)
        if self.cols is not None:
            recs = ingest.column_event_records(self.cols, rows)
            if not self.multi_source:
                for r in recs:
                    r.pop("source", None)
            return recs
        torch = self.torch
        r = torch.from_numpy(rows).to(self.dev)
        ts, pid = self.d_ts[r].cpu().numpy(), self.d_pid[r].cpu().numpy().view(np.uint32)
        slot = self.d_raw_slot[r].cpu().numpy()
        po = self.d_poff[torch.stack([r, r + 1], 1)].cpu().numpy() if rows.size else np.zeros((0, 2), np.int64)
        src = None if self.d_source is None or not self.multi_source else (self.d_source[r].to(torch.int64) & 0xffff).cpu().numpy()
        kinds = {v: k for k, v in G._EVENT_SLOT.items()}
        out = []
        for k in range(rows.size):
            a, b = int(po[k, 0]), int(po[k, 1])
            path = bytes(self.d_pdata[a:b].cpu().numpy()).decode("utf-8", "replace") if b > a else ""
            rec = {"time": float(ts[k]), "pid": int(pid[k]), "syscall": kinds.get(int(slot[k]), "other"), "path": path}
            if src is not None:
                rec["source"] = int(src[k])
            out.append(rec)
        return out

    def sequences_device(self, g: G.TemporalGraph, only_nodes, events=False):
        """LSTM sequences of the given file nodes of window graph `g`, built ON THE DEVICE (nerrf_trace_sequences) from the
        resident columns and the graph's own CSR rows: -> (seq fp32 [A, T_MAX, 16], lengths int32 [A]) CUDA tensors in the
        order of `only_nodes`.  Needs the two-edges-per-event graph of merge mode (g.meta['perm']).
        events=True: also the stream row of each step's event (int64 [A, T_MAX], -1 at padded steps; the ids of
        g.meta["edge_event"] / event_records), from nerrf_trace_sequences_ex."""
        import ctypes as C
        from . import _lib
        from .ai.models import lstm
        torch = self.torch
        perm = g.meta.get("perm")
        if perm is None:
            raise _lib.NerrfError("sequences_device needs a merge-mode window graph (two edges per event)")
        lo, hi = g.meta["window_ranks"]
        only_nodes = np.asarray(only_nodes, np.int64).reshape(-1)
        if only_nodes.size and (only_nodes.min() < 0 or only_nodes.max() >= g.num_nodes):   # the kernel reads rowptr[f], rowptr[f + 1]
            raise _lib.NerrfError("sequences_device: candidate node ids must lie in [0, %d)" % g.num_nodes)
        cand = torch.as_tensor(only_nodes).to(self.dev)
        A = int(cand.shape[0])
        seq = torch.empty(A, lstm.T_MAX, lstm.D_IN, dtype=torch.float32, device=self.dev)
        ln = torch.empty(A, dtype=torch.int32, device=self.dev)
        ev = torch.empty(A, lstm.T_MAX, dtype=torch.int64, device=self.dev) if events else None
        with torch.cuda.device(self.dev):
            _lib.check(_lib.lib().nerrf_trace_sequences_ex(_lib.ptr(cand), A, _lib.ptr(g.rowptr), int(g.rowptr.dtype == torch.int64),
                                                           _lib.ptr(perm), _lib.ptr(self.d_order[lo:hi]), _lib.ptr(self.d_ts),
                                                           _lib.ptr(self.d_slot), _lib.ptr(self.d_bytes), _lib.ptr(self.d_pf_raw),
                                                           float(g.meta["t0"]), float(g.meta["span"]), lstm.T_MAX, _lib.ptr(seq),
                                                           _lib.ptr(ln), _lib.ptr(ev), _lib.current_stream_ptr()),
                       "nerrf_trace_sequences_ex")
        return (seq, ln, ev) if events else (seq, ln)

    def sequences(self, g: G.TemporalGraph, only_nodes, events=False):
        """LSTM sequences of the given file nodes of window graph `g` (ingest.sequences_core on the window's events);
        events=True: also the stream row of each step's event (sequences_core(return_events=True))."""
        if self.cols is None:
            from . import _lib
            raise _lib.NerrfError("a live stream builds its sequences on the device (sequences_device)")
        lo, hi = g.meta["window_ranks"]
        order = self.order[lo:hi]
        if "_F_host" not in g.meta:
            g.meta["_F_host"] = self.node_f[self.d_order[lo:hi]].cpu().numpy().astype(np.int64)
        return ingest.sequences_core(self.cols, order, g.meta["_F_host"], self.ts_sorted[lo:hi], g.meta["t0"], g.meta["span"],
                                     g.num_nodes, None, self.observable, only_nodes, events)


@dataclass
class TickResult:
    t_hi: float
    events: int
    nodes: int
    edges: int
    planned: list                  # paths this tick's plan reverts (new ones only); (host, path) with several sources
    timings_ms: dict
    truncated: bool = False
    restored: list = field(default_factory=list)   # directories this tick's plan restores from the snapshot
    evidence: dict = field(default_factory=dict)   # StreamingPlanner(explain=k): plan key of each node step this tick
                                                   # planned (as in `planned`, kills included) -> its explanation
    sequence_evidence: dict = field(default_factory=dict)   # StreamingPlanner(explain_sequences=k): plan key of each file
                                                            # step this tick planned -> the BiLSTM explanation of its sequence
    incidents: dict = field(default_factory=dict)   # StreamingPlanner(incidents=True): incident id -> this tick's record
                                                    # (incident.incidents; "files" as plan keys)
    step_incident: dict = field(default_factory=dict)   # StreamingPlanner(incidents=True): plan key of each step this tick
                                                        # planned (as in `planned`, kills included) -> its incident id
    contamination: dict = field(default_factory=dict)   # StreamingPlanner(contamination=True): incident id -> this tick's
                                                        # contaminated nodes (taint.contamination; "key" = the node's plan key)


@dataclass
class StreamingPlanner:
    """Tick loop: every `tick_s` seconds of trace time the events of the last `window_s` seconds become a temporal graph
    (features + CSR on the GPU), GraphSAGE_T scores it, the top-A anomalous files that were not reverted yet go
    through the LSTM and the MCTS planner, and the resulting reversions are added to the running undo plan."""
    model: object
    scorer: object
    window_s: float = 60.0
    tick_s: float = 30.0
    top_a: int = 4096
    n_rollouts: int = 1024
    depth: int = 32
    iterations: int = 8
    commit_per_search: int = 64
    kill_candidates: bool = False  # also propose "kill process" actions (planner spec v1: reversions need their writer gone)
    restore_candidates: bool = False   # also propose directory restores (planner spec v2, one GPU); covered files count as reverted
    max_restores: int = 4
    min_restore_files: int = 8
    explain: int = 0               # k > 0: each tick's TickResult.evidence explains its new steps (pipeline.run(explain=k))
    explain_sequences: int = 0     # k > 0: TickResult.sequence_evidence explains its new file steps' sequences (one GPU)
    incidents: object = False      # True: ticks label their steps with incidents (pipeline.run(incidents=True), one GPU);
                                   # then, from construction on, the running incidents: id -> {"id", "host", "process",
                                   # "onset" / "onset_event" (min over ticks), "end" / "end_event" (max), "files" (union
                                   # of plan keys), "n_files"}
    incident_tau: float = 0.5
    contamination: object = False  # True (needs incidents): TickResult.contamination lists what each incident spread to
                                   # (pipeline.run(contamination=True)); then, from construction on, the running records:
                                   # incident id -> {node key: record with the earliest "since" over ticks}
    contamination_hops: int = -1
    device: str = "cuda"
    dist_ctx: object = None        # pipeline.DistContext for the multi-GPU form
    reverted: set = field(default_factory=set)
    _reverted_hash: set = field(default_factory=set)
    ingest_ms: float = 0.0         # one-time: stream columns -> HBM (DeviceStream)
    killed: set = field(default_factory=set)
    restored_dirs: list = field(default_factory=list)
    ticks: list = field(default_factory=list)
    lateness_s: float = 0.0        # live feed: a tick at t_hi fires once every open source has delivered an event with ts > t_hi + lateness_s
    live: object = None            # live feed: the DeviceStream the bytes go to
    sources: dict = field(default_factory=dict)    # source name -> source id (add_source); ids number the hosts from 0
    _open: set = field(default_factory=set)        # ids of the sources the watermark waits for
    _latest: dict = field(default_factory=dict)    # source id -> latest event time it delivered
    _carry: dict = field(default_factory=dict)     # source id -> cut-off record bytes carried to its next chunk
    _names: list = field(default_factory=list)     # source id -> name
    _host_keys: bool = None        # plan names are (host, name) pairs: fixed by the first tick, for the planner's lifetime
    _t0: float = None
    _t_hi: float = None

    def __post_init__(self):
        if isinstance(self.incidents, bool):
            self.incidents = {} if self.incidents else None
        if isinstance(self.contamination, bool):
            if self.contamination and self.incidents is None:
                raise ValueError("contamination=True needs incidents=True (the closure is seeded by the incidents)")
            self.contamination = {} if self.contamination else None

    def add_source(self, name: str) -> int:
        """Register a source (a host's tracker stream) -> its id (the next free one; an existing name keeps its id).
        Names are 1-64 characters of [A-Za-z0-9._-], not "." or "..": they name per-host plan files.
        Register every host before feeding: the watermark only waits for registered sources.  A host registered after
        ticks have fired joins the watermark from then on, and its events at or before the last tick are late data (later
        windows hold them, fired ticks do not).  A second source cannot join once ticks have fired with one, whose plans
        name files without a host: that raises ValueError."""
        from .ai.planner import emit
        emit.check_host_name(name)
        if name not in self.sources:
            if len(self.sources) >= (1 << 16):
                raise ValueError("at most 65536 sources")
            if self._host_keys is False:
                raise ValueError("source %r registered after ticks fired with one source: register every source before "
                                 "the first tick" % name)
            self.sources[name] = len(self._names)
            self._names.append(name)
            self._open.add(self.sources[name])
        return self.sources[name]

    def host_name(self, source: int) -> str:
        """the registered name of source id `source` (its decimal id when it has none)"""
        return self._names[source] if 0 <= source < len(self._names) else str(int(source))

    def feed(self, chunk, source: str = "default") -> list:
        """Live form of run(): `chunk` = the next bytes of source `source`'s EventBatch stream (registered on first use;
        with several hosts, register them all with add_source before the first chunk), cut anywhere: a partial record is carried over to that source's next call, never glued to another source's bytes.
        The bytes are decoded and appended on the device; every tick that can no longer change fires: with several
        sources, once every open source has delivered an event past it (the low watermark).  -> the TickResults fired by
        this call.  Ticks, windows and plans are those run() computes over the whole stream when no event arrives more
        than lateness_s late."""
        if self.dist_ctx is not None and self.dist_ctx.world > 1:
            raise NotImplementedError("live feeding runs on one GPU")
        sid = self.add_source(source)
        if sid not in self._open:
            raise ValueError("source %r was closed" % source)
        if self.live is None:
            self.live = DeviceStream.live(self.device, observable=True)
        buf = self._carry.get(sid, b"") + bytes(chunk)
        used = self.live.append(buf, partial=True, source=sid)
        self._carry[sid] = buf[used:]
        self._note_latest(sid)
        return self._fire(final=False)

    def _note_latest(self, sid: int):
        a, b = self.live.appended
        if b > a:
            t = float(self.live.d_ts[a:b].max())
            self._latest[sid] = max(self._latest.get(sid, -np.inf), t)

    def close_source(self, name: str) -> list:
        """Source `name` has ended: the watermark stops waiting for it.  A carried-over partial record of it is malformed
        input.  -> the TickResults this releases."""
        sid = self.sources[name]
        if self._carry.get(sid):
            self.live.append(self._carry[sid], source=sid)    # raises: the source ended inside a record
        self._carry[sid] = b""
        self._open.discard(sid)
        if self.live is None:
            return []
        return self._fire(final=False)

    def flush(self) -> list:
        """End of the stream (of every source): fire the remaining ticks, the last one at the last event (like run()).
        A carried-over partial record is malformed input."""
        if self.live is None:
            return []
        for sid, rest in self._carry.items():
            if rest:
                self.live.append(rest, source=sid)             # raises: the stream ended inside a record
        return self._fire(final=True)

    def _fire(self, final: bool) -> list:
        import torch
        ds, out = self.live, []
        dev = torch.device(self.device)
        while ds.n_keep:
            first, last = ds.span()
            t0 = self._t0 if self._t0 is not None else first     # fixed by the first tick: earlier events have arrived
            t_hi = self._t_hi if self._t_hi is not None else t0
            if final:
                if not t_hi < last:
                    break
                nxt = min(t_hi + self.tick_s, last)
            else:
                nxt = t_hi + self.tick_s
                mark = last                                      # one source: the latest surviving event
                if len(self.sources) > 1 and self._open:         # several: the low watermark over the open sources
                    mark = min(self._latest.get(sid, -np.inf) for sid in self._open)
                if not mark > nxt + self.lateness_s:
                    break
            self._t0, self._t_hi = t0, nxt
            k = len(self.ticks)
            self._tick(ds, nxt, t0, dev, True, False, None)
            out += self.ticks[k:]
            ds.compact(nxt - self.window_s)                      # no later window reaches back past this tick's
        return out

    def run(self, cols: ingest.EventColumns):
        """cols: the event stream (multi-GPU: only rank 0's copy is read -- rank 0 does the host-side ingest of every tick
        and broadcasts the device graph, the exclusion mask and the candidates' sequences; names stay on rank 0)."""
        import time
        import torch
        ctx = self.dist_ctx
        multi = ctx is not None and ctx.world > 1
        if multi and self.restore_candidates:
            raise NotImplementedError("restore candidates are planned on one GPU (dist_ctx.world > 1 is not supported)")
        if multi and (self.explain or self.explain_sequences):
            raise NotImplementedError("explanations are computed on one GPU (dist_ctx.world > 1 is not supported)")
        if multi and self.incidents is not None:
            raise NotImplementedError("incidents are computed on one GPU (dist_ctx.world > 1 is not supported)")
        lead = not multi or ctx.rank == 0
        dev = torch.device(self.device)
        if multi:
            import torch.distributed as dist

            def bcast(t, shape=None, dtype=None):
                """broadcast a tensor from rank 0 (shape / dtype known to everybody, or sent first)"""
                if shape is None:
                    hdr = torch.tensor(list(t.shape) + [-1] * (4 - t.dim()) if lead else [0] * 4, device=dev, dtype=torch.int64)
                    dist.broadcast(hdr, 0)
                    shape = [int(v) for v in hdr.tolist() if v >= 0]
                buf = t.to(dev).contiguous() if lead else torch.empty(shape, device=dev, dtype=dtype)
                dist.broadcast(buf, 0)
                return buf
        ds = None
        if lead:
            # the stream becomes device resident ONCE (in production: batch by batch as the tracker delivers it); from here
            # on a tick touches no string on the host except the names of the nodes its plan reverts
            a = time.perf_counter()
            ds = DeviceStream(cols, self.device, observable=True)
            torch.cuda.synchronize()
            self.ingest_ms = (time.perf_counter() - a) * 1e3
            span = torch.tensor(list(ds.span()), dtype=torch.float64, device=dev)
        else:
            span = torch.zeros(2, dtype=torch.float64, device=dev)
        if multi:
            dist.broadcast(span, 0)
        t0, t1 = float(span[0]), float(span[1])
        t_hi = t0
        while t_hi < t1:
            t_hi = min(t_hi + self.tick_s, t1)
            self._tick(ds, t_hi, t0, dev, lead, multi, bcast if multi else None)
        return self.ticks

    def _tick(self, ds, t_hi, t0, dev, lead, multi, bcast):
        """One tick: the window (t_hi - window_s, t_hi] becomes a graph, is scored and planned; appends a TickResult
        (nothing when the window is empty).  Shared by run() and the live loop (feed / flush)."""
        from . import pipeline
        import time
        import torch
        if multi:
            import torch.distributed as dist
        tm = {}
        names, g, n_events = None, None, 0
        a = time.perf_counter()
        if lead:
            # window = a slice of the time-sorted index array; interning (hash table), features, edges, CSR on the GPU
            g = ds.window_graph(t_hi - self.window_s, t_hi, self.window_s)
            torch.cuda.synchronize()
            n_events = g.meta["events"] if g is not None else 0
        if multi:
            ne = torch.tensor([n_events], device=dev); dist.broadcast(ne, 0); n_events = int(ne)
        if n_events == 0:
            return
        if lead:
            names = g.meta["names"]
        if multi:                                      # the device graph travels over NVLink; the strings do not
            x = bcast(g.x if lead else None, dtype=torch.float32)
            rp = bcast(g.rowptr.to(torch.int64) if lead else None, dtype=torch.int64).to(torch.int32)
            col = bcast(g.col if lead else None, dtype=torch.int32)
            ew = bcast(g.ew if lead else None, dtype=torch.float32)
            kind_t = bcast(torch.from_numpy(np.asarray(g.meta["node_kind"]).astype(np.int64)) if lead else None, dtype=torch.int64)
            size_t = bcast(torch.from_numpy(np.asarray(g.meta["size_mb"], np.float32)) if lead else None, dtype=torch.float32)
            if not lead:
                g = G.TemporalGraph(rp, col, ew, x, {"kind": "trace", "node_kind": kind_t.cpu().numpy(), "size_mb": size_t.cpu().numpy()})
        tm["graph_build"] = (time.perf_counter() - a) * 1e3
        kind = np.asarray(g.meta["node_kind"])
        nodes = np.nonzero(kind == 0)[0]

        # LSTM sequences are built lazily, for the top-A candidates only (a window holds ~10^6 file nodes)
        def seq(cand, g=g, events=False):
            if lead and not multi:                      # built on the device from the resident columns, in candidate order
                if events:                              # (explain_sequences: one GPU, so never the multi-GPU branch below)
                    sq_d, ln_d, ev_d = ds.sequences_device(g, cand, events=True)
                    return sq_d, ln_d, None, ev_d
                sq_d, ln_d = ds.sequences_device(g, cand)
                return sq_d, ln_d, None
            if lead:
                sq, ln, have = ds.sequences(g, cand)
            if multi:
                sq_t = bcast(torch.from_numpy(sq) if lead else None, dtype=torch.float32)
                ln_t = bcast(torch.from_numpy(ln) if lead else None, dtype=torch.int32)
                hv_t = bcast(torch.from_numpy(have) if lead else None, dtype=torch.int64)
                return sq_t.cpu().numpy(), ln_t.cpu().numpy(), hv_t.cpu().numpy()
            return sq, ln, have

        new, truncated, restored, evidence, seq_evidence, tick_inc, step_inc = [], False, [], {}, {}, {}, {}
        tick_nodes = {}                                  # incident id -> node ids of its tick record
        tick_cont = {}                                   # incident id -> {node key: contaminated record}
        want_cont = self.contamination is not None
        want_inc = self.incidents is not None
        if lead and self._host_keys is None:             # decided once per planner, so reverted / killed hold one form
            self._host_keys = len(self.sources) > 1 or ds.multi_source
        inc_hosts = None
        if want_inc and lead and self._host_keys:
            node_src = np.asarray(g.meta["node_source"])
            inc_hosts = [self.host_name(s_) for s_ in range(max(len(self._names), int(node_src.max(initial=0)) + 1))]
        for rnd in range(4):
            # a planning pass proposes at most 32 process kills (planner spec v1: guards live in state word 0); a tick
            # with more suspicious processes than that plans again over what is still unreverted
            skip = None
            if lead and self.reverted:               # files already reverted by an earlier tick: matched by name hash on the device
                rh = torch.tensor(sorted(self._reverted_hash), dtype=torch.int64, device=dev)
                skip = torch.isin(g.meta["name_hash"][torch.from_numpy(nodes).to(dev)], rh).cpu().numpy()
            if multi:
                flag = torch.tensor([1 if (lead and skip is not None) else 0], device=dev); dist.broadcast(flag, 0)
                if int(flag):
                    skip = bcast(torch.from_numpy(skip) if lead else None, shape=[nodes.shape[0]], dtype=torch.bool).cpu().numpy()
            res = pipeline.run(g, seq, None, nodes, self.model, self.scorer, top_a=self.top_a, n_rollouts=self.n_rollouts,
                               depth=self.depth, iterations=self.iterations, device=self.device, exclude=skip,
                               commit_per_search=self.commit_per_search, dist_ctx=self.dist_ctx,
                               kill_candidates=self.kill_candidates, restore_candidates=self.restore_candidates,
                               max_restores=self.max_restores, min_restore_files=self.min_restore_files, explain=self.explain,
                               explain_sequences=self.explain_sequences, incidents=want_inc, incident_tau=self.incident_tau,
                               host_names=inc_hosts, contamination=want_cont, contamination_hops=self.contamination_hops)
            for k, v in res.timings_ms.items():
                tm[k] = tm.get(k, 0.0) + float(v)
            got = []
            if lead:
                node_src = g.meta.get("node_source")
                multi_src = self._host_keys
                # several sources: a file or process is named (host, name), and its hash is qualified by its source
                key = (lambda n, nm: (self.host_name(int(node_src[n])), nm)) if multi_src else (lambda n, nm: nm)
                src_of = (lambda n: int(node_src[n])) if multi_src else (lambda n: 0)

                def revert(nodes, node_names):
                    """mark the files not reverted yet as reverted -> their keys, in plan order"""
                    fresh = {}
                    for n, nm in zip(nodes, node_names):
                        if kind[n] == 0 and key(n, nm) not in self.reverted:
                            fresh.setdefault(key(n, nm), name_hash(nm, src_of(n)))
                    self.reverted.update(fresh)
                    self._reverted_hash.update(fresh.values())
                    return list(fresh)
                plan_names = names.take(res.plan_nodes)           # one bulk fetch (device names of a live stream)
                fresh_kills = [key(n, nm) for n, nm in zip(res.plan_nodes, plan_names) if kind[n] == 1 and key(n, nm) not in self.killed]
                self.killed.update(key(n, nm) for n, nm in zip(res.plan_nodes, plan_names) if kind[n] == 1)
                got = revert(res.plan_nodes, plan_names)
                if res.evidence is not None:
                    fresh = set(got) | set(fresh_kills)
                    for n, nm in zip(res.plan_nodes, plan_names):
                        if key(n, nm) in fresh and key(n, nm) not in evidence:
                            evidence[key(n, nm)] = res.evidence.get(n)
                if res.sequence_evidence is not None:
                    fresh = set(got)
                    for n, nm in zip(res.plan_nodes, plan_names):
                        if key(n, nm) in fresh and key(n, nm) not in seq_evidence and n in res.sequence_evidence:
                            seq_evidence[key(n, nm)] = res.sequence_evidence[n]
                if res.incidents is not None:
                    self._note_incidents(res, g, names, key, set(got) | set(fresh_kills), plan_names, tick_inc, tick_nodes, step_inc)
                if res.contamination is not None:
                    self._note_contamination(res, key, tick_cont)
                new += got
                for r in res.restores:                         # a restored directory brings back every file it covers
                    cov = revert(r["covers"], names.take(r["covers"]))
                    d = key(r["covers"][0], r["dir"]) if r["covers"] else r["dir"]
                    restored.append(d); self.restored_dirs.append(d)
                    got = got + cov
            # a pass proposes at most 32 - (restores) kills (word 0 holds both): plan again while the budget was used up
            more = bool(self.kill_candidates and res.n_kill >= 32 - res.n_restore and got)
            if multi:
                flag = torch.tensor([int(more)], device=dev); dist.broadcast(flag, 0); more = bool(int(flag))
            truncated = truncated or bool(res.plan.truncated)
            if not more:
                break
        tick_cont = {i: sorted(recs.values(), key=lambda r: (r["since"], str(r["key"]))) for i, recs in tick_cont.items()}
        self.ticks.append(TickResult(t_hi - t0, n_events, g.num_nodes, g.num_edges, new, tm, truncated, restored, evidence,
                                     seq_evidence, tick_inc, step_inc, tick_cont))

    def _note_contamination(self, res, key, tick_cont):
        """this planning pass's contamination -> the tick's records (a later pass of the same tick adds its new nodes and
        keeps the earlier "since" of a node both passes reach) and the running records (earliest "since" per (incident,
        node key) over ticks)"""
        for i, recs in res.contamination.items():
            tick = tick_cont.setdefault(i, {})
            run = self.contamination.setdefault(i, {})
            for r in recs:
                k = key(r["node"], r["name"])
                rec = dict(r, key=k)
                for into in (tick, run):
                    if k not in into or rec["since"] < into[k]["since"]:
                        into[k] = rec

    _RUNNING_FIELDS = ("id", "host", "process", "onset", "onset_event", "end", "end_event", "files", "n_files")

    def _note_incidents(self, res, g, names, key, fresh, plan_names, tick_inc, tick_nodes, step_inc):
        """this planning pass's incidents -> the tick's records (files as plan keys), the fresh steps' incident ids, and the
        running records.  A later pass of the same tick (same window, more seeds) folds its new files into the tick's
        record: n_files, size_mb, later_other_events and max_score over the union, onset min, end max.  Running records
        keep the fields that fold across windows: onset min, end max, files (plan keys) union."""
        size = np.asarray(g.meta["size_mb"], np.float32)
        score = res.node_score.detach().cpu().numpy()
        for r in res.incidents:
            files = [key(v, nm) for v, nm in zip(r["files"], names.take(r["files"]))]
            rec = dict(r, files=files)
            if r["id"] not in tick_inc:
                tick_inc[r["id"]] = rec
                tick_nodes[r["id"]] = set(r["files"])
            else:
                t = tick_inc[r["id"]]
                extra = sorted(set(r["files"]) - tick_nodes[r["id"]])
                tick_nodes[r["id"]].update(extra)
                _fold_span(t, rec)
                t["files"] = t["files"] + [key(v, nm) for v, nm in zip(extra, names.take(extra))]
                t["n_files"] = len(t["files"])
                t["size_mb"] = float(t["size_mb"]) + sum(float(size[v]) for v in extra)
                t["later_other_events"] = int(t["later_other_events"]) + sum(int(res.file_recovery[v][2]) for v in extra)
                ms = [float(score[v]) for v in extra if not np.isnan(score[v])] + ([] if t["max_score"] is None else [t["max_score"]])
                t["max_score"] = max(ms) if ms else None
            run = self.incidents.get(r["id"])
            if run is None:
                run = self.incidents[r["id"]] = {k: rec[k] for k in self._RUNNING_FIELDS}
                run["files"] = []
            _fold_span(run, rec)
            run["files"] = sorted(set(run["files"]) | set(files), key=str)
            run["n_files"] = len(run["files"])
        for n, nm in zip(res.plan_nodes, plan_names):
            k = key(n, nm)
            if k in fresh and k not in step_inc:
                step_inc[k] = res.step_incident.get(int(n))


def _fold_span(into: dict, rec: dict):
    """an incident record's onset / end widened by another record of the same incident (earliest onset, latest end)"""
    if rec["onset"] is not None and (into["onset"] is None or rec["onset"] < into["onset"]):
        into["onset"], into["onset_event"] = rec["onset"], rec["onset_event"]
    if rec["end"] is not None and (into["end"] is None or rec["end"] > into["end"]):
        into["end"], into["end_event"] = rec["end"], rec["end_event"]
