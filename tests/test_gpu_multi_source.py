"""Several sources (one tracker per node) on the device (needs an H100).  The oracle is the relabelling that defines a
source: a K-source stream must give, node for node, the graph of the same stream relabelled as ONE source (every
(source, pid) a pid of its own, every non-empty path prefixed per source) through the single-source path.  Also: the
_ex entry points with no source column are today's entry points bit for bit, colliding hosts stay apart, the live
planner ticks on the low watermark of its sources, and the widened (source, pid) regroup sort at its tile boundaries."""
import ctypes as C

import numpy as np
import pytest
import torch

from nerrf_b200 import _lib, ingest, stream
from test_gpu_live_stream import _records_in_batches, _same_graph
from test_gpu_stream_kernels import BASE, SORT_CHUNK, _order_ref, _path_off, _same_order, _times
from test_ingest import _tracker_style_events

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("lib_built")]

SCALARS = ("ts_sec", "ts_nanos", "pid", "tid", "flags", "ret_val", "bytes", "event_slot", "path_flags")


# ------------------------------------------------------------------------------------------------------------ helpers
def _tracker(k):
    """k hosts running the same tracker-style trace (same pids and paths, path-less writes), clocks 1 ms apart"""
    parts = []
    for h in range(k):
        c = stream.with_source(ingest.decode_event_batch(ingest.encode_event_batch(_tracker_style_events())), h)
        c.ts_nanos = (c.ts_nanos.astype(np.int64) + 1_000_000 * h).astype(np.int32)
        parts.append(c)
    return stream.concat_columns(parts)


def _fleet(k):
    return stream.concat_columns([c for c, _, _ in stream.host_streams(k, 12, 2, seed=5, bystanders=1)])


def _partition(h):
    """canonical labels of the partition a hash array induces (labels in order of first occurrence)"""
    _, first, inv = np.unique(np.asarray(h), return_index=True, return_inverse=True)
    return np.argsort(np.argsort(first))[inv.reshape(-1)]


def _same_as_relabelled(g, w, cols, edge_labels=False):
    """g: graph of the multi-source stream `cols`; w: the same window of relabel_single_source(cols)"""
    if w is None:
        assert g is None
        return
    assert g.num_nodes == w.num_nodes and g.meta["events"] == w.meta["events"]
    assert torch.equal(g.rowptr, w.rowptr) and torch.equal(g.col, w.col)
    assert torch.equal(g.ew.view(torch.int32), w.ew.view(torch.int32)) and torch.equal(g.x.view(torch.int32), w.x.view(torch.int32))
    for k in ("label", "node_kind"):
        assert np.array_equal(g.meta[k], w.meta[k]), k
    assert np.array_equal(g.meta["size_mb"].view(np.uint32), w.meta["size_mb"].view(np.uint32))
    assert (g.meta["t0"], g.meta["span"]) == (w.meta["t0"], w.meta["span"])
    if edge_labels:
        assert torch.equal(g.meta["edge_label"], w.meta["edge_label"])
    src = g.meta["node_source"]
    keys = np.unique(ingest.process_keys(cols))
    every = np.arange(g.num_nodes)
    if cols.source is None:                                          # one source 0: relabelling is the identity
        assert g.meta["names"].take(every) == w.meta["names"].take(every) and not src.any()
        every = every[:0]
    for v, a, b in zip(every.tolist(), g.meta["names"].take(every), w.meta["names"].take(every)):
        if a.startswith("pid:"):                                     # the relabelled pid is the rank of (source, pid)
            assert int(keys[int(b[4:])]) == (int(src[v]) << 32) | int(a[4:]), (v, a, b)
        else:
            assert b == "@%d/%s" % (src[v], a), (v, a, b)
    assert np.array_equal(_partition(g.meta["name_hash"].cpu().numpy()), _partition(w.meta["name_hash"].cpu().numpy()))
    assert np.array_equal(_partition(g.meta["dir_hash"]().cpu().numpy()), _partition(w.meta["dir_hash"]().cpu().numpy()))


def _windows(ds):
    t0, t1 = ds.span()
    return [(t0 - 1, t0 + 30), (t0 + 10, t0 + 70), (t0 + 40, t1), (t1 + 5, t1 + 9), (t0 - 1, t1)]


def _per_source_pieces(cols, mode, rng):
    """[(source, bytes)] interleaved across sources in time: 1-s batches, single records, or random byte chunks"""
    out = []
    for s in np.unique(cols.source).tolist():
        sel = np.nonzero(cols.source == s)[0]
        part = ingest.EventColumns(n=sel.size, source=cols.source[sel],
                                   strings={k: ingest._gather_strings(*cols.strings[k], sel) for k in ingest.STRING_COLUMNS},
                                   **{k: getattr(cols, k)[sel] for k in SCALARS})
        batches = _records_in_batches(part, width=1.0)
        t = np.sort(part.timestamp)
        bounds = np.cumsum([0] + [len(b) for b in batches])
        if mode == "batches":
            out += [(t[bounds[i]], s, b"".join(b)) for i, b in enumerate(batches)]
        elif mode == "records":
            recs = [r for b in batches for r in b]
            out += [(t[i], s, r) for i, r in enumerate(recs)]
        else:
            buf = b"".join(b"".join(b) for b in batches)
            cuts = np.unique(np.r_[0, rng.integers(1, len(buf), max(len(buf) // 200, 1)), len(buf)])
            out += [(t[min(int(c0) * part.n // len(buf), part.n - 1)], s, buf[c0:c1]) for c0, c1 in zip(cuts[:-1], cuts[1:])]
    out.sort(key=lambda x: x[0])
    return [(s, b) for _, s, b in out]


def _feed_live(ds, pieces):
    carry = {}
    for s, b in pieces:
        data = carry.get(s, b"") + b
        carry[s] = data[ds.append(data, partial=True, source=s):]
    assert not any(carry.values())


# ------------------------------------------------------------------------------------------------ relabel equivalence
@pytest.mark.parametrize("k", [1, 2, 3, 8])
@pytest.mark.parametrize("trace", ["fleet", "tracker"])
def test_whole_trace_equals_the_relabelled_stream(k, trace):
    cols = _fleet(k) if trace == "fleet" else _tracker(k)
    rel = stream.relabel_single_source(cols)
    for merge, observable in [(True, True), (False, False), (True, False), (False, True)]:
        ds = stream.DeviceStream(cols, "cuda", observable=observable, merge_renames=merge)
        ref = stream.DeviceStream(rel, "cuda", observable=observable, merge_renames=merge)
        for lo, hi in _windows(ref):
            _same_as_relabelled(ds.window_graph(lo, hi, 60.0, edge_labels=True), ref.window_graph(lo, hi, 60.0, edge_labels=True),
                                cols, edge_labels=True)


@pytest.mark.parametrize("mode", ["batches", "records", "chunks"])
@pytest.mark.parametrize("k", [1, 2, 3, 8])
def test_live_stream_equals_the_relabelled_stream(k, mode):
    cols = _fleet(k) if mode != "records" else _tracker(k)
    pieces = _per_source_pieces(cols, mode, np.random.default_rng(k))
    for merge, observable in [(True, True), (False, False)]:
        ds = stream.DeviceStream.live("cuda", observable=observable, merge_renames=merge)
        _feed_live(ds, pieces)
        arrived = ds._dc.host(ds.n)                                  # stored (arrival) order: ties in time keep it
        assert ds.resident_events == cols.n and (np.sort(ingest.process_keys(arrived)) == np.sort(ingest.process_keys(cols))).all()
        ref = stream.DeviceStream(stream.relabel_single_source(arrived), "cuda", observable=observable, merge_renames=merge)
        assert ds.span() == ref.span()
        assert ds._key_bits == (48 if k > 1 else 32)
        t0, t1 = ref.span()
        mid = t0 + 0.5 * (t1 - t0)                                  # a window cutting the encryption phase in half
        for lo, hi in _windows(ref) + [(t0 - 1, mid)]:
            _same_as_relabelled(ds.window_graph(lo, hi, 60.0, edge_labels=True), ref.window_graph(lo, hi, 60.0, edge_labels=True),
                                arrived, edge_labels=True)


def test_single_source_five_is_todays_graph_with_other_hashes():
    cols = _tracker(1)
    base = ingest.EventColumns(**{**cols.__dict__, "source": None})
    five = stream.with_source(base, 5)
    for merge in (True, False):
        a = stream.DeviceStream(base, "cuda", observable=True, merge_renames=merge)
        b = stream.DeviceStream(five, "cuda", observable=True, merge_renames=merge)
        live = stream.DeviceStream.live("cuda", observable=True, merge_renames=merge)
        live.append(b"".join(ingest.encode_columns(base)), source=5)
        for lo, hi in _windows(a):
            ga, gb, gl = a.window_graph(lo, hi, 60.0), b.window_graph(lo, hi, 60.0), live.window_graph(lo, hi, 60.0)
            if ga is None:
                assert gb is None and gl is None
                continue
            for g in (gb, gl):
                g.meta["name_hash"], nh = ga.meta["name_hash"], g.meta["name_hash"]
                _same_graph(g, ga)
                g.meta["name_hash"] = nh
                assert not torch.equal(nh, ga.meta["name_hash"])
                assert (g.meta["node_source"] == 5).all()
                assert np.array_equal(_partition(nh.cpu().numpy()), _partition(ga.meta["name_hash"].cpu().numpy()))
            names = ga.meta["names"].take(np.arange(ga.num_nodes))
            assert ga.meta["name_hash"].cpu().tolist() == [stream.name_hash(nm) for nm in names]
            assert gb.meta["name_hash"].cpu().tolist() == [stream.name_hash(nm, 5) for nm in names]
            assert gb.meta["dir_hash"]().cpu().tolist() == [stream.dir_hash(nm, 5) for nm in names]


# ---------------------------------------------------------------------------------------------------------- collisions
def test_same_lockbit_trace_on_two_hosts_gives_two_disjoint_equal_copies():
    from nerrf_b200.ai.models import GraphSAGE_T
    one, _ = stream.fleet_columns(6, 2, seed=2, bystanders=1)
    two = stream.concat_columns([stream.with_source(one, 0), stream.with_source(one, 1)])
    g1 = stream.DeviceStream(one, "cuda", observable=True).window_graph(-np.inf, np.inf, 60.0)
    g2 = stream.DeviceStream(two, "cuda", observable=True).window_graph(-np.inf, np.inf, 60.0)
    assert g2.num_nodes == 2 * g1.num_nodes and g2.num_edges == 2 * g1.num_edges
    src = g2.meta["node_source"]
    names2 = g2.meta["names"].take(np.arange(g2.num_nodes))
    names1 = g1.meta["names"].take(np.arange(g1.num_nodes))
    at = {(int(s), nm): v for v, (s, nm) in enumerate(zip(src, names2))}
    assert len(at) == g2.num_nodes
    copies = [np.asarray([at[(h, nm)] for nm in names1]) for h in (0, 1)]
    rp, col = g2.rowptr.cpu().numpy(), g2.col.cpu().numpy()
    for h, c in enumerate(copies):                                   # every edge of a copy stays inside it
        for v in c[:200].tolist():
            assert (src[col[rp[v]:rp[v + 1]]] == h).all()
    torch.manual_seed(0)
    model = GraphSAGE_T(32, 128, 2).cuda()
    s2 = model(g2.x, g2.rowptr, g2.col, g2.ew)[1]
    a, b = s2[torch.from_numpy(copies[0]).cuda()], s2[torch.from_numpy(copies[1]).cuda()]
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def _cols(events, s):
    return stream.with_source(ingest.decode_event_batch(ingest.encode_event_batch(events)), s)


def test_pathless_write_and_rename_stay_on_their_host():
    a = _cols([{"timestamp": 10.0, "event": "openat", "path": "/app/uploads/a.dat", "pid": 7},
               {"timestamp": 11.0, "event": "rename", "path": "/app/uploads/a.dat", "new_path": "/app/uploads/b.lockbit3", "pid": 7}], 0)
    b = _cols([{"timestamp": 12.0, "event": "write", "path": "", "pid": 7, "size": 5},
               {"timestamp": 13.0, "event": "openat", "path": "/app/uploads/b.txt", "pid": 8}], 1)
    cols = stream.concat_columns([a, b])
    for live in (False, True):
        if live:
            ds = stream.DeviceStream.live("cuda", observable=True)
            ds.append(b"".join(ingest.encode_columns(a)), source=0); ds.append(b"".join(ingest.encode_columns(b)), source=1)
        else:
            ds = stream.DeviceStream(cols, "cuda", observable=True)
        g = ds.window_graph(0.0, 100.0, 60.0)
        assert g.meta["events"] == 3                                  # B's write is dropped, not given A's file
        names = g.meta["names"].take(np.arange(g.num_nodes))
        files = sorted((int(s), nm) for s, nm, k in zip(g.meta["node_source"], names, g.meta["node_kind"]) if k == 0)
        assert files == [(0, "/app/uploads/b.lockbit3"), (1, "/app/uploads/b.txt")]   # no alias across hosts


def test_two_hosts_uploads_get_separate_restores():
    from nerrf_b200 import pipeline
    one, _ = stream.fleet_columns(6, 2, seed=2)
    two = stream.concat_columns([stream.with_source(one, 0), stream.with_source(one, 1)])
    g = stream.DeviceStream(two, "cuda", observable=True).window_graph(-np.inf, np.inf, 60.0)
    files = np.nonzero(g.meta["node_kind"] == 0)[0]
    dh = pipeline.node_dir_hashes(g, files).cpu().numpy()
    src = g.meta["node_source"][files]
    for d in np.unique(dh).tolist():                                 # a directory group never spans two hosts
        assert np.unique(src[dh == d]).size == 1


def test_host_built_graph_restores_stay_on_one_host(models):
    """graph_from_columns (the CLI's and the multi-GPU path's graph) over two hosts running the same 1000-file attack:
    the planner's directory groups are qualified by the host, so no restore covers files of both"""
    from nerrf_b200 import pipeline, trace_sim
    from nerrf_b200.ai.planner import emit
    model, scorer = models
    one = ingest.decode_event_batch(ingest.encode_event_batch(trace_sim.lockbit_trace(n_files=1000, benign_files=10, seed=5)))
    cols = stream.concat_columns([stream.with_source(one, 0), stream.with_source(one, 1)])
    g = ingest.graph_from_columns(cols, device="cuda", observable=True)
    seq, lengths, nodes = ingest.sequences_from_columns(cols, observable=True)
    res = pipeline.run(g, seq, lengths, nodes, model, scorer, top_a=2048, n_rollouts=1024, depth=40, iterations=8,
                       commit_per_search=64, kill_candidates=True, restore_candidates=True)
    assert res.restores                                              # each host's encrypted files fill its own /app/uploads
    src = g.meta["node_source"]
    for r in res.restores:
        assert r["dir"] == "/app/uploads" and np.unique(src[np.asarray(r["covers"])]).size == 1
    plan = emit.from_pipeline(g, res, host_names=["nodeA", "nodeB"])
    dirs = [s_ for s_ in plan["steps"] if s_["op"] == "restore_snapshot_dir"]
    assert dirs and all(s_["host"] in ("nodeA", "nodeB") for s_ in dirs)


# --------------------------------------------------------------------------- _ex with no source = today, bit for bit
def _up(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a).view(dt) if np.asarray(a).dtype.itemsize == np.dtype(dt).itemsize
                            else np.ascontiguousarray(a, dt)).cuda()


def _order_ex(sec, nanos, pid, off, horizon, source, key_bits, old=False):
    n = int(sec.shape[0])
    d_sec, d_nan, d_off = _up(sec, np.int64), _up(nanos, np.int32), _up(off, np.int64)
    d_pid = _up(np.asarray(pid, np.uint32), np.int32)
    d_src = None if source is None else _up(np.asarray(source, np.uint16), np.int16)
    h = _lib.lib()
    need = C.c_int64()
    _lib.check(h.nerrf_trace_stream_order_workspace_bytes(n, C.byref(need)), "ws")
    ws = torch.empty(need.value + 256, dtype=torch.uint8, device="cuda")
    e = lambda dt: torch.empty(max(n, 1), dtype=dt, device="cuda")
    ts, order, ts_sorted, src, retain = e(torch.float64), e(torch.int64), e(torch.float64), e(torch.int64), e(torch.int64)
    res_off = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    counts = (C.c_int64 * 3)()
    tail = (_lib.ptr(ts), _lib.ptr(order), _lib.ptr(ts_sorted), _lib.ptr(src), _lib.ptr(res_off), _lib.ptr(retain), counts,
            C.c_void_p((ws.data_ptr() + 255) & ~255), need.value, _lib.current_stream_ptr())
    if old:
        _lib.check(h.nerrf_trace_stream_order(n, _lib.ptr(d_sec), _lib.ptr(d_nan), _lib.ptr(d_pid), _lib.ptr(d_off), float(horizon), *tail), "order")
    else:
        _lib.check(h.nerrf_trace_stream_order_ex(n, _lib.ptr(d_sec), _lib.ptr(d_nan), _lib.ptr(d_pid), _lib.ptr(d_src), key_bits,
                                                 _lib.ptr(d_off), float(horizon), *tail), "order_ex")
    nk, nr = int(counts[0]), int(counts[1])
    host = lambda t, k: t[:k].cpu().numpy()
    return {"counts": tuple(int(c) for c in counts), "ts": host(ts, n), "src": host(src, n), "order": host(order, nk),
            "ts_sorted": host(ts_sorted, nk), "res_path_off": host(res_off, n + 1), "retain": host(retain, nr)}


def _rank_pids(pid, source):
    """(source, pid) -> a uint32 pid in the same order: the single-source reference of the 48-bit regroup"""
    key = (np.asarray(source, np.uint64) << np.uint64(32)) | np.asarray(pid, np.uint32).astype(np.uint64)
    return np.unique(key, return_inverse=True)[1].reshape(-1).astype(np.uint32)


def test_stream_order_ex_without_sources_is_todays():
    rng = np.random.default_rng(0)
    n = 3 * 4096 + 17
    sec, nanos = _times("random", n, rng)
    pid = rng.integers(0, 50, n).astype(np.uint32)
    off = _path_off("random", n, rng, sec, nanos, pid)
    h = float(np.median(sec.astype(np.float64)))
    want = _order_ex(sec, nanos, pid, off, h, None, 32, old=True)
    zeros, fives = np.zeros(n, np.uint16), np.full(n, 5, np.uint16)
    for source, bits in [(None, 32), (zeros, 32), (zeros, 48), (fives, 32), (fives, 48)]:
        _same_order(_order_ex(sec, nanos, pid, off, h, source, bits), want, f"bits={bits}")
    with pytest.raises(_lib.NerrfError, match="key_bits"):
        _order_ex(sec, nanos, pid, off, h, None, 48)


def _intern_ex(cols, fn, source, merge):
    n = cols.n
    order = np.argsort(cols.timestamp, kind="stable")
    cap = 3 * n
    (poff, pdata), (goff, gdata) = cols.strings["path"], cols.strings["new_path"]
    d = [_up(order, np.int64), _up(cols.pid, np.int32), _up(poff, np.int64), _up(pdata, np.uint8), _up(goff, np.int64),
         _up(gdata if gdata.size else np.zeros(1, np.uint8), np.uint8)]
    d_src = None if source is None else _up(np.asarray(source, np.uint16), np.int16)
    out = [torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(3)]
    kind, ne, nw = (torch.zeros(cap, dtype=dt, device="cuda") for dt in (torch.int8, torch.int64, torch.int8))
    need = C.c_int64()
    _lib.check(_lib.lib().nerrf_trace_intern_device_workspace_bytes(n, cap, C.byref(need)), "ws")
    ws = torch.empty(need.value + 256, dtype=torch.uint8, device="cuda")
    nn = C.c_int64()
    head = (n, n, _lib.ptr(d[0]), _lib.ptr(d[1]))
    rest = (_lib.ptr(d[2]), _lib.ptr(d[3]), _lib.ptr(d[4]), _lib.ptr(d[5]), int(merge), *(_lib.ptr(t) for t in out), C.byref(nn),
            _lib.ptr(kind), _lib.ptr(ne), _lib.ptr(nw), cap, C.c_void_p((ws.data_ptr() + 255) & ~255), need.value,
            _lib.current_stream_ptr())
    h = _lib.lib()
    if fn == "old":
        _lib.check(h.nerrf_trace_intern_device(*head, *rest), "intern")
    else:
        _lib.check(h.nerrf_trace_intern_device_ex(*head, _lib.ptr(d_src), *rest), "intern_ex")
    N = nn.value
    hashes = []
    for name in ("name", "dir"):
        hh = torch.empty(N, dtype=torch.int64, device="cuda")
        args = (N, _lib.ptr(ne), _lib.ptr(nw), _lib.ptr(d[1]))
        tail = (_lib.ptr(d[2]), _lib.ptr(d[3]), _lib.ptr(d[4]), _lib.ptr(d[5]), _lib.ptr(hh), _lib.current_stream_ptr())
        if fn == "old":
            _lib.check(getattr(h, "nerrf_trace_%s_hash" % name)(*args, *tail), name)
        else:
            _lib.check(getattr(h, "nerrf_trace_%s_hash_ex" % name)(*args, _lib.ptr(d_src), *tail), name)
        hashes.append(hh.cpu().numpy())
    nodes = [t.cpu().numpy() for t in out] + [kind[:N].cpu().numpy(), ne[:N].cpu().numpy(), nw[:N].cpu().numpy()]
    return nodes, hashes


@pytest.mark.parametrize("merge", [True, False])
def test_intern_and_hashes_ex_without_sources_are_todays(merge):
    cols = ingest.resolve_columns(ingest.EventColumns(**{**_fleet(1).__dict__, "source": None}))
    want_nodes, want_hash = _intern_ex(cols, "old", None, merge)
    for source in (None, np.zeros(cols.n, np.uint16)):
        nodes, hashes = _intern_ex(cols, "ex", source, merge)
        assert all(np.array_equal(a, b) for a, b in zip(nodes, want_nodes))
        assert all(np.array_equal(a, b) for a, b in zip(hashes, want_hash))
    nodes, hashes = _intern_ex(cols, "ex", np.full(cols.n, 5, np.uint16), merge)
    assert all(np.array_equal(a, b) for a, b in zip(nodes, want_nodes))
    assert not any(np.array_equal(a, b) for a, b in zip(hashes, want_hash))


def _decode(wire, ex, source=0, col=True):
    raw = np.frombuffer(wire, np.uint8)
    dc = stream._DeviceColumns(torch.device("cuda"), 1, [1, 1, 1, 1])
    bad, rec_at, body_off, body_len, _ = ingest._frame(raw, False)
    m = int(rec_at.shape[0])
    dc.reserve(0, [0] * 4, m, [int(body_len.sum())] * 4)
    dc.source.fill_(7)
    wire_d, rec_d = torch.from_numpy(raw.copy()).cuda(), torch.from_numpy(np.stack([rec_at, body_off, body_len])).cuda()
    need = C.c_int64()
    _lib.check(_lib.lib().nerrf_trace_decode_device_workspace_bytes(m, C.byref(need)), "ws")
    ws = torch.empty(need.value + 256, dtype=torch.uint8, device="cuda")
    status = torch.empty(1, dtype=torch.int64, device="cuda")
    a = (_lib.ptr(wire_d), _lib.ptr(rec_d[0]), _lib.ptr(rec_d[1]), _lib.ptr(rec_d[2]), m, 0, dc.ptrs())
    b = (_lib.ptr(status), C.c_void_p((ws.data_ptr() + 255) & ~255), need.value, _lib.current_stream_ptr())
    if ex:
        _lib.check(_lib.lib().nerrf_trace_decode_device_ex(*a, _lib.ptr(dc.source) if col else None, source, *b), "decode_ex")
    else:
        _lib.check(_lib.lib().nerrf_trace_decode_device(*a, *b), "decode")
    assert int(status.item()) == -1
    return dc, dc.host(m)


def _src(c):
    return np.zeros(c.n, np.uint16) if c.source is None else c.source


def test_decoder_and_gather_ex_without_sources_are_todays():
    from test_gpu_live_stream import _same_columns
    wire = b"".join(ingest.encode_columns(_tracker(1)))
    _, want = _decode(wire, False)
    assert (_src(want) == 7).all()                                   # the entry point without a column leaves it alone
    _, got = _decode(wire, True, 0, col=False)
    _same_columns(got, want)
    assert (_src(got) == 7).all()
    for s in (0, 1, 65535):
        dc, got = _decode(wire, True, s)
        _same_columns(got, want)
        assert (_src(got) == s).all() and (got.source is None) == (s == 0)
    with pytest.raises(_lib.NerrfError, match="out of range"):
        _decode(wire, True, 65536)
    rows = torch.tensor([0, 3, 4, 9], dtype=torch.int64, device="cuda")
    outs = []
    for ex in (False, True):
        out = stream._DeviceColumns(dc.dev, dc.rows, [d.numel() for d in dc.data])
        need = C.c_int64()
        _lib.check(_lib.lib().nerrf_trace_gather_rows_workspace_bytes(4, C.byref(need)), "ws")
        ws_t = torch.empty(need.value + 256, dtype=torch.uint8, device="cuda")
        ws = C.c_void_p((ws_t.data_ptr() + 255) & ~255)
        if ex:
            _lib.check(_lib.lib().nerrf_trace_gather_rows_ex(dc.ptrs(), _lib.ptr(dc.source), _lib.ptr(rows), 4, out.ptrs(),
                                                             _lib.ptr(out.source), ws, need.value, _lib.current_stream_ptr()), "g")
        else:
            _lib.check(_lib.lib().nerrf_trace_gather_rows(dc.ptrs(), _lib.ptr(rows), 4, out.ptrs(), ws, need.value,
                                                          _lib.current_stream_ptr()), "g")
        torch.cuda.synchronize()
        outs.append(out.host(4))
    _same_columns(outs[1], outs[0])
    assert (_src(outs[1]) == 65535).all() and outs[0].source is None


# ---------------------------------------------------------------------------------- widened regroup: kernel boundaries
def _check_ex(sec, nanos, pid, source, off, horizon, tag):
    want = _order_ref(sec, nanos, _rank_pids(pid, source), off, horizon)
    _same_order(_order_ex(sec, nanos, pid, off, horizon, source, 48), want, tag)


@pytest.mark.parametrize("n", [4095, 4096, 4097, 2 * 4096 + 1, 3 * 4096 + 5])
def test_48_bit_keys_across_the_sort_tile(n):
    rng = np.random.default_rng(n)
    sec, nanos = _times("random", n, rng)
    pid = rng.choice(np.asarray([1, 7, 0xFFFFFFFF, 0x80000000], np.uint32), n)
    source = rng.choice(np.asarray([0, 1, 255, 256, 65535], np.uint16), n)
    off = _path_off("random", n, rng, sec, nanos, _rank_pids(pid, source))
    for h in (-np.inf, float(np.median(sec.astype(np.float64)))):
        _check_ex(sec, nanos, pid, source, off, h, f"n={n}")


def test_48_bit_keys_where_the_histogram_enters_its_second_chunk():
    """2^24 + 8193 pairs: the regroup's 6 passes each scan a histogram past its first chunk; 64 (source, pid) keys that
    share their pids across sources, so equal keys run across many sort tiles"""
    n = SORT_CHUNK + 8193
    rng = np.random.default_rng(48)
    sec = BASE + rng.integers(0, 60, n); nanos = (rng.integers(0, 1000, n) * 1_000_000).astype(np.int32)
    pid = rng.integers(0, 8, n).astype(np.uint32) * np.uint32(0x20000001)
    source = (rng.integers(0, 8, n) * 9000).astype(np.uint16)
    off = np.zeros(n + 1, np.int64)
    np.cumsum(np.where(rng.random(n) < 0.3, rng.integers(1, 40, n), 0), out=off[1:])
    _check_ex(sec, nanos, pid, source, off, float(BASE + 30), "17M")


def test_source_pid_segments_starting_on_scan_tile_boundaries():
    """(source, pid) segments that begin at 1024 k - 1, 1024 k and 1024 k + 1 of the regroup; neighbouring segments share
    the pid and differ only in the source, so only the upper 16 key bits cut them"""
    starts = sorted({0} | {1024 * k + d for k in (1, 2, 3, 17, 1023, 1024) for d in (-1, 0, 1)})
    n = starts[-1] + 1500
    rng = np.random.default_rng(3)
    seg = np.searchsorted(np.asarray(starts), np.arange(n), "right") - 1
    source = seg.astype(np.uint16)
    pid = np.full(n, 4242, np.uint32)
    sec, nanos = _times("random", n, rng)
    p = rng.permutation(n)
    source, pid = source[p], pid[p]
    off = _path_off("random", n, rng, sec, nanos, _rank_pids(pid, source))
    for h in (-np.inf, float(np.median(sec.astype(np.float64)))):
        _check_ex(sec, nanos, pid, source, off, h, f"h={h}")


# ---------------------------------------------------------------------------------------------------------- live ticks
@pytest.fixture(scope="module")
def models():
    from nerrf_b200.ai import train as T
    from nerrf_b200.ai.models import GraphSAGE_T
    from nerrf_b200.ai.models.lstm import LSTMScorer
    torch.manual_seed(0)
    model, scorer = GraphSAGE_T(32, 128, 2), LSTMScorer()
    T.train(model, scorer, T.toy_set(range(100, 104)), epochs=25, lr=3e-3)
    return model.cuda(), scorer.cuda()


def _planner(models, **kw):
    model, scorer = models
    return stream.StreamingPlanner(model, scorer, top_a=1024, n_rollouts=512, depth=24, iterations=8, commit_per_search=32,
                                   kill_candidates=True, **kw)


def _host_wires(k, n_procs=40, n_att=3):
    hs = stream.host_streams(k, n_procs, n_att, seed=7, bystanders=1)
    return hs, [(c, _records_in_batches(c, 1.0)) for c, _, _ in hs]


def test_no_tick_while_a_source_lags_and_close_source_releases_it(models):
    _, wires = _host_wires(2)                                        # host 0 attacked (~100 s of trace), host 1 benign (shorter)
    sp = _planner(models)
    sp.add_source("a"); sp.add_source("b")
    fired = []
    for b in wires[1][1]:
        fired += sp.feed(b"".join(b), source="b")
    assert fired == [] and sp.ticks == []                            # a has delivered nothing
    for b in wires[0][1]:
        fired += sp.feed(b"".join(b), source="a")
    t_b = float(wires[1][0].timestamp.max())
    assert fired and all(sp._t0 + t.t_hi < t_b for t in fired)      # up to b's watermark, no further
    n = len(sp.ticks)
    more = sp.close_source("b")                                      # b is done: a alone holds the watermark
    assert more and len(sp.ticks) == n + len(more) and all(sp._t0 + t.t_hi > t_b - sp.tick_s for t in more)
    with pytest.raises(ValueError, match="closed"):
        sp.feed(b"".join(wires[1][1][0]), source="b")


def _apart(cols, h):
    """host h's clock h microseconds later: no two hosts share a timestamp, so stored order never breaks a tie between
    hosts and the arrival order of interleaved chunks cannot change the time order"""
    nanos = cols.ts_nanos.astype(np.int64) + 1000 * h
    return ingest.EventColumns(**{**cols.__dict__, "ts_sec": cols.ts_sec + nanos // 1_000_000_000,
                                  "ts_nanos": (nanos % 1_000_000_000).astype(np.int32)})


def test_feed_of_interleaved_sources_plans_like_run_over_the_merged_columns(models):
    """4 hosts (0 and 2 attacked; 1 and 3 benign, reusing the attackers' pids), each host's bytes cut at random offsets
    (records split across calls) and interleaved with the other hosts' chunks; one malformed chunk of host 1 is refused
    and rolled back alone.  Ticks, plans, kills and reversions equal run() over the merged columns."""
    hs = stream.host_streams(4, 40, 3, seed=7, bystanders=1)
    cols = [_apart(c, h) for h, (c, _, _) in enumerate(hs)]
    names = ["n%d" % h for h in range(4)]
    want = _planner(models)
    for name in names:
        want.add_source(name)
    want.run(stream.concat_columns(cols))
    rng = np.random.default_rng(11)
    chunks = []
    for h, c in enumerate(cols):
        recs = ingest.encode_columns(c)
        order = np.argsort(c.timestamp, kind="stable")
        wire = b"".join(recs[i] for i in order.tolist())
        starts = np.cumsum([0] + [len(recs[i]) for i in order.tolist()])
        ts = c.timestamp[order]
        cuts = np.unique(np.r_[0, rng.integers(1, len(wire), len(wire) // 3000), starts[len(starts) // 2], len(wire)])
        for a, b in zip(cuts[:-1].tolist(), cuts[1:].tolist()):
            chunks.append((float(ts[min(np.searchsorted(starts, a, "right") - 1, len(ts) - 1)]), h, wire[a:b],
                           h == 1 and b == int(starts[len(starts) // 2])))
    chunks.sort(key=lambda x: (x[0], x[1]))
    last = {h: j for j, (_, h, _, _) in enumerate(chunks)}
    got = _planner(models)
    for name in names:
        got.add_source(name)
    peak, refused = 0, 0
    for j, (_, h, b, at_record_end) in enumerate(chunks):
        got.feed(b, source=names[h])
        if at_record_end:                                            # host 1's carry is empty here: a malformed record
            before = (got.live.resident_events, got.live.n_keep, dict(got._carry), len(got.ticks))
            with pytest.raises(_lib.NerrfError, match="malformed"):
                got.feed(b"\x0a\x02\x0b\x00", source="n1")
            assert (got.live.resident_events, got.live.n_keep, dict(got._carry), len(got.ticks)) == before
            refused += 1
        if last[h] == j:                                             # a host that has sent everything stops holding the watermark
            got.close_source(names[h])
        peak = max(peak, got.live.resident_events)
    got.flush()
    assert refused == 1
    assert len(got.ticks) == len(want.ticks) >= 3
    for a, b in zip(got.ticks, want.ticks):
        assert (a.t_hi, a.events, a.nodes, a.edges, a.planned) == (b.t_hi, b.events, b.nodes, b.edges, b.planned)
    assert got.killed == want.killed and got.reverted == want.reverted
    assert peak < sum(c.n for c in cols)
    # kills name (host, pid): attackers are killed on their own hosts, never the benign hosts' processes that share their pids
    attackers = {(names[h], p) for h, (_, _, pids) in enumerate(hs) for p in pids}
    assert got.killed & attackers
    assert not any(h in ("n1", "n3") for h, _ in got.killed)
    enc = {(names[h], p) for h, (_, e, _) in enumerate(hs) for p in e}
    assert {h for h, _ in enc} == {"n0", "n2"}
    assert len(got.reverted & enc) >= 0.95 * len(enc)
    assert not any(h in ("n1", "n3") and p.endswith(".lockbit3") for h, p in got.reverted)
    assert all(isinstance(k, tuple) for k in got.reverted | got.killed)


def test_a_second_source_cannot_join_after_one_source_ticks(models):
    _, wires = _host_wires(2)
    sp = _planner(models)
    for b in wires[0][1]:
        sp.feed(b"".join(b), source="a")
    assert sp.ticks and all(isinstance(k, str) for k in sp.reverted | sp.killed)
    with pytest.raises(ValueError, match="register every source"):
        sp.feed(b"".join(wires[1][1][0]), source="b")


def test_retention_keeps_the_latest_named_event_per_host_and_pid():
    a = _cols([{"timestamp": 10.0, "event": "openat", "path": "/d/a.dat", "pid": 7}], 0)
    b = _cols([{"timestamp": 11.0, "event": "openat", "path": "/d/b.dat", "pid": 7}], 1)
    wa = _cols([{"timestamp": 200.0, "event": "write", "path": "", "pid": 7, "size": 1}], 0)
    wb = _cols([{"timestamp": 201.0, "event": "write", "path": "", "pid": 7, "size": 1}], 1)
    ds = stream.DeviceStream.live("cuda", observable=True)
    for c, s in ((a, 0), (b, 1)):
        ds.append(b"".join(ingest.encode_columns(c)), source=s)
    ds.compact(100.0)
    assert ds.resident_events == 2                                   # one named event per (source, pid), both kept
    for c, s in ((wa, 0), (wb, 1)):
        ds.append(b"".join(ingest.encode_columns(c)), source=s)
    g = ds.window_graph(150.0, 300.0, 60.0)
    names = g.meta["names"].take(np.arange(g.num_nodes))
    files = sorted((int(s), nm) for s, nm, k in zip(g.meta["node_source"], names, g.meta["node_kind"]) if k == 0)
    assert files == [(0, "/d/a.dat"), (1, "/d/b.dat")]


# ---------------------------------------------------------------------------------------------------------- end to end
def test_cli_with_two_traces_plans_like_the_library_over_the_merged_columns(models, tmp_path):
    from nerrf_b200 import pipeline, undo
    from nerrf_b200.ai.planner import emit
    model, scorer = models
    ck = {"sage": model.state_dict(), "lstm": scorer.state_dict(), "layers": 2,
          "edge_head_trained": bool(getattr(model, "edge_head_trained", False))}
    torch.save(ck, tmp_path / "w.pt")
    hs = stream.host_streams(2, 8, 2, seed=3)
    args, parts = [], []
    for h, (c, _, _) in enumerate(hs):
        p = tmp_path / ("h%d.pb" % h)
        p.write_bytes(b"".join(ingest.encode_columns(ingest.EventColumns(**{**c.__dict__, "source": None}))))
        args += ["--trace", "node%d=%s" % (h, p)]
        parts.append(stream.with_source(ingest.decode_event_batch(p.read_bytes()), h))
    opts = ["--rollouts", "256", "--iterations", "4"]
    plan = undo.main(args + ["--weights", str(tmp_path / "w.pt"), "--out", str(tmp_path / "plan.json"),
                             "--shell-dir", str(tmp_path / "sh")] + opts)
    cols = stream.concat_columns(parts)
    g = ingest.graph_from_columns(cols, device="cuda", observable=True)
    seq, lengths, nodes = ingest.sequences_from_columns(cols, observable=True)
    res = pipeline.run(g, seq, lengths, nodes, model, scorer, top_a=1024, n_rollouts=256, depth=50, iterations=4, device="cuda")
    want = emit.from_pipeline(g, res, host_names=["node0", "node1"])
    assert plan["steps"] == want["steps"] and plan["steps"]
    assert {s_["host"] for s_ in plan["steps"] if s_["op"] == "rename"} == {"node0"}            # only host 0 was attacked
    for h in ("node0", "node1"):
        assert (tmp_path / "sh" / (h + ".sh")).read_text() == emit.to_shell(want, host=h)
    assert "lockbit3" not in (tmp_path / "sh" / "node1.sh").read_text()
    one = undo.main(["--trace", args[1], "--weights", str(tmp_path / "w.pt"), "--shell-dir", str(tmp_path / "one")] + opts)
    assert all("host" not in s_ for s_ in one["steps"])                                    # one source: no host fields
    assert (tmp_path / "one" / "node0.sh").read_text() == emit.to_shell(one)
