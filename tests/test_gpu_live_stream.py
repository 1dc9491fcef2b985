"""The live stream (needs an H100): EventBatch bytes decoded on the device, appended to the resident stream as they
arrive, resolved / ordered / trimmed there, and planned tick by tick -- pinned bit for bit against the whole-trace path
(ingest.decode_event_batch -> DeviceStream(cols) -> StreamingPlanner.run)."""
import re

import numpy as np
import pytest
import torch
from hypothesis import given, settings, strategies as st

from nerrf_b200 import ingest, stream
from nerrf_b200._lib import NerrfError
from test_ingest import _random_batch, _tracker_style_events

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("lib_built")]

SCALARS = ("ts_sec", "ts_nanos", "pid", "tid", "flags", "ret_val", "bytes", "event_slot", "path_flags")


def _same_columns(a, b):
    assert a.n == b.n
    for k in SCALARS:
        x, y = getattr(a, k), getattr(b, k)
        assert x.dtype == y.dtype and np.array_equal(x, y), k
    for k in ingest.STRING_COLUMNS:
        assert np.array_equal(a.strings[k][0], b.strings[k][0]) and np.array_equal(a.strings[k][1], b.strings[k][1]), k


def _offset(e):
    return int(re.search(r"byte offset (\d+)", str(e)).group(1))


# ------------------------------------------------------------------------------------------------------ 1 decoder parity
@pytest.mark.parametrize("n,rich,seed", [(0, False, 0), (1, False, 1), (200, False, 2), (300, True, 3)])
def test_device_decoder_equals_host_decoder(n, rich, seed):
    wire = _random_batch(np.random.default_rng(seed), n, rich).SerializeToString()
    _same_columns(stream.decode_event_batch_device(wire), ingest.decode_event_batch(wire))


def test_device_decoder_on_concatenated_batches():
    rng = np.random.default_rng(4)
    wire = b"".join(_random_batch(rng, k, rich=k % 2 == 1).SerializeToString() for k in (3, 0, 5, 1, 40))
    _same_columns(stream.decode_event_batch_device(wire), ingest.decode_event_batch(wire))


@settings(max_examples=150, deadline=None)
@given(st.binary(max_size=200))
def test_fuzz_device_decoder_same_verdict_and_offset(data):
    try:
        want = ingest.decode_event_batch(data)
    except NerrfError as e:
        with pytest.raises(NerrfError) as got:
            stream.decode_event_batch_device(data)
        assert _offset(got.value) == _offset(e)
        return
    _same_columns(stream.decode_event_batch_device(data), want)


# ------------------------------------------------------------------------------------------------------- 2 graph parity
def _records_in_batches(cols, width=1.0):
    """the rows of `cols` as wire records, grouped into batches of `width` seconds of trace time (time order)"""
    recs = ingest.encode_columns(cols)
    ts = cols.timestamp
    order = np.argsort(ts, kind="stable")
    key = np.floor((ts[order] - ts.min()) / width).astype(np.int64)
    cuts = np.nonzero(np.diff(key))[0] + 1
    return [[recs[i] for i in part] for part in np.split(order, cuts)]


def _same_graph(g, w):
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
    assert torch.equal(g.meta["name_hash"], w.meta["name_hash"])
    every = np.arange(g.num_nodes)
    assert g.meta["names"].take(every) == w.meta["names"].take(every)


def _windows(ref):
    t0, t1 = ref.span()
    return [(t0 - 1, t0 + 30), (t0 + 10, t0 + 70), (t0 + 40, t1), (t1 + 5, t1 + 9), (t0 - 1, t1)]


def _feed(ds, pieces, chunked=False, rng=None):
    if not chunked:
        for p in pieces:
            ds.append(p)
        return
    buf = b"".join(pieces)
    carry, pos = b"", 0
    while pos < len(buf):
        k = int(rng.integers(1, 400))
        data = carry + buf[pos:pos + k]
        pos += k
        carry = data[ds.append(data, partial=True):]
    assert carry == b""


def _fleet():
    cols, _ = stream.fleet_columns(60, 4, seed=3)
    return cols


def _tracker():
    return ingest.decode_event_batch(ingest.encode_event_batch(_tracker_style_events()))


@pytest.mark.parametrize("mode", ["batches", "records", "chunks"])
@pytest.mark.parametrize("trace", ["fleet", "tracker"])
def test_live_stream_windows_equal_the_whole_trace(trace, mode):
    cols = _fleet() if trace == "fleet" else _tracker()
    batches = _records_in_batches(cols)
    wire = b"".join(b"".join(b) for b in batches)
    for merge, observable in [(True, True), (False, False), (True, False)]:
        ref = stream.DeviceStream(ingest.decode_event_batch(wire), "cuda", observable=observable, merge_renames=merge)
        ds = stream.DeviceStream.live("cuda", observable=observable, merge_renames=merge)
        pieces = [b"".join(b) for b in batches] if mode == "batches" else [r for b in batches for r in b]
        _feed(ds, pieces, chunked=mode == "chunks", rng=np.random.default_rng(1))
        assert ds.resident_events == cols.n and ds.span() == ref.span()
        for lo, hi in _windows(ref):
            _same_graph(ds.window_graph(lo, hi, 60.0), ref.window_graph(lo, hi, 60.0))


def test_named_event_arriving_after_its_pathless_write():
    """a write's path comes from the pid's open, which reaches us one batch later (it is older): the write is dropped
    while unattributable, then resolved once the open is resident"""
    recs = ingest.encode_columns(_tracker())
    ev = _tracker_style_events()
    op = next(i for i, e in enumerate(ev) if e["event"] == "openat")
    wr = next(i for i, e in enumerate(ev) if i > op and e["event"] == "write" and e["pid"] == ev[op]["pid"])
    late = [recs[i] for i in range(len(recs)) if i != op]
    late.insert(wr, recs[op])                                    # the open arrives right after its write
    wire = b"".join(late)
    for merge in (True, False):
        ref = stream.DeviceStream(ingest.decode_event_batch(wire), "cuda", observable=True, merge_renames=merge)
        ds = stream.DeviceStream.live("cuda", observable=True, merge_renames=merge)
        ds.append(b"".join(late[:wr]))
        kept = ds.n_keep
        ds.append(late[wr])
        assert ds.n_keep == kept + 2                             # the open and, now attributable, its write
        ds.append(b"".join(late[wr + 1:]))
        for lo, hi in _windows(ref):
            _same_graph(ds.window_graph(lo, hi, 60.0), ref.window_graph(lo, hi, 60.0))


# ----------------------------------------------------------------------------------------------- 4 retention (+ parity)
@pytest.mark.parametrize("trace", ["fleet", "tracker"])
def test_retention_keeps_what_future_windows_need(trace):
    cols = _fleet() if trace == "fleet" else _tracker()
    batches = _records_in_batches(cols, width=1.0 if trace == "fleet" else 0.25)
    wire = b"".join(b"".join(b) for b in batches)
    window, tick = (60.0, 30.0) if trace == "fleet" else (1.0, 0.5)
    ref = stream.DeviceStream(ingest.decode_event_batch(wire), "cuda", observable=True)
    ts_all = ingest.decode_event_batch(wire).timestamp
    t0, t1 = ref.span()
    ds = stream.DeviceStream.live("cuda", observable=True)
    t_hi, seen, pids, fired = t0, 0, set(), 0
    for b in batches:
        ds.append(b"".join(b))
        seen += len(b)
        pids |= set(ingest.decode_event_batch(b"".join(b)).pid.tolist())
        while ds.span()[1] > t_hi + tick:
            t_hi += tick
            _same_graph(ds.window_graph(t_hi - window, t_hi, window), ref.window_graph(t_hi - window, t_hi, window))
            ds.compact(t_hi - window)
            fired += 1
            newer = int((ts_all[:seen] > t_hi - window).sum())
            assert ds.resident_events <= newer + len(pids)
    assert fired >= 2
    assert ds.resident_events < cols.n or trace == "tracker"
    for lo, hi in [(t_hi - window, t1), (t_hi - window / 2, t1)]:
        _same_graph(ds.window_graph(lo, hi, window), ref.window_graph(lo, hi, window))


# -------------------------------------------------------------------------------------------------------- 5 atomicity
def test_malformed_append_leaves_the_stream_unchanged():
    cols = _fleet()
    recs = ingest.encode_columns(cols)
    ds = stream.DeviceStream.live("cuda")
    ds.append(b"".join(recs[:500]))
    before = (ds.resident_events, ds.n_keep, ds.span())
    g0 = ds.window_graph(-np.inf, np.inf, 60.0)
    bad_body = b"\x0a\x02\x0b\x00"                               # an Event whose body holds a group
    for bad in (b"".join(recs[500:600]) + bad_body + recs[600], b"".join(recs[500:510]) + b"\x0b\x00", recs[500][:-2]):
        with pytest.raises(NerrfError, match="malformed EventBatch at byte offset") as e:
            ds.append(bad)
        with pytest.raises(NerrfError) as want:
            ingest.decode_event_batch(bad)
        assert _offset(e.value) == _offset(want.value)
        assert (ds.resident_events, ds.n_keep, ds.span()) == before
        _same_graph(ds.window_graph(-np.inf, np.inf, 60.0), g0)
    assert ds.append(b"") == 0 and (ds.resident_events, ds.n_keep, ds.span()) == before
    ds.append(b"".join(recs[500:]))
    ref = stream.DeviceStream(ingest.decode_event_batch(b"".join(recs)), "cuda")
    _same_graph(ds.window_graph(-np.inf, np.inf, 60.0), ref.window_graph(-np.inf, np.inf, 60.0))


# ------------------------------------------------------------------------------------------------------ 3 planner parity
@pytest.fixture(scope="module")
def models():
    from nerrf_b200.ai import train as T
    from nerrf_b200.ai.models import GraphSAGE_T
    from nerrf_b200.ai.models.lstm import LSTMScorer
    torch.manual_seed(0)
    model, scorer = GraphSAGE_T(32, 128, 2), LSTMScorer()
    T.train(model, scorer, T.toy_set(range(100, 104)), epochs=25, lr=3e-3)
    return model.cuda(), scorer.cuda()


def _planner(models, kills, lateness=0.0):
    model, scorer = models
    return stream.StreamingPlanner(model, scorer, top_a=1024, n_rollouts=512, depth=24, iterations=8, commit_per_search=32,
                                   kill_candidates=kills, lateness_s=lateness)


@pytest.mark.parametrize("kills,lateness", [(False, 0.0), (True, 0.0), (True, 2.0)])
def test_feed_and_flush_plan_like_run(models, kills, lateness):
    cols, enc = stream.fleet_columns(120, 5, seed=9)
    recs = ingest.encode_columns(cols)
    ts = cols.timestamp
    rng = np.random.default_rng(3)
    arrival = ts + (rng.random(cols.n) * lateness * 0.9 if lateness else 0.0)     # displaced by less than lateness_s
    order = np.argsort(arrival, kind="stable")
    wire = b"".join(recs[i] for i in order)
    want = _planner(models, kills)
    want.run(ingest.decode_event_batch(wire))
    got = _planner(models, kills, lateness)
    fired, peak, k = [], 0, 0
    while k < len(wire):
        step = int(rng.integers(1, 64 << 10))
        fired += got.feed(wire[k:k + step])
        k += step
        peak = max(peak, got.live.resident_events)
    fired += got.flush()
    assert len(fired) == len(got.ticks) == len(want.ticks) >= 3
    for a, b in zip(got.ticks, want.ticks):
        assert (a.t_hi, a.events, a.nodes, a.edges, a.planned) == (b.t_hi, b.events, b.nodes, b.edges, b.planned)
    assert got.killed == want.killed and got.reverted == want.reverted
    assert len(got.reverted & enc) >= 0.95 * len(enc)
    assert peak < cols.n                                          # retention kept the resident set below the whole trace


def test_live_feed_is_single_gpu(models):
    sp = _planner(models, False)
    sp.dist_ctx = type("Ctx", (), {"world": 2, "rank": 0})()
    with pytest.raises(NotImplementedError):
        sp.feed(b"")
