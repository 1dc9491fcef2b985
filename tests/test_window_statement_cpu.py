"""The exact statement of the window-graph model inputs (oracle/window_ref.py) against the event-by-event spec
(graph.graph_from_events, pipeline.file_sequences) on the reference's m0 / m1 traces and on random rename-heavy traces
with byte counts from the whole uint64 range.  The GPU kernels are checked against this statement in
test_gpu_window_kernels.py, so here it earns that role without a GPU.  The host twins (ingest.graph_from_columns,
ingest.sequences_from_columns) are held to it as well."""
import json
import os

import numpy as np
import pytest

from nerrf_b200 import graph as G, ingest, pipeline
from nerrf_b200.ai.models import lstm
from oracle import window_ref as W

GOLD = os.path.join(os.path.dirname(__file__), "golden")
BYTE_EDGES = (0, 1, 0x7ffff000, 0x7ffff001, 2 ** 63 - 1, 2 ** 63, 2 ** 64 - 1)


def plain_columns(cols, merge=True, observable=False):
    """events -> the statement's plain columns, in time order: node ids from the host interning (nerrf_trace_intern)"""
    cols = ingest.resolve_columns(cols)
    ts = cols.timestamp
    order = np.argsort(ts, kind="stable")
    node_p, node_f, node_g, kind, _, _ = ingest.intern_nodes(cols, order, merge)
    raw = cols.event_slot[order].astype(np.int64)
    pf = cols.path_flags[order]
    if merge:                                                 # a rename's .lockbit target is the same node
        pf = pf | (ingest.path_flags_of(*cols.strings["new_path"])[order] & np.uint8(1))
    return dict(P=node_p[order], F=node_f[order], G=node_g[order] if not merge else None, kind=kind,
                t_abs=ts[order], t=ts[order] - ts[order[0]], raw=raw,
                slot=np.asarray(G.OBSERVABLE_SLOT, np.int64)[raw] if observable else raw,
                bytes=cols.bytes[order], pf=pf, pf_raw=cols.path_flags[order])


def rename_heavy_events(n, seed, files=120, huge_bytes=True):
    """random openat / write / rename / encrypt / note events over a small set of stems, many renames (chains, targets
    that already exist, .lockbit3 twins), equal timestamps, gaps above 10 s, byte counts from the whole uint64 range"""
    rng = np.random.default_rng(seed)
    kinds = ["openat", "write", "rename", "file_encrypt_start", "file_encrypt_complete", "ransom_note_created", "unlink"]
    ev, sec = [], 1_700_000_000
    for i in range(n):
        sec += int(rng.choice([0, 0, 1, 3, 11]))
        k = kinds[int(rng.integers(len(kinds)))]
        stem = "/srv/%s/f%d" % (["tmp", "data", "README"][int(rng.integers(3))], rng.integers(files))
        path = stem + [".dat", ".lockbit3", "", ".a.b"][int(rng.integers(4))]
        if rng.random() < 0.05:
            path = "/tmp/x%d" % rng.integers(10)
        b = int(rng.choice(BYTE_EDGES)) if huge_bytes and rng.random() < 0.3 else int(rng.integers(0, 1 << 20))
        e = {"ts": (sec, int(rng.integers(0, 4)) * 250_000_000), "pid": int(rng.integers(1, 9)), "syscall": k, "path": path,
             "bytes": b}
        if k == "rename":
            e["new_path"] = "/srv/data/f%d%s" % (rng.integers(files), [".lockbit3", ".dat", ""][int(rng.integers(3))])
        ev.append(e)
    return ev


def _traces():
    out = []
    for m in ("m0", "m1"):
        out.append((m, [json.loads(l) for l in open(os.path.join(GOLD, f"{m}_trace.jsonl"))]))
    out.append(("random", rename_heavy_events(4000, 1)))
    return out


def _cols(events):
    return ingest.decode_event_batch(ingest.encode_event_batch(events))


def _ulp1(a, b):
    return np.all(np.abs(a.astype(np.float64) - b) <= np.spacing(np.abs(b)).astype(np.float64))


@pytest.mark.parametrize("trace", ["m0", "m1", "random"])
@pytest.mark.parametrize("merge", [True, False])
@pytest.mark.parametrize("observable", [False, True])
def test_node_features_and_edge_labels_equal_the_event_by_event_spec(trace, merge, observable):
    ev = dict(_traces())[trace]
    cols = _cols(ev)
    c = plain_columns(cols, merge, observable)
    want = G.graph_from_events(ingest.events_from_columns(cols), merge_renames=merge, window=60.0, observable=observable)
    x, label, size_mb, acc = W.node_features(c["P"], c["F"], c["G"], c["t"], c["slot"], c["bytes"], c["pf"], c["kind"], 60.0)
    assert x.shape == want.x.shape and np.array_equal(c["kind"], want.meta["node_kind"])
    assert np.all(np.isfinite(x)) and np.all(np.isfinite(size_mb))
    # log1p columns: the two float64 log1p implementations may differ in the last bit of the double
    assert _ulp1(x, want.x)
    exact = [0, 1, 2, 14, 15, 16, 17, 18, 19] + list(range(20, 32))
    assert np.array_equal(x[:, exact], want.x[:, exact])
    assert np.array_equal(size_mb.view(np.uint32), want.meta["size_mb"].view(np.uint32))
    if not observable:                                        # the spec's labels come from the annotations
        assert np.array_equal(label, want.meta["label"])
    assert np.array_equal(acc["deg"], np.diff(want.rowptr))   # in-degree == out-degree == the CSR row length
    lab = W.edge_labels(c["P"], c["F"], c["raw"], W.csr_rows(want.rowptr), want.col)
    assert np.array_equal(lab, want.meta["edge_label"])
    # the host twin is held to the same statement
    host = ingest.graph_from_columns(cols, merge_renames=merge, window=60.0, observable=observable)
    assert _ulp1(host.x, x) and np.array_equal(host.x[:, exact], x[:, exact])
    assert np.array_equal(host.meta["size_mb"].view(np.uint32), size_mb.view(np.uint32))


@pytest.mark.parametrize("trace", ["m0", "m1", "random"])
@pytest.mark.parametrize("t_max", [1, 3, lstm.T_MAX])
def test_file_sequences_equal_the_event_by_event_spec(trace, t_max):
    ev = dict(_traces())[trace]
    cols = _cols(ev)
    c = plain_columns(cols, True, True)
    g = G.graph_from_events(ingest.events_from_columns(cols), observable=True)
    seq_w, len_w, nodes = pipeline.file_sequences(ingest.events_from_columns(cols), g, t_max=t_max, observable=True)
    span = max(c["t_abs"][-1] - c["t_abs"][0], 1e-6)
    seq, ln = W.file_sequences(nodes, c["F"], c["t_abs"], c["slot"], c["bytes"], c["pf_raw"], c["t_abs"][0], span, t_max)
    assert np.array_equal(ln, len_w)
    assert np.all(np.isfinite(seq))
    assert _ulp1(seq, seq_w)
    assert np.array_equal(np.delete(seq, 8, axis=2), np.delete(seq_w, 8, axis=2))
    seq_h, len_h, nodes_h = ingest.sequences_from_columns(cols, t_max=t_max, observable=True)
    assert np.array_equal(nodes_h, nodes) and np.array_equal(len_h, ln) and _ulp1(seq_h, seq)


def test_byte_counts_are_clamped_and_summed_exactly():
    # one file, writes of every edge value: the sum is over the clamped values, exactly, and nothing is non-finite
    ev = [{"ts": (100 + i, 0), "pid": 7, "syscall": "write", "path": "/d/a.dat", "bytes": b} for i, b in enumerate(BYTE_EDGES)]
    ev.append({"ts": (200, 0), "pid": 7, "syscall": "write", "path": "/d/a.dat", "bytes": 100})
    cols = _cols(ev)
    assert int(cols.bytes[-2]) == 2 ** 64 - 1                 # the wire value itself is kept
    c = plain_columns(cols)
    x, _, size_mb, acc = W.node_features(c["P"], c["F"], None, c["t"], c["slot"], c["bytes"], c["pf"], c["kind"], 60.0)
    want_sum = sum(min(b, G.MAX_RW_COUNT) for b in BYTE_EDGES) + 100
    f = int(c["F"][0])
    assert acc["bytes"][f] == want_sum and acc["bytes"][int(c["P"][0])] == want_sum
    assert x[f, 13] == np.float32(np.log1p(float(want_sum)) / 20.0)
    assert size_mb[f] == np.float32(float(want_sum) / 1.0 / 1e6)   # writes are slot 5: k = max(c0 + c1 + c2, 1) = 1
    g = G.graph_from_events(ingest.events_from_columns(cols), window=60.0)
    assert g.x[f, 13] == x[f, 13] and g.meta["size_mb"][f] == size_mb[f]
    seq, ln = W.file_sequences([f], c["F"], c["t_abs"], c["slot"], c["bytes"], c["pf_raw"], c["t_abs"][0], 100.0, 16)
    assert ln[0] == 8 and np.all(np.isfinite(seq))
    assert np.array_equal(seq[0, :8, 8], (np.log1p(np.minimum(np.asarray(BYTE_EDGES + (100,), np.float64), G.MAX_RW_COUNT))
                                          / 20.0).astype(np.float32))
    assert G.clamp_bytes(2 ** 64 - 1) == G.MAX_RW_COUNT == W.MAX_RW_COUNT
