"""Contamination on the GPU (nerrf_b200.taint; DESIGN.md 1.5) against the per-row numpy statement (oracle/taint_ref.py):
T as float64 bits, levels, preds, labels, the tainted list, rounds and levels, on the m1 trace, fleet windows with
bystanders, colliding hosts, a hub row of more than 2^16 edges, int64 rowptr, empty and full seed sets and
H in {0, 1, 2, -1}; ground truth on a constructed trace; per-host identity; agreement across graph builders; and the
stream and CLI end to end."""
import json
import math
import os
import time

import numpy as np
import pytest
import torch

from nerrf_b200 import graph as G, incident as I, ingest, pipeline, stream, taint
from nerrf_b200.ai.planner import emit
from oracle import taint_ref as R
from taint_trace import A, APP, B, NIGHTLY, NOTE, OLD, constructed_trace

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M1 = os.path.join(ROOT, "tests", "golden", "m1_trace.jsonl")
INF = math.inf


def host(a):
    if callable(a):
        a = a()
    return a.cpu().numpy() if torch.is_tensor(a) else np.asarray(a)


def dev_graph(g, rp64=False):
    t = lambda a: (a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))).cuda()
    rp = t(g.rowptr)
    rp = rp.to(torch.int64) if rp64 else rp.to(torch.int32)
    return G.TemporalGraph(rp, t(g.col).to(torch.int32), t(g.ew), t(g.x), g.meta)


def bits(a):
    return np.asarray(a, np.float64).view(np.int64)


def seed_sets(g, rng):
    n = g.num_nodes
    et = host(g.meta["edge_time"])
    times = et[~np.isnan(et)] if et.size else np.zeros(1)
    some = rng.permutation(n)[:max(1, n // 20)]
    st = rng.choice(times, some.size) - rng.integers(0, 2, some.size) * 0.5
    st[: min(2, some.size)] = [-INF, INF][: min(2, some.size)]
    full = np.arange(n)
    return [([], [], []), (some, st, rng.integers(0, 4, some.size)),
            (full, rng.choice(times, n), rng.integers(0, 3, n))]


def check(g, seeds, st, sl, hops=(0, 1, 2, -1), rp64=False):
    """kernel == statement bit for bit, two runs give the same bits"""
    gd = dev_graph(g, rp64)
    rowptr, col, kind = host(g.rowptr), host(g.col), np.asarray(g.meta["node_kind"])
    fl, et = host(g.meta["edge_flow"]), host(g.meta["edge_time"])
    for h in hops:
        o = R.closure(rowptr, col, kind, fl, et, seeds, st, sl, h)
        runs = []
        for _ in range(2):
            r = taint.closure(gd, seeds, st, sl, h)
            runs.append({k: (host(v) if torch.is_tensor(v) else v) for k, v in r.items()})
        d = runs[0]
        nodes = o["nodes"]
        assert np.array_equal(d["nodes"], nodes), h
        assert np.array_equal(bits(d["time"]), bits(o["T"][nodes])), h
        assert np.array_equal(d["level"], o["level"][nodes]) and np.array_equal(d["pred"], o["pred"][nodes]), h
        assert np.array_equal(d["label"], o["label"][nodes]), h
        assert (d["rounds"], d["levels"]) == (o["rounds"], o["levels"]), h
        assert all(np.asarray(runs[0][k]).tobytes() == np.asarray(runs[1][k]).tobytes() for k in d)
        if h == -1:
            ea = R.earliest_arrival(rowptr, col, kind, fl, et, seeds, st)
            assert np.array_equal(bits(ea), bits(o["T"]))
    return d


def test_m1_trace_seed_sets_and_hops():
    g = G.graph_from_jsonl(M1, observable=True)
    rng = np.random.default_rng(0)
    for s, st, sl in seed_sets(g, rng):
        check(g, s, st, sl)


@pytest.mark.parametrize("bystanders", [0, 2])
def test_fleet_windows(bystanders):
    cols, _ = stream.fleet_columns(12, 3, seed=3, n_files=12, benign_files=8, bystanders=bystanders)
    ts = cols.timestamp
    w = stream.window(cols, float(ts.min()) + 5.0, float(ts.min()) + 65.0)
    g = ingest.graph_from_columns(w, device="cuda", observable=True)
    rng = np.random.default_rng(bystanders)
    for s, st, sl in seed_sets(g, rng)[1:]:
        check(g, s, st, sl, hops=(2, -1))


@pytest.mark.parametrize("k", [2, 3])
def test_colliding_hosts(k):
    cols = stream.concat_columns([c for c, _, _ in stream.host_streams(k, 6, 2, seed=4, bystanders=1)])
    g = ingest.graph_from_columns(cols, device="cuda", observable=True)
    s, st, sl = seed_sets(g, np.random.default_rng(k))[1]
    check(g, s, st, sl, hops=(1, -1))


def hub_graph(n_hub_edges=(1 << 16) + 3001, n_procs=40, seed=5):
    """process 0's row holds > 2^16 edges from files; file rows hold edges from processes; times unsorted in rows"""
    rng = np.random.default_rng(seed)
    n_files = 60
    N = n_procs + n_files
    kind = np.zeros(N, np.int64); kind[:n_procs] = 1
    rows = [rng.integers(n_procs, N, n_hub_edges)] + [rng.integers(0, N, rng.integers(0, 30)) for _ in range(N - 1)]
    rowptr = np.zeros(N + 1, np.int64); rowptr[1:] = np.cumsum([r.size for r in rows])
    col = np.concatenate(rows).astype(np.int32)
    E = col.size
    et = np.round(rng.random(E) * 200.0, 1) + 1.7e9
    et[rng.random(E) < 0.01] = np.nan
    meta = {"node_kind": kind, "edge_time": et, "edge_flow": rng.integers(0, 4, E).astype(np.uint8),
            "edge_event": rng.permutation(E).astype(np.int64), "node_source": np.zeros(N, np.int64)}
    return G.TemporalGraph(rowptr.astype(np.int32), col, np.ones(E, np.float32), np.zeros((N, 32), np.float32), meta)


@pytest.mark.parametrize("rp64", [False, True])
def test_hub_row_over_2_16_edges_and_int64_rowptr(rp64):
    g = hub_graph()
    n = g.num_nodes
    seeds = np.array([45, 50, 7])
    d = check(g, seeds, np.array([1.7e9 + 10.0, 1.7e9 + 100.0, 1.7e9 + 150.0]), np.array([0, 1, 2]), hops=(1, -1), rp64=rp64)
    assert 0 in d["nodes"].tolist()                                   # the hub row is reached
    gd = dev_graph(g, rp64)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(5):
        taint.closure(gd, seeds, [1.7e9 + 10.0, 1.7e9 + 100.0, 1.7e9 + 150.0], [0, 1, 2])
    print("hub graph (%d nodes, %d edges, hub row %d): closure %.3f ms per call"
          % (n, g.num_edges, int(g.rowptr[1]), (time.perf_counter() - t0) / 5 * 1e3))


def test_invalid_input_is_refused():
    g = hub_graph(n_hub_edges=5000)
    col = np.array(g.col)
    pos = int(g.rowptr[1]) + 3                                        # an edge of a small row nobody reaches
    col[pos] = g.num_nodes
    with pytest.raises(ValueError, match="col holds node ids"):
        taint.closure(dev_graph(G.TemporalGraph(g.rowptr, col, g.ew, g.x, g.meta)), [1], [0.0], [0])
    gd = dev_graph(g)
    with pytest.raises(ValueError, match="distinct"):
        taint.closure(gd, [1, 1], [0.0, 1.0], [0, 0])
    with pytest.raises(ValueError, match="NaN"):
        taint.closure(gd, [1], [math.nan], [0])
    with pytest.raises(ValueError, match="labels"):
        taint.closure(gd, [1], [0.0], [-1])
    with pytest.raises(ValueError, match="seed node ids"):
        taint.closure(gd, [g.num_nodes], [0.0], [0])
    with pytest.raises(ValueError, match="max_hops"):
        taint.closure(gd, [1], [0.0], [0], max_hops=-2)
    bad = dict(g.meta, edge_flow=np.where(np.arange(g.num_edges) == pos, 4, g.meta["edge_flow"]).astype(np.uint8))
    with pytest.raises(ValueError, match="edge_flow"):
        taint.closure(dev_graph(G.TemporalGraph(g.rowptr, g.col, g.ew, g.x, bad)), [1], [0.0], [0])
    assert taint.closure(gd, [1], [0.0], [0])["nodes"].numel() >= 1  # the same call on valid input


# ---- ground truth on the constructed trace
def _incidents(g, names):
    enc = [v for v, nm in enumerate(names) if nm.endswith(".lockbit3")]
    ea = torch.as_tensor(host(g.meta["edge_label"])).float().cuda()
    return I.incidents(g, torch.zeros(g.num_nodes, device="cuda"), tau=INF, seeds=enc, edge_attack=ea, return_files=True)


def _contamination(g, only=None):
    names = g.meta["names"]
    names = names.take(list(range(g.num_nodes))) if hasattr(names, "take") else list(names)
    recs, per_file = _incidents(g, names)
    return taint.contamination(g, recs, per_file, only=only), recs


def test_constructed_trace_ground_truth():
    ev, a_open, a_write = constructed_trace()
    g = dev_graph(G.graph_from_events(ev, observable=True))
    cont, recs = _contamination(g)
    assert [r["id"] for r in recs] == ["pid:454"]
    got = {c["name"]: c for c in cont["pid:454"]}
    assert set(got) == {"pid:%d" % A, NIGHTLY, NOTE}
    first = G.event_record(a_open[0])
    assert got["pid:%d" % A]["hops"] == 1 and got["pid:%d" % A]["since_event"] == first
    assert got[NIGHTLY]["hops"] == 2 and got[NIGHTLY]["via"] == [first, G.event_record(a_write)]
    assert got[NIGHTLY]["since"] == G._parse_ts(a_write["timestamp"]) and got[NIGHTLY]["kind"] == "file"
    assert got[NOTE]["hops"] == 1 and got[NOTE]["via"][0]["syscall"] == "ransom_note_created"
    assert not ({"pid:%d" % APP, "pid:%d" % B, OLD} & set(got))
    assert cont == taint.contamination(g, recs, _incidents(g, g.meta["names"])[1], only="pid:454")


def test_constructed_trace_with_bystanders():
    ev, _, _ = constructed_trace(bystanders=2)
    g = dev_graph(G.graph_from_events(ev, observable=True))
    cont, recs = _contamination(g)
    got = {c["name"]: c for c in cont["pid:454"]}
    assert set(got) == {"pid:%d" % A, NIGHTLY, NOTE, "pid:455", "pid:456"}
    t = lambda e: G._parse_ts(e["timestamp"])
    start = {}
    for e in ev:
        if e["event"] == "file_encrypt_start":
            start.setdefault(G._stem(e["path"]), t(e))
    for pid in (455, 456):                   # since its first open of an encrypted file after that file's encrypt_start
        first = min(t(e) for e in ev if e["pid"] == pid and e["event"] == "openat" and G._stem(e["path"]) in start
                    and t(e) >= start[G._stem(e["path"])])
        assert got["pid:%d" % pid]["since"] == first and got["pid:%d" % pid]["hops"] == 1


def _whole_stream(cols):
    ds = stream.DeviceStream(cols, "cuda", observable=True)
    t0, t1 = ds.span()
    return ds, ds.window_graph(t0 - 1.0, t1, t1 - t0 + 1.0, edge_labels=True)


def test_per_host_identity():
    ev, _, _ = constructed_trace()
    benign = [e for e in ev if e["pid"] != 454]                    # host b: the same paths and processes, no attacker
    cols = stream.concat_columns([stream.with_source(ingest.decode_event_batch(ingest.encode_event_batch(x)), s)
                                  for s, x in enumerate((ev, benign))])
    _, g = _whole_stream(cols)
    src = np.asarray(g.meta["node_source"])
    names = g.meta["names"].take(list(range(g.num_nodes)))
    enc = [v for v, nm in enumerate(names) if nm.endswith(".lockbit3") and src[v] == 0]
    recs, per_file = I.incidents(g, torch.zeros(g.num_nodes, device="cuda"), tau=INF, seeds=enc,
                                 edge_attack=g.meta["edge_label"].float(), host_names=["a", "b"], return_files=True)
    cont = taint.contamination(g, recs, per_file)
    nodes = [c["node"] for cs in cont.values() for c in cs]
    assert nodes and all(src[v] == 0 for v in nodes)
    assert {names[v] for v in nodes} == {"pid:%d" % A, NIGHTLY, NOTE}


def _records(g, ea):
    names = g.meta["names"]
    names = names.take(list(range(g.num_nodes))) if hasattr(names, "take") else list(names)
    enc = [v for v, nm in enumerate(names) if nm.endswith(".lockbit3")]
    recs, per_file = I.incidents(g, torch.zeros(g.num_nodes, device="cuda"), tau=INF, seeds=enc, edge_attack=ea,
                                 return_files=True)
    cont = taint.contamination(g, recs, per_file)
    strip = lambda e: None if e is None else (e["time"], e["pid"], e["path"])
    return {i: sorted((c["name"], c["since"], c["hops"], tuple(strip(e) for e in c["via"])) for c in cs) for i, cs in cont.items()}


def test_every_builder_gives_the_same_records():
    ev, _, _ = constructed_trace(bystanders=1)
    cols = ingest.decode_event_batch(ingest.encode_event_batch(ev))
    ds, gw = _whole_stream(cols)
    ea = gw.meta["edge_label"].float()
    want = _records(gw, ea)
    assert want["pid:454"]
    g_ev = G.graph_from_events(ev, observable=True)
    assert _records(dev_graph(g_ev), torch.as_tensor(g_ev.meta["edge_label"]).float().cuda()) == want
    for dev in (None, "cuda"):
        gc = ingest.graph_from_columns(cols, device=dev, observable=True)
        assert np.array_equal(host(gc.col), host(gw.col))               # the same CSR: the window's labels apply
        assert _records(dev_graph(gc), ea) == want
    live = stream.DeviceStream.live("cuda", observable=True)
    order = np.argsort(cols.timestamp, kind="stable")
    live.append(b"".join(ingest.encode_columns(cols)[i] for i in order.tolist()))
    t0, t1 = live.span()
    gl = live.window_graph(t0 - 1.0, t1, t1 - t0 + 1.0, edge_labels=True)
    assert np.array_equal(host(gl.meta["edge_flow"]), host(gw.meta["edge_flow"]))
    assert _records(gl, gl.meta["edge_label"].float()) == want


def _planner(**kw):
    from nerrf_b200.ai.models import GraphSAGE_T
    from nerrf_b200.ai.models.lstm import LSTMScorer
    model = GraphSAGE_T(G.F_IN, 128, 2, seed=1).cuda()
    return stream.StreamingPlanner(model, LSTMScorer().cuda(), window_s=60.0, tick_s=30.0, top_a=64, n_rollouts=256, depth=16,
                                   iterations=4, kill_candidates=True, **kw)


def test_stream_run_and_feed_agree_and_plans_unchanged():
    ev, _, _ = constructed_trace(bystanders=2, n_files=20)
    cols = ingest.decode_event_batch(ingest.encode_event_batch(ev))
    plain = _planner(incidents=True).run(cols)
    sp = _planner(incidents=True, contamination=True, incident_tau=float("-inf"))
    ticks = sp.run(cols)
    assert [t.planned for t in plain] == [t.planned for t in _planner(incidents=True, contamination=True).run(cols)]
    assert any(t.contamination for t in ticks)
    for i, run in sp.contamination.items():                          # running: the earliest since per node key
        for k, r in run.items():
            assert r["since"] == min(x["since"] for t in ticks for x in t.contamination.get(i, []) if x["key"] == k)
    live = _planner(incidents=True, contamination=True, incident_tau=float("-inf"))
    order = np.argsort(cols.timestamp, kind="stable")
    wire = b"".join(ingest.encode_columns(cols)[i] for i in order.tolist())
    out = []
    for k in range(0, len(wire), len(wire) // 8 + 1):
        out += live.feed(wire[k:k + len(wire) // 8 + 1])
    out += live.flush()
    strip = lambda t: {i: [(r["key"], r["since"], r["hops"]) for r in rs] for i, rs in t.contamination.items()}
    assert [strip(t) for t in out] == [strip(t) for t in ticks]


def test_undo_cli_lists_the_archive_under_one_incident(tmp_path):
    from nerrf_b200 import undo
    ev, _, _ = constructed_trace(n_files=20)
    path = tmp_path / "trace.jsonl"
    path.write_text("".join(json.dumps(e) + "\n" for e in ev))
    # a flagged file is a seed of the closure, not contaminated: flag the plan's file steps only (tau = inf), and offer
    # the planner the 20 most anomalous files
    base = ["--trace", str(path), "--train-epochs", "25", "--rollouts", "256", "--top-a", "20", "--incident-threshold=inf"]
    plain = undo.main(base + ["--incidents", "--out", str(tmp_path / "plain.json")])
    full = undo.main(base + ["--incidents", "--contamination", "--out", str(tmp_path / "full.json")])
    owners = [i["id"] for i in full["incidents"] if any(c["name"] == NIGHTLY for c in i["contaminated"])]
    seen = "plan steps %s; incidents %s" % ([s.get("path", s.get("node")) for s in full["steps"]],
                                            {i["id"]: [c["name"] for c in i["contaminated"]] for i in full["incidents"]})
    assert len(owners) == 1, seen
    print("nightly.tar is contaminated under incident %s" % owners[0])
    entry = next(c for i in full["incidents"] for c in i["contaminated"] if c["name"] == NIGHTLY)
    assert entry["recovery_point"]["before"] == entry["since"] and entry["recovery_point"]["event"]["path"] == NIGHTLY
    strip = lambda p: {k: v for k, v in p.items() if k != "stats"}
    assert strip(dict(full, incidents=[{k: v for k, v in i.items() if k != "contaminated"} for i in full["incidents"]])) == strip(plain)
    one = undo.main(base + ["--incident", owners[0], "--contamination", "--out", str(tmp_path / "one.json")])
    assert any(c["name"] == NIGHTLY for i in one["incidents"] if i["id"] == owners[0] for c in i["contaminated"])
    # a plan made without the option: the same bytes as the incidents-only code path of the parent
    again = undo.main(base + ["--incidents", "--out", str(tmp_path / "again.json")])
    assert emit.to_json(strip(again)) == emit.to_json(strip(plain))
    assert '"contaminated"' not in (tmp_path / "plain.json").read_text()
