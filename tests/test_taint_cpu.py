"""Contamination on the CPU (DESIGN.md 1.5): the flow-class table (the oracle and the library's one definition), the two
restatements of the closure against each other on hand-built graphs, every invalid-input rule, the ground truth of the
constructed trace by the statement, the emitter fields and the CLI argument rules."""
import argparse
import math

import numpy as np
import pytest

from nerrf_b200 import graph as G, ingest, stream, undo
from nerrf_b200.ai.planner import emit
from oracle import incident_ref as IR
from oracle import taint_ref as R
from taint_trace import A, APP, B, NIGHTLY, NOTE, OLD, constructed_trace

INF = math.inf
SIM_KINDS = ("file_created", "file_encrypt_start", "file_encrypt_complete", "ransom_note_created", "write", "rename")


def test_flow_class_table():
    for k in SIM_KINDS:
        assert R.flow_class(k) == R.P2F, k
    assert R.flow_class("openat", 0) == R.F2P
    assert R.flow_class("openat", 1) == R.P2F
    for f in (2, 0o101, 0o1102, -1, 1 << 40):
        assert R.flow_class("openat", f) == R.P2F | R.F2P, f
    for k in ("process_enum", "unlink", "seed_start", "simulation_start", 7):
        assert R.flow_class(k) == 0 and R.flow_class(k, 0) == 0
    for k in SIM_KINDS + ("openat",):
        assert R.flow_class(k, 0, -1) == 0 and R.flow_class(k, 2, -13) == 0
    assert R.flow_class(4, 0) == R.F2P and R.flow_class(5) == R.P2F          # by raw slot


def test_library_flow_class_is_the_table():
    """the host columns' one definition (nerrf_trace_flow_class) gives the oracle's table on every case above"""
    cases = [(s, f, r) for s in range(8) for f in (0, 1, 2, 0o101, -1, 1 << 40) for r in (0, 5, -1, -(1 << 40))]
    slot, fl, rv = (np.asarray(c, np.int64) for c in zip(*cases))
    got = G.event_flow(slot.astype(np.uint8), fl, rv)
    assert got.tolist() == [R.flow_class(int(s), int(f), int(r)) for s, f, r in cases]


def test_builders_read_flags_and_ret_val_and_default_them_to_zero():
    ev = [{"timestamp": 1.0 + i, "pid": 7, "event": k, "path": "/d/f", **x} for i, (k, x) in enumerate(
        [("openat", {}), ("openat", {"flags": 1}), ("openat", {"flags": 2}), ("write", {"ret_val": -9}), ("unlink", {})])]
    g = G.graph_from_events(ev)
    flow = g.meta["edge_flow"]()
    by_event = dict(zip(g.meta["edge_event"].tolist(), flow.tolist()))
    assert [by_event[i] for i in range(5)] == [R.F2P, R.P2F, 3, 0, 0]
    h = ingest.graph_from_columns(ingest.decode_event_batch(ingest.encode_event_batch(ev)))
    assert np.array_equal(h.meta["edge_flow"](), flow) and np.array_equal(h.meta["edge_time"](), g.meta["edge_time"]())


# ---- hand-built graphs: CSR by destination; kind 0 file, 1 process
def csr(n, edges):
    """edges: (u, v, t, flow) in the order they appear in their rows"""
    rows = [[] for _ in range(n)]
    for u, v, t, f in edges:
        rows[v].append((u, t, f))
    rowptr = np.zeros(n + 1, np.int64)
    rowptr[1:] = np.cumsum([len(r) for r in rows])
    flat = [e for r in rows for e in r]
    col = np.asarray([e[0] for e in flat], np.int64)
    et = np.asarray([e[1] for e in flat], np.float64)
    fl = np.asarray([e[2] for e in flat], np.uint8)
    return rowptr, col, et, fl


def both(kind, edges, seeds, st, labels=None, hops=(0, 1, 2, -1)):
    rowptr, col, et, fl = csr(len(kind), edges)
    labels = list(range(len(seeds))) if labels is None else labels
    out = {h: R.closure(rowptr, col, kind, fl, et, seeds, st, labels, h) for h in hops}
    ea = R.earliest_arrival(rowptr, col, kind, fl, et, seeds, st)
    assert np.array_equal(out[-1]["T"].view(np.int64), ea.view(np.int64))
    for h, o in out.items():
        check_invariants(rowptr, col, kind, fl, et, seeds, st, labels, o)
    return out


def check_invariants(rowptr, col, kind, fl, et, seeds, st, labels, o):
    """every reached node is levelled; a pred chain reaches a root of the node's label in `level` steps, times
    non-decreasing along it"""
    T, lv, pr, lab = o["T"], o["level"], o["pred"], o["label"]
    assert set(np.nonzero(T < INF)[0]) <= set(o["nodes"].tolist())
    for v in o["nodes"].tolist():
        steps, u, t = 0, v, T[v]
        while lv[u] > 0:
            p = pr[u]
            assert rowptr[u] <= p < rowptr[u + 1] and et[p] == T[u] <= t
            t, u, steps = T[u], int(col[p]), steps + 1
        assert steps == lv[v] and lab[v] == lab[u] and u in list(seeds)


def test_chain_through_equal_time_events():
    # p0 -> f1 at 5, f1 -> p2 at 5 (read), p2 -> f3 at 5: one instant, three hops
    kind = [1, 0, 1, 0]
    out = both(kind, [(0, 1, 5.0, R.P2F), (1, 2, 5.0, R.F2P), (2, 3, 5.0, R.P2F)], [0], [1.0])
    o = out[-1]
    assert o["T"].tolist() == [1.0, 5.0, 5.0, 5.0] and o["level"].tolist() == [0, 1, 2, 3]
    assert o["rounds"] == 4 and o["levels"] == 4
    assert out[2]["T"].tolist() == [1.0, 5.0, 5.0, INF] and out[2]["rounds"] == 2
    assert out[0]["T"].tolist() == [1.0, INF, INF, INF] and out[0]["rounds"] == 0 and out[0]["levels"] == 1


def test_equal_time_two_cycle_does_not_loop():
    # an O_RDWR open: both directions at once between p1 and f2
    kind = [0, 1, 0]
    out = both(kind, [(0, 1, 3.0, R.F2P), (1, 2, 4.0, 3), (2, 1, 4.0, 3)], [0], [0.0])
    o = out[-1]
    assert o["T"].tolist() == [0.0, 3.0, 4.0] and o["level"].tolist() == [0, 1, 2]


def test_seed_reached_before_its_own_seed_time_is_not_a_root():
    kind = [1, 0, 1]
    out = both(kind, [(0, 1, 2.0, R.P2F), (1, 2, 3.0, R.F2P)], [0, 1], [1.0, 9.0], labels=[0, 1])
    o = out[-1]
    assert o["T"].tolist() == [1.0, 2.0, 3.0] and o["level"].tolist() == [0, 1, 2] and o["label"].tolist() == [0, 0, 0]
    assert out[0]["level"].tolist() == [0, 0, -1] and out[0]["label"].tolist() == [0, 1, -1]


def test_infinite_seeds_and_nan_times():
    kind = [1, 0, 1, 0]
    edges = [(0, 1, -5.0, R.P2F), (2, 3, 7.0, R.P2F), (0, 3, math.nan, R.P2F), (1, 2, math.nan, R.F2P)]
    o = both(kind, edges, [0, 2], [-INF, INF])[-1]
    assert o["T"].tolist() == [-INF, -5.0, INF, INF]
    assert o["level"].tolist() == [0, 1, 0, -1]                       # +inf seed: a root that reaches nothing


def test_rows_not_sorted_by_time_and_direction_and_kind_rules():
    # row of f3 holds a late edge first; file <-> file and process <-> process edges never open; a p->f edge needs bit 0
    kind = [1, 1, 0, 0, 0]
    edges = [(0, 3, 9.0, R.P2F), (1, 3, 4.0, R.P2F), (0, 1, 2.0, 3), (2, 3, 1.0, 3), (0, 4, 1.5, R.F2P), (0, 2, 1.0, R.P2F),
             (2, 1, 3.0, R.F2P)]
    o = both(kind, edges, [0], [0.0])[-1]
    assert o["T"].tolist() == [0.0, 3.0, 1.0, 4.0, INF]
    assert o["pred"][3] == csr(5, edges)[0][3] + 1                    # the row's second position: the 4.0 edge


def test_ties_take_the_lowest_position_and_labels_follow_it():
    kind = [1, 1, 0]
    o = both(kind, [(1, 2, 5.0, R.P2F), (0, 2, 5.0, R.P2F)], [0, 1], [1.0, 2.0], labels=[3, 4])[-1]
    assert o["pred"][2] == 0 and o["label"][2] == 4                   # row 2 starts at position 0


def test_random_graphs_both_restatements():
    rng = np.random.default_rng(3)
    for trial in range(30):
        n = int(rng.integers(2, 14))
        kind = rng.integers(0, 2, n)
        m = int(rng.integers(0, 40))
        edges = [(int(rng.integers(n)), int(rng.integers(n)), float(rng.integers(0, 6)) if rng.random() > 0.05 else math.nan,
                  int(rng.integers(0, 4))) for _ in range(m)]
        k = int(rng.integers(0, n + 1))
        seeds = rng.permutation(n)[:k].tolist()
        st = [float(rng.integers(-1, 5)) for _ in seeds]
        both(kind, edges, seeds, st, labels=[int(x) for x in rng.integers(0, 3, k)])


def test_invalid_inputs():
    rowptr, col, et, fl = csr(3, [(0, 1, 1.0, R.P2F), (1, 2, 2.0, R.F2P)])
    kind = [1, 0, 1]
    ok = dict(rowptr=rowptr, col=col, node_kind=kind, edge_flow=fl, edge_time=et, seeds=[0], seed_time=[0.0], seed_label=[0])
    R.closure(**ok)
    bad = [(dict(col=np.array([0, 3])), "col holds"), (dict(col=np.array([-1, 1])), "col holds"),
           (dict(node_kind=[1, 2, 1]), "node_kind"), (dict(edge_flow=np.array([1, 4], np.uint8)), "edge_flow"),
           (dict(seeds=[3]), "seed node ids"), (dict(seeds=[-1]), "seed node ids"),
           (dict(seeds=[0, 0], seed_time=[0.0, 1.0], seed_label=[0, 0]), "distinct"),
           (dict(seed_time=[math.nan]), "NaN"), (dict(seed_label=[-1]), "labels")]
    for kw, msg in bad:
        with pytest.raises(ValueError, match=msg):
            R.closure(**dict(ok, **kw))
    with pytest.raises(ValueError, match="max_hops"):
        R.closure(**ok, max_hops=-2)


# ---- ground truth of the constructed trace, by the statement (the GPU test runs the kernels on it)
def _statement_contamination(ev, only_pid="pid:454"):
    g = G.graph_from_events(ev, observable=True)
    kind = np.asarray(g.meta["node_kind"])
    names = g.meta["names"]
    enc = [v for v, nm in enumerate(names) if nm.endswith(".lockbit3")]
    et, eev = g.meta["edge_time"](), g.meta["edge_event"]
    fl = IR.flagged(g.rowptr, g.col, kind, np.zeros(g.num_nodes, np.float32), INF, enc, g.meta["edge_label"].astype(np.float32),
                    et, eev)
    incs = IR.incidents(fl, None)
    seeds, st, sl = [], [], []
    for i, r in enumerate(incs):
        if r["owner"] >= 0:
            seeds.append(r["owner"]); st.append(r["onset"]); sl.append(i)
        for v in r["files"]:
            j = int(np.nonzero(fl["files"] == v)[0][0])
            seeds.append(v); st.append(fl["onset"][j]); sl.append(i)
    o = R.closure(g.rowptr, g.col, kind, g.meta["edge_flow"](), et, seeds, st, sl)
    lab = {names[r["owner"]]: i for i, r in enumerate(incs)}[only_pid]
    got = {names[v]: v for v in o["nodes"].tolist() if o["level"][v] >= 1 and o["label"][v] == lab}
    return g, o, got


def test_constructed_trace_ground_truth_by_the_statement():
    ev, a_open, a_write = constructed_trace()
    g, o, got = _statement_contamination(ev)
    assert set(got) == {"pid:%d" % A, NIGHTLY, NOTE}
    assert o["level"][got[NIGHTLY]] == 2 and o["level"][got[NOTE]] == 1 and o["level"][got["pid:%d" % A]] == 1
    assert not ({"pid:%d" % APP, "pid:%d" % B, OLD} & set(got))


def test_constructed_trace_with_bystanders_by_the_statement():
    ev, _, _ = constructed_trace(bystanders=2)
    g, o, got = _statement_contamination(ev)
    assert set(got) == {"pid:%d" % A, NIGHTLY, NOTE, "pid:455", "pid:456"}


# ---- emitter and CLI
def _inc(i="pid:454"):
    return {"id": i, "host": None, "process": i, "owner": 1, "files": [0], "n_files": 1, "onset": 1.0, "onset_event": None,
            "end": 2.0, "end_event": None, "size_mb": 1.0, "later_other_events": 0, "max_score": None}


def test_emitter_contaminated_fields_and_hostile_names():
    names = ["/a/x.lockbit3", "pid:454", "/b/n.tar", "pid:600"]
    ev = lambda t, pid, sc, p: {"time": t, "pid": pid, "syscall": sc, "path": p}
    o, w = ev(5.0, 600, "openat", names[0]), ev(9.0, 600, "write", names[2])
    cont = {"pid:454": [{"node": 3, "name": "pid:600", "kind": "process", "since": 5.0, "since_event": o, "hops": 1, "via": [o]},
                        {"node": 2, "name": names[2], "kind": "file", "since": 9.0, "since_event": w, "hops": 2, "via": [o, w]}]}
    plan = emit.undo_plan(names, [0], incidents=[_inc(), _inc("pid:9")], step_incident={0: "pid:454"}, file_recovery={},
                          contamination=cont)
    c = plan["incidents"][0]["contaminated"]
    assert [x["name"] for x in c] == ["pid:600", "/b/n.tar"] and plan["incidents"][1]["contaminated"] == []
    assert "recovery_point" not in c[0] and c[1]["recovery_point"] == {"before": 9.0, "event": w}
    assert c[1]["via"] == [o, w] and c[1]["hops"] == 2 and not any("hostile_name" in x for x in c)
    hostile = {"pid:454": [dict(cont["pid:454"][1], name="/b/\x1b]x.tar")],
               "pid:9": [dict(cont["pid:454"][0], via=[ev(5.0, 600, "openat", "/a/\n")])]}
    plan = emit.undo_plan(names, [0], incidents=[_inc(), _inc("pid:9")], step_incident={0: "pid:454"}, file_recovery={},
                          contamination=hostile)
    assert all(i["contaminated"][0]["hostile_name"] for i in plan["incidents"])
    assert plan["steps"] == emit.undo_plan(names, [0], incidents=[_inc(), _inc("pid:9")], step_incident={0: "pid:454"},
                                           file_recovery={})["steps"]


def test_plan_without_contamination_is_byte_identical():
    names = ["/a/x.lockbit3", "pid:7", "/a/y.dat"]
    kw = dict(scores=[0.0, 1.0, 2.0, 2.5], restores=[{"position": 1, "dir": "/a", "covers": [2]}])
    base = emit.to_json(emit.undo_plan(names, [0, 1, 2], **kw))
    assert emit.to_json(emit.undo_plan(names, [0, 1, 2], contamination=None, **kw)) == base
    inc = dict(incidents=[_inc("pid:7")], step_incident={0: "pid:7"}, file_recovery={0: (1.0, None, 0)})
    assert emit.to_json(emit.undo_plan(names, [0, 1, 2], **kw, **inc)) == \
        emit.to_json(emit.undo_plan(names, [0, 1, 2], contamination=None, **kw, **inc))
    assert '"contaminated"' not in emit.to_json(emit.undo_plan(names, [0, 1, 2], **kw, **inc))


def _args(**kw):
    d = dict(incidents=False, incident=None, incident_threshold=None, contamination=False, contamination_hops=None)
    d.update(kw)
    return argparse.Namespace(**d)


def test_cli_contamination_argument_rules():
    undo.check_contamination_args(_args())
    undo.check_contamination_args(_args(incidents=True, contamination=True))
    undo.check_contamination_args(_args(incident="pid:4", contamination=True, contamination_hops=2))
    undo.check_contamination_args(_args(incidents=True, contamination=True, contamination_hops=-1))
    with pytest.raises(SystemExit, match="needs --incidents"):
        undo.check_contamination_args(_args(contamination=True))
    with pytest.raises(SystemExit, match="needs --contamination"):
        undo.check_contamination_args(_args(incidents=True, contamination_hops=3))
    with pytest.raises(SystemExit, match="-1"):
        undo.check_contamination_args(_args(incidents=True, contamination=True, contamination_hops=-2))


def test_stream_keeps_the_earliest_since_per_node_key():
    from types import SimpleNamespace
    sp = stream.StreamingPlanner(None, None, incidents=True, contamination=True)
    r = lambda node, name, since: {"node": node, "name": name, "kind": "file", "since": since, "since_event": None, "hops": 1,
                                   "via": []}
    tick = {}
    sp._note_contamination(SimpleNamespace(contamination={"pid:1": [r(4, "/x", 7.0)]}), lambda n, nm: nm, tick)
    sp._note_contamination(SimpleNamespace(contamination={"pid:1": [r(9, "/x", 5.0), r(2, "/y", 8.0)]}), lambda n, nm: nm, tick)
    assert {k: v["since"] for k, v in tick["pid:1"].items()} == {"/x": 5.0, "/y": 8.0}
    assert {k: v["since"] for k, v in sp.contamination["pid:1"].items()} == {"/x": 5.0, "/y": 8.0}
    with pytest.raises(ValueError, match="needs incidents"):
        stream.StreamingPlanner(None, None, contamination=True)
