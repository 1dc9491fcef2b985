"""Incidents without a GPU: the numpy statement of DESIGN.md 1.4 (oracle/incident_ref.py) on hand-built graphs, the
factored attribution rule (pipeline.file_owners) against the rule process_kill_candidates applied before it was
factored out, the plan fields of the emitter, and the CLI's argument rules."""
import argparse
import json
import math
import os

import numpy as np
import pytest
import torch

from nerrf_b200 import graph as G, ingest, pipeline, stream, undo
from nerrf_b200.ai.planner import emit
from oracle import incident_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M1 = os.path.join(ROOT, "tests", "golden", "m1_trace.jsonl")

# nodes: 0 file A, 1 proc P, 2 proc Q, 3 file B, 4 file C (empty row), 5 file D (only a file source), 6 file E
KIND = np.array([0, 1, 1, 0, 0, 0, 0])
ROWS = {0: [1, 2, 1, 2], 1: [0], 2: [0], 3: [1, 5], 4: [], 5: [3], 6: [2, 2, 1]}


def hand_graph():
    rowptr = np.zeros(len(KIND) + 1, np.int64)
    col = []
    for v in range(len(KIND)):
        col += ROWS[v]
        rowptr[v + 1] = len(col)
    col = np.asarray(col, np.int64)
    E = col.shape[0]
    return rowptr, col, 100.0 + np.arange(E, dtype=np.float64), 1000 + np.arange(E, dtype=np.int64)


def test_writer_rule_positions_and_later_counts():
    rp, col, t, ev = hand_graph()
    fl = R.flagged(rp, col, KIND, np.ones(7, np.float32), 0.5, edge_time=t, edge_event=ev)
    assert fl["files"].tolist() == [0, 3, 4, 5, 6]
    by = {int(v): i for i, v in enumerate(fl["files"])}
    a = by[0]                                       # row [P, Q, P, Q]: last process Q; Q at 1 and 3; P at 2 is later
    assert (fl["owner"][a], fl["first"][a], fl["last"][a], fl["later"][a]) == (2, 1, 3, 1)
    assert fl["onset"][a] == t[1] and fl["onset_event"][a] == ev[1] and fl["end"][a] == t[3]
    b = by[3]                                       # row [P, D]: the last toucher is a file -> P
    assert (fl["owner"][b], fl["first"][b], fl["last"][b], fl["later"][b]) == (1, 6, 6, 0)
    c = by[4]                                       # empty row
    assert fl["owner"][c] == -1 and fl["first"][c] == -1 and math.isnan(fl["onset"][c]) and fl["onset_event"][c] == -1
    d = by[5]                                       # no process source: the row's first / last position, later 0
    assert (fl["owner"][d], fl["first"][d], fl["last"][d], fl["later"][d]) == (-1, 8, 8, 0)
    e = by[6]                                       # row [Q, Q, P]: writer P at 11; nothing after it
    assert (fl["owner"][e], fl["first"][e], fl["later"][e]) == (1, 11, 0)


def test_edge_rule_ties_to_the_later_position_and_nan_ranks_highest():
    rp, col, t, ev = hand_graph()
    ea = np.zeros(col.shape[0], np.float32)
    ea[0:4] = [0.9, 0.1, 0.9, 0.2]                  # tie between P at 0 and P at 2 -> 2 -> owner P
    ea[9:12] = [0.3, np.nan, 0.99]                  # NaN ranks above every number -> Q at 10
    fl = R.flagged(rp, col, KIND, np.ones(7, np.float32), 0.5, edge_attack=ea, edge_time=t, edge_event=ev)
    by = {int(v): i for i, v in enumerate(fl["files"])}
    assert (fl["owner"][by[0]], fl["first"][by[0]], fl["last"][by[0]], fl["later"][by[0]]) == (1, 0, 2, 2)
    assert (fl["owner"][by[6]], fl["first"][by[6]], fl["later"][by[6]]) == (2, 9, 1)


def test_threshold_nan_scores_and_seeds():
    rp, col, _, _ = hand_graph()
    s = np.array([0.5, 0.9, 0.9, np.nextafter(np.float32(0.5), np.float32(0)), np.nan, 0.1, 0.7], np.float32)
    assert R.flagged(rp, col, KIND, s, 0.5)["files"].tolist() == [0, 6]        # s = tau flagged, NaN never, processes never
    assert R.flagged(rp, col, KIND, s, 0.5, seeds=[4, 4, 3])["files"].tolist() == [0, 3, 4, 6]
    with pytest.raises(ValueError, match="not a file"):
        R.flagged(rp, col, KIND, s, 0.5, seeds=[1])
    with pytest.raises(ValueError, match="seed node ids"):
        R.flagged(rp, col, KIND, s, 0.5, seeds=[7])
    with pytest.raises(ValueError, match="NaN"):
        R.flagged(rp, col, KIND, s, float("nan"))
    with pytest.raises(ValueError, match="node_kind"):
        R.flagged(rp, col, np.where(KIND == 1, 2, 0), s, 0.5)


def test_one_unattributed_incident_per_host_and_the_order():
    rp, col, t, ev = hand_graph()
    src = np.array([0, 0, 0, 0, 1, 1, 1])
    fl = R.flagged(rp, col, KIND, np.ones(7, np.float32), 0.5, edge_time=t, edge_event=ev)
    inc = R.incidents(fl, src, np.arange(7, dtype=np.float32), np.linspace(0, 1, 7, dtype=np.float32))
    keys = [(r["source"], r["owner"]) for r in inc]
    # onsets: (0, Q) 101, (0, P) 106, (1, -1) 108 (file D; file C has no time), (1, P) 111
    assert keys == [(0, 2), (0, 1), (1, -1), (1, 1)]
    un = inc[2]
    assert un["files"] == [4, 5] and un["onset"] == t[8] and un["later"] == 0
    assert inc[0]["size_mb"] == 0.0 and inc[1]["size_mb"] == 3.0
    assert sum(1 for r in inc if r["owner"] == -1) == 1            # host 0 has no unattributed file here


def _old_owners(g, cand, edge_attack=None):
    """process_kill_candidates' attribution as it was written before file_owners was factored out of it"""
    kind = torch.as_tensor(np.asarray(g.meta["node_kind"]))
    rp = torch.from_numpy(np.asarray(g.rowptr)).long()
    col = torch.from_numpy(np.asarray(g.col)).long()
    cand = torch.from_numpy(np.asarray(cand, np.int64))
    if edge_attack is not None:
        return pipeline._edge_owners(kind, rp, col, cand, np.asarray(edge_attack, np.float32))
    owner = np.full(cand.shape[0], -1, np.int64)
    last = rp[cand + 1] - 1
    has = (rp[cand + 1] > rp[cand]).numpy()
    src = col[last.clamp_min(0)]
    is_proc = (kind[src] == 1).numpy() & has
    owner[is_proc] = src.numpy()[is_proc]
    for i in np.nonzero(has & ~is_proc)[0].tolist():
        n = int(cand[i]); s_ = col[rp[n]:rp[n + 1]]; s_ = s_[kind[s_] == 1]
        if s_.numel():
            owner[i] = int(s_[-1])
    return owner


def _graphs():
    yield G.graph_from_jsonl(M1, observable=True)
    for by in (0, 2):
        cols, _ = stream.fleet_columns(30, 3, seed=4, n_files=12, benign_files=8, bystanders=by)
        yield ingest.graph_from_columns(cols, observable=True)
    yield G.graph_from_jsonl(M1, observable=True, merge_renames=False)


@pytest.mark.parametrize("rule", ["writer", "edges"])
def test_file_owners_is_the_kill_attribution_and_the_statement(rule):
    rng = np.random.default_rng(3)
    for g in _graphs():
        kind = np.asarray(g.meta["node_kind"])
        files = np.nonzero(kind == 0)[0]
        ea = None
        if rule == "edges":
            ea = rng.random(g.num_edges).astype(np.float32)
            ea[rng.random(g.num_edges) < 0.3] = 0.5                  # many ties
        got = pipeline.file_owners(g, files, ea)
        assert np.array_equal(got, _old_owners(g, files, ea))
        fl = R.flagged(g.rowptr, g.col, kind, np.zeros(g.num_nodes, np.float32), 0.5, seeds=files, edge_attack=ea)
        assert np.array_equal(fl["owner"], got)


def test_edge_time_is_the_event_time():
    g = G.graph_from_jsonl(M1, observable=True)
    info = g.meta["event_info"]
    et, ev = g.meta["edge_time"](), g.meta["edge_event"]
    assert et.dtype == np.float64 and et.shape == ev.shape
    pick = np.arange(0, ev.shape[0], 97)
    assert [r["time"] for r in info(ev[pick])] == et[pick].tolist()


def _inc(host=None, path="/a/x.lockbit3"):
    ev = {"time": 10.0, "pid": 7, "syscall": "write", "path": path}
    return {"id": "pid:7" if host is None else host + "/pid:7", "host": host, "process": "pid:7", "owner": 1, "files": [0, 2],
            "n_files": 2, "onset": 10.0, "onset_event": ev, "end": 12.0, "end_event": dict(ev, time=12.0), "size_mb": 1.5,
            "later_other_events": 3, "max_score": 0.9}


def test_emitter_incident_fields_restore_points_and_hostile_names():
    names = ["/a/x.lockbit3", "pid:7", "/a/y.lockbit3", "/a/z\n.lockbit3"]
    ev = lambda t, p: {"time": t, "pid": 7, "syscall": "write", "path": p}
    rec = {0: (10.0, ev(10.0, names[0]), 1), 2: (9.0, ev(9.0, names[2]), 2), 3: (9.0, ev(9.0, names[3]), 4)}
    restores = [{"position": 0, "dir": "/a", "covers": [2, 3]}]
    plan = emit.undo_plan(names, [0, 1], restores=restores, incidents=[_inc()],
                          step_incident={0: "pid:7", 1: "pid:7", 2: "pid:7", 3: "unattributed"}, file_recovery=rec)
    assert plan["incidents"][0]["onset"] == {"time": 10.0, "event": ev(10.0, names[0])}
    assert plan["incidents"][0]["files"] == [0, 2] and "hostile_name" not in plan["incidents"][0]
    r, f, k = plan["steps"]
    assert r["incidents"] == ["pid:7", "unattributed"]
    # the earliest cover (9.0, ties to the lower node id 2), later events summed over the covers
    assert r["recovery_point"] == {"before": 9.0, "event": ev(9.0, names[2]), "later_other_events": 6}
    assert f["incident"] == "pid:7" and f["recovery_point"]["later_other_events"] == 1
    assert k["incident"] == "pid:7" and "recovery_point" not in k
    bad = emit.undo_plan(names, [3], incidents=[_inc(path="/a/\x1b[2J")], step_incident={3: None}, file_recovery=rec)
    assert bad["incidents"][0]["hostile_name"] and bad["steps"][0]["hostile_name"] and bad["steps"][0]["incident"] is None
    assert emit.to_shell(plan) == emit.to_shell(emit.undo_plan(names, [0, 1], restores=restores))
    with pytest.raises(ValueError, match="bad host name"):
        emit.undo_plan(names, [0], incidents=[_inc(host="../x")], step_incident={}, file_recovery={})


def test_plan_without_incidents_has_none_of_the_fields():
    names = ["/a/x.lockbit3", "pid:7", "/a/y.dat"]
    base = emit.to_json(emit.undo_plan(names, [0, 1, 2], scores=[0.0, 1.0, 2.0, 2.5],
                                       restores=[{"position": 1, "dir": "/a", "covers": [2]}]))
    again = emit.to_json(emit.undo_plan(names, [0, 1, 2], scores=[0.0, 1.0, 2.0, 2.5],
                                        restores=[{"position": 1, "dir": "/a", "covers": [2]}], incidents=None,
                                        step_incident=None, file_recovery=None))
    assert base == again
    assert not any(k in base for k in ('"incident', '"recovery_point'))


def _args(**kw):
    d = dict(incidents=False, incident=None, incident_threshold=None)
    d.update(kw)
    return argparse.Namespace(**d)


def test_cli_incident_argument_rules():
    undo.check_incident_args(_args())
    undo.check_incident_args(_args(incidents=True, incident_threshold=0.3))
    undo.check_incident_args(_args(incident="a/pid:4", incident_threshold=float("inf")))
    with pytest.raises(SystemExit, match="needs --incidents"):
        undo.check_incident_args(_args(incident_threshold=0.3))
    with pytest.raises(SystemExit, match="must be a number"):
        undo.check_incident_args(_args(incidents=True, incident_threshold=float("nan")))
    with pytest.raises(SystemExit, match="needs an incident id"):
        undo.check_incident_args(_args(incident=""))


def test_restore_takes_the_incidents_of_its_covers_as_the_pipeline_labels_them():
    from types import SimpleNamespace
    names = ["/a/x.lockbit3", "pid:7", "/a/y.lockbit3", "/a/z.lockbit3", "pid:8"]
    kind = np.array([0, 1, 0, 0, 1])
    recs = [dict(_inc(), owner=1), dict(_inc(), id="pid:8", process="pid:8", owner=4, files=[3])]
    ev = lambda t, p: {"time": t, "pid": 7, "syscall": "write", "path": p}
    per_file = {0: {"incident": "pid:7", "onset": 10.0, "event": ev(10.0, names[0]), "later": 0},
                2: {"incident": "pid:7", "onset": 9.0, "event": ev(9.0, names[2]), "later": 1},
                3: {"incident": "pid:8", "onset": 11.0, "event": ev(11.0, names[3]), "later": 0}}
    restores = [{"position": 1, "dir": "/a", "covers": [2, 3]}]          # covered files are not plan nodes
    step_inc = pipeline.step_incidents([1, 0], restores, kind, recs, per_file)
    assert step_inc == {1: "pid:7", 0: "pid:7", 2: "pid:7", 3: "pid:8"}
    res = SimpleNamespace(node_score=np.zeros(5, np.float32), plan_nodes=[1, 0], plan=SimpleNamespace(scores=None),
                          restores=restores, incidents=recs, step_incident=step_inc,
                          file_recovery={v: (f["onset"], f["event"], f["later"]) for v, f in per_file.items()})
    g = SimpleNamespace(meta={"names": names})
    kill, rst, f = emit.from_pipeline(g, res)["steps"]
    assert rst["op"] == "restore_snapshot_dir" and rst["incidents"] == ["pid:7", "pid:8"]
    assert rst["recovery_point"] == {"before": 9.0, "event": ev(9.0, names[2]), "later_other_events": 1}
    assert kill["incident"] == "pid:7" and f["incident"] == "pid:7"


class _Names(list):
    def take(self, idx):
        return [self[int(i)] for i in idx]


def test_stream_folds_a_second_planning_pass_into_the_tick_record():
    from types import SimpleNamespace
    names = _Names(["/a/x", "pid:7", "/a/y", "/a/z"])
    g = SimpleNamespace(meta={"size_mb": np.array([1.0, 0.0, 2.0, 4.0], np.float32)})
    score = torch.tensor([0.9, 0.0, 0.2, 0.7])
    rec = lambda files, onset, end: {"id": "pid:7", "host": None, "process": "pid:7", "owner": 1, "files": files,
                                     "n_files": len(files), "onset": onset, "onset_event": {"t": onset}, "end": end,
                                     "end_event": {"t": end}, "size_mb": float(g.meta["size_mb"][files].sum()),
                                     "later_other_events": 2 * len(files), "max_score": 0.9}
    rec_ = {0: (5.0, None, 2), 2: (4.0, None, 2), 3: (6.0, None, 2)}
    one = SimpleNamespace(incidents=[rec([0], 5.0, 8.0)], node_score=score, file_recovery=rec_, plan_nodes=[0],
                          step_incident={0: "pid:7"})
    two = SimpleNamespace(incidents=[rec([0, 2, 3], 4.0, 9.0)], node_score=score, file_recovery=rec_, plan_nodes=[2],
                          step_incident={2: "pid:7"})
    sp = stream.StreamingPlanner(None, None, incidents=True)
    key = lambda n, nm: nm
    tick, nodes, steps = {}, {}, {}
    sp._note_incidents(one, g, names, key, {"/a/x"}, ["/a/x"], tick, nodes, steps)
    sp._note_incidents(two, g, names, key, {"/a/y"}, ["/a/y"], tick, nodes, steps)
    t = tick["pid:7"]
    assert t["files"] == ["/a/x", "/a/y", "/a/z"] and t["n_files"] == 3
    assert (t["onset"], t["end"], t["size_mb"], t["later_other_events"], t["max_score"]) == (4.0, 9.0, 7.0, 6, 0.9)
    assert steps == {"/a/x": "pid:7", "/a/y": "pid:7"}
    run = sp.incidents["pid:7"]
    assert set(run) == set(stream.StreamingPlanner._RUNNING_FIELDS)
    assert run["files"] == ["/a/x", "/a/y", "/a/z"] and (run["onset"], run["end"]) == (4.0, 9.0)
