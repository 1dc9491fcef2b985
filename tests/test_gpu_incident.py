"""Incidents on the GPU (nerrf_b200.incident; DESIGN.md 1.4) against the per-row numpy statement (oracle/incident_ref.py):
flagged lists, owners, positions, counts, event ids and float64 times bit for bit, size_mb within 1e-12 relative, on the
m1 trace, fleet windows, a hub row, int64 rowptr, empty / full F and streams of several colliding hosts; the same
incidents from every graph builder; ground truth from the simulator's attacker pids; and the plan fields end to end."""
import json
import math
import os

import numpy as np
import pytest
import torch

from nerrf_b200 import graph as G, incident as I, ingest, pipeline, stream
from nerrf_b200.ai.models import GraphSAGE_T
from nerrf_b200.ai.models.lstm import LSTMScorer
from nerrf_b200.ai.planner import emit
from oracle import incident_ref as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M1 = os.path.join(ROOT, "tests", "golden", "m1_trace.jsonl")
GT = os.path.join(ROOT, "tests", "golden", "m1_ground_truth.csv")


def host(a):
    if callable(a):
        a = a()
    return a.cpu().numpy() if torch.is_tensor(a) else np.asarray(a)


def dev_graph(g, rp64=False):
    t = lambda a: (a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))).cuda()
    rp = t(g.rowptr)
    rp = rp.to(torch.int64) if rp64 else rp
    return G.TemporalGraph(rp, t(g.col).to(torch.int32), t(g.ew), t(g.x), g.meta)


def bits(a):
    return np.asarray(a, np.float64).view(np.int64)


def device_run(gd, score, tau, seeds, ea):
    kind = torch.from_numpy(np.asarray(gd.meta["node_kind"]).astype(np.int8)).cuda()
    sc = torch.as_tensor(score).cuda().float()
    et = torch.as_tensor(host(gd.meta["edge_time"])).cuda().double()
    ev = torch.as_tensor(host(gd.meta["edge_event"])).cuda().long()
    ea_t = None if ea is None else torch.as_tensor(ea).cuda().float()
    files, fi, fr = I.flag_files(gd.rowptr, gd.col, kind, sc, tau, seeds, ea_t, et, ev)
    src = torch.from_numpy(np.asarray(gd.meta.get("node_source", np.zeros(gd.num_nodes)), np.int64).astype(np.int32)).cuda()
    size = torch.from_numpy(np.asarray(gd.meta["size_mb"], np.float32)).cuda()
    ii, ir, grouped, fin = I.group_files(files, fi, fr, src, size, sc)
    return [host(a) for a in (files, fi, fr, ii, ir, grouped, fin)]


def check(g, score, tau=0.5, seeds=None, ea=None, rp64=False):
    """kernels == statement, device owners == pipeline.file_owners, two runs == the same bits -> the oracle incidents"""
    gd = dev_graph(g, rp64)
    score = np.asarray(score, np.float32)
    out = device_run(gd, score, tau, seeds, ea)
    files, fi, fr, ii, ir, grouped, fin = out
    fl = R.flagged(host(g.rowptr), host(g.col), g.meta["node_kind"], score, tau, seeds, ea, host(g.meta["edge_time"]),
                   host(g.meta["edge_event"]))
    assert np.array_equal(files, fl["files"])
    for c, k in enumerate(("owner", "first", "last", "later", "onset_event", "end_event")):
        assert np.array_equal(fi[:, c], fl[k]), k
    assert np.array_equal(bits(fr[:, 0]), bits(fl["onset"])) and np.array_equal(bits(fr[:, 1]), bits(fl["end"]))
    assert np.array_equal(fi[:, 0], pipeline.file_owners(g, files, ea))
    src = g.meta.get("node_source")
    inc = R.incidents(fl, src, g.meta["size_mb"], score)
    assert ii.shape[0] == len(inc)
    for r, o in enumerate(inc):
        assert (ii[r, 0], ii[r, 1], ii[r, 3], ii[r, 4], ii[r, 5], ii[r, 6]) == (o["source"], o["owner"], o["n_files"],
                                                                                o["onset_event"], o["end_event"], o["later"])
        assert grouped[ii[r, 2]:ii[r, 2] + ii[r, 3]].tolist() == o["files"]
        assert bits(ir[r, :2]).tolist() == bits([o["onset"], o["end"]]).tolist()
        assert abs(ir[r, 2] - o["size_mb"]) <= 1e-12 * max(abs(o["size_mb"]), 1e-300)
        assert (math.isnan(ir[r, 3]) and math.isnan(o["max_score"])) or ir[r, 3] == o["max_score"]
        assert set(files[fin == r].tolist()) == set(o["files"])
    again = device_run(gd, score, tau, seeds, ea)
    for a, b in zip(out, again):
        assert a.tobytes() == b.tobytes()
    return inc


def rules(g, seed=0):
    rng = np.random.default_rng(seed)
    ea = rng.random(g.num_edges).astype(np.float32)
    ea[rng.random(g.num_edges) < 0.2] = 0.75                   # ties
    return [None, ea]


def scores(g, seed=0):
    rng = np.random.default_rng(seed)
    s = rng.random(g.num_nodes).astype(np.float32)
    s[rng.random(g.num_nodes) < 0.05] = 0.5                    # s = tau
    s[rng.random(g.num_nodes) < 0.02] = np.nan
    return s


def test_m1_trace_both_rules_and_empty_and_full_sets():
    g = G.graph_from_jsonl(M1, observable=True)
    files = np.nonzero(np.asarray(g.meta["node_kind"]) == 0)[0]
    for ea in rules(g):
        check(g, scores(g), 0.5, seeds=files[::7], ea=ea)
        assert check(g, scores(g), float("inf"), ea=ea) == []
        full = check(g, scores(g), float("-inf"), ea=ea)
        assert sum(o["n_files"] for o in full) == int(np.isfinite(scores(g)[files]).sum())   # NaN is never flagged


@pytest.mark.parametrize("bystanders", [0, 2])
def test_fleet_windows(bystanders):
    cols, _ = stream.fleet_columns(60, 4, seed=3, n_files=20, benign_files=15, bystanders=bystanders)
    ts = cols.timestamp
    w = stream.window(cols, float(ts.min()) + 5.0, float(ts.min()) + 65.0)
    g = ingest.graph_from_columns(w, device="cuda", observable=True)
    for ea in rules(g, 1):
        check(g, scores(g, 2), 0.5, ea=ea)


def hub_graph(n_hub_edges=(1 << 16) + 3001, n_procs=40, seed=5):
    """file 0 with a row of > 2^16 edges from processes and files, plus small rows; times and events random"""
    rng = np.random.default_rng(seed)
    N = 1 + n_procs + 30
    kind = np.zeros(N, np.int64); kind[1:1 + n_procs] = 1
    rows = [rng.integers(1, N, n_hub_edges)] + [rng.integers(1, N, rng.integers(0, 40)) for _ in range(N - 1)]
    rowptr = np.zeros(N + 1, np.int64); rowptr[1:] = np.cumsum([r.size for r in rows])
    col = np.concatenate(rows).astype(np.int32)
    E = col.size
    meta = {"node_kind": kind, "size_mb": rng.random(N).astype(np.float32) * 3, "node_source": np.zeros(N, np.int64),
            "edge_time": np.sort(rng.random(E)) * 1e3 + 1.7e9, "edge_event": rng.permutation(E).astype(np.int64)}
    return G.TemporalGraph(rowptr.astype(np.int32), col, np.ones(E, np.float32), np.zeros((N, 32), np.float32), meta)


@pytest.mark.parametrize("rp64", [False, True])
def test_hub_row_over_2_16_edges_and_int64_rowptr(rp64):
    g = hub_graph()
    for ea in rules(g, 7):
        check(g, scores(g, 3), 0.5, seeds=[0], ea=ea, rp64=rp64)


@pytest.mark.parametrize("k", [1, 2, 3, 8])
def test_colliding_hosts(k):
    cols = stream.concat_columns([c for c, _, _ in stream.host_streams(k, 10, 2, seed=4, bystanders=1)])
    g = ingest.graph_from_columns(cols, device="cuda", observable=True)
    for ea in rules(g, k):
        inc = check(g, scores(g, k), 0.5, ea=ea)
        assert len({(o["source"], o["owner"]) for o in inc}) == len(inc)


def _gt_graph(bystanders, n=40, k=3):
    cols, enc, pids = stream.fleet_columns(n, k, seed=6, n_files=45, benign_files=20, return_pids=True, bystanders=bystanders)
    g = ingest.graph_from_columns(cols, device="cuda", observable=True)
    names = g.meta["names"]
    seeds = [v for v, nm in enumerate(names) if nm in enc]
    return g, seeds, pids, enc


def _by_attacker(recs, g):
    names = g.meta["names"]
    return {r["process"]: {names[v] for v in r["files"]} for r in recs}


def test_ground_truth_one_incident_per_attacker():
    g, seeds, pids, enc = _gt_graph(0)
    recs = I.incidents(g, torch.zeros(g.num_nodes, device="cuda"), tau=float("inf"), seeds=seeds)
    got = _by_attacker(recs, g)
    assert set(got) == pids and len(recs) == 3
    assert all(len(f) == 45 for f in got.values()) and set().union(*got.values()) == enc


def test_ground_truth_with_bystanders_edge_rule_and_writer_split():
    cols, enc, pids = stream.fleet_columns(40, 3, seed=6, n_files=45, benign_files=20, return_pids=True, bystanders=2)
    ds = stream.DeviceStream(cols, "cuda", observable=True)
    t0, t1 = ds.span()
    g = ds.window_graph(t0 - 1.0, t1, t1 - t0 + 1.0, edge_labels=True)         # the whole stream, with its edge labels
    names = g.meta["names"].take(list(range(g.num_nodes)))
    seeds = [v for v, nm in enumerate(names) if nm in enc]
    zero = torch.zeros(g.num_nodes, device="cuda")
    recs = I.incidents(g, zero, tau=float("inf"), seeds=seeds, edge_attack=g.meta["edge_label"].float())
    got = {r["process"]: {names[v] for v in r["files"]} for r in recs}
    assert set(got) == pids and all(len(f) == 45 for f in got.values()) and set().union(*got.values()) == enc
    writer = I.incidents(g, zero, tau=float("inf"), seeds=seeds)
    # DESIGN.md 2.7: a bystander that opened an encrypted file after the attacker is its last writer
    print("writer rule with bystanders: %d incidents, files per incident %s" % (len(writer), {r["id"]: r["n_files"] for r in writer}))
    assert len(writer) >= len(pids)


def test_two_hosts_same_pid_get_host_prefixed_ids():
    parts = stream.host_streams(2, 8, 1, attacked_hosts=[0, 1], seed=2)
    cols = stream.concat_columns([c for c, _, _ in parts])
    g = ingest.graph_from_columns(cols, device="cuda", observable=True)
    names = g.meta["names"]
    seeds = [v for v, nm in enumerate(names) if nm in parts[0][1]]
    recs = I.incidents(g, torch.zeros(g.num_nodes, device="cuda"), tau=float("inf"), seeds=seeds, host_names=["a", "b"])
    pid = next(iter(parts[0][2]))
    assert {"a/" + pid, "b/" + pid} <= {r["id"] for r in recs}


def test_device_stream_window_equals_columns_builder():
    cols, _ = stream.fleet_columns(40, 3, seed=8, n_files=20, benign_files=10, bystanders=1)
    ds = stream.DeviceStream(cols, "cuda", observable=True)
    t0, t1 = ds.span()
    for lo in (t0 - 1.0, t0 + 20.0):
        a = ds.window_graph(lo, lo + 60.0, 60.0)
        b = ingest.graph_from_columns(stream.window(cols, lo, lo + 60.0), device="cuda", observable=True)
        key = lambda g: {r["id"]: (r["n_files"], r["onset"], r["end"], r["later_other_events"],
                                   sorted(g.meta["names"].take(r["files"]) if hasattr(g.meta["names"], "take")
                                          else [g.meta["names"][v] for v in r["files"]]))
                         for r in I.incidents(g, torch.as_tensor(g.meta["label"]).float().cuda(), tau=0.5)}
        assert key(a) == key(b) and key(a)


def _planner(**kw):
    model = GraphSAGE_T(G.F_IN, 128, 2, seed=1).cuda()
    return stream.StreamingPlanner(model, LSTMScorer().cuda(), window_s=60.0, tick_s=30.0, top_a=64, n_rollouts=256, depth=16,
                                   iterations=4, kill_candidates=True, **kw)


def test_stream_run_feed_and_plans_unchanged():
    cols, _, pids = stream.fleet_columns(30, 2, seed=1, n_files=15, benign_files=10, return_pids=True)
    plain = _planner().run(cols)
    sp = _planner(incidents=True)
    ticks = sp.run(cols)
    assert [t.planned for t in plain] == [t.planned for t in ticks]
    for t in ticks:
        assert set(t.planned) <= set(t.step_incident)
        for k_, i_ in t.step_incident.items():
            assert i_ is None or i_ in t.incidents
    # stable ids: one running record per id seen in any tick, onset = the min over ticks, files = the union
    assert sp.incidents and set(sp.incidents) == set().union(*[set(t.incidents) for t in ticks])
    for i_, run in sp.incidents.items():
        per = [t.incidents[i_] for t in ticks if i_ in t.incidents]
        assert run["onset"] == min((r["onset"] for r in per if r["onset"] is not None), default=None)
        assert set(run["files"]) == set().union(*[set(r["files"]) for r in per]) and run["n_files"] == len(run["files"])
    live = _planner(incidents=True)
    order = np.argsort(cols.timestamp, kind="stable")                             # a tracker delivers in time order
    wire = b"".join(ingest.encode_columns(cols)[i] for i in order.tolist())
    out = []
    for k in range(0, len(wire), len(wire) // 16 + 1):                         # chunks cut anywhere
        out += live.feed(wire[k:k + len(wire) // 16 + 1])
    out += live.flush()
    strip = lambda t: {i: (r["n_files"], r["onset"], r["end"], sorted(r["files"])) for i, r in t.incidents.items()}
    assert [strip(t) for t in out] == [strip(t) for t in ticks]


def test_stream_running_onset_is_the_whole_stream_onset():
    cols, enc, pids = stream.fleet_columns(20, 2, seed=9, n_files=15, benign_files=10, return_pids=True)
    sp = _planner(incidents=True, incident_tau=float("-inf"))                   # every file of every window is flagged
    ticks = sp.run(cols)
    ids = [set(t.incidents) for t in ticks]
    g = ingest.graph_from_columns(cols, device="cuda", observable=True)                # the whole stream, per the statement
    kind = np.asarray(g.meta["node_kind"])
    fl = R.flagged(host(g.rowptr), host(g.col), kind, np.zeros(g.num_nodes, np.float32), float("-inf"),
                   edge_time=host(g.meta["edge_time"]), edge_event=host(g.meta["edge_event"]))
    names = g.meta["names"]
    whole = {("unattributed" if r["owner"] < 0 else names[r["owner"]]): r for r in R.incidents(fl, g.meta["node_source"])}
    assert pids <= set(whole)
    for pid in pids:
        assert pid in sp.incidents and sp.incidents[pid]["onset"] == whole[pid]["onset"]
        assert sp.incidents[pid]["end"] == whole[pid]["end"]
    assert set(sp.incidents) == set().union(*ids)


def _toy_models():
    from nerrf_b200.ai import train as T
    model, scorer = GraphSAGE_T(G.F_IN, 128, 2), LSTMScorer()
    torch.manual_seed(0)
    T.train(model, scorer, T.toy_set(range(100, 104)), epochs=25)
    return model.cuda(), scorer.cuda()


def test_m1_lockbit_plan_incidents():
    events = G.read_trace_jsonl(M1)
    g = G.graph_from_events(events, observable=True)
    seq, lengths, nodes = pipeline.file_sequences(events, g, observable=True)
    model, scorer = _toy_models()
    kw = dict(top_a=64, n_rollouts=256, depth=20, iterations=8, kill_candidates=True)
    r0 = pipeline.run(g, seq, lengths, nodes, model, scorer, **kw)
    r1 = pipeline.run(g, seq, lengths, nodes, model, scorer, incidents=True, **kw)
    assert r0.plan.actions == r1.plan.actions and r0.plan_nodes == r1.plan_nodes
    kind = np.asarray(g.meta["node_kind"])
    assert all(r1.step_incident[n] is not None for n in r1.plan_nodes if kind[n] == 0)
    lab = np.asarray(g.meta["label"])
    enc = set(np.nonzero(lab == 1)[0].tolist())
    assert len(enc) == 45
    ransom = {r["id"]: r for r in r1.incidents}["pid:454"]
    assert enc <= set(ransom["files"])
    gt = open(GT).read().splitlines()
    head, row = gt[0].split(","), gt[1].split(",")
    lo, hi = G._parse_ts(row[head.index("start_iso")]), G._parse_ts(row[head.index("end_iso")])
    assert lo <= ransom["onset"] <= ransom["end"] <= hi, (lo, ransom["onset"], ransom["end"], hi)
    p0, p1 = emit.from_pipeline(g, r0), emit.from_pipeline(g, r1)
    drop = ("incident", "incidents", "recovery_point", "hostile_name")
    assert [{k: v for k, v in s.items() if k not in drop} for s in p1["steps"]] == p0["steps"]
    assert emit.to_shell(p0) == emit.to_shell(p1)


def test_undo_cli_plans_one_incident_of_two(tmp_path):
    from nerrf_b200 import undo
    cols, enc, pids = stream.fleet_columns(6, 2, seed=3, n_files=12, benign_files=6, return_pids=True)
    pb = tmp_path / "two.pb"
    pb.write_bytes(b"".join(ingest.encode_columns(cols)))
    base = ["--trace", str(pb), "--train-epochs", "25", "--rollouts", "256", "--incident-threshold=-inf"]
    full = undo.main(base + ["--incidents", "--out", str(tmp_path / "full.json")])
    known = {i["id"]: i for i in full["incidents"]}
    with pytest.raises(SystemExit, match="unknown incident"):
        undo.main(base + ["--incident", "pid:999999"])
    att = sorted(pids)
    assert set(att) <= set(known)                                              # every file is flagged at tau = -inf
    pid = att[0]
    one = undo.main(base + ["--incident", pid, "--out", str(tmp_path / "one.json")])
    assert one["attack_id"] == pid
    steps = [s for s in one["steps"] if "node" in s]
    assert steps and all(s["incident"] == pid for s in steps)
    assert {s["node"] for s in steps} <= set(known[pid]["files"])
    assert not ({s["node"] for s in steps} & set(known[att[1]]["files"]))
    names = ingest.graph_from_columns(cols, observable=True).meta["names"]          # the same node numbering, on the host
    mine = {names[v] for v in known[pid]["files"]} & enc                         # the incident's encrypted files ...
    assert mine and mine <= {s.get("from", s.get("path")) for s in steps}       # ... every one reverted by the plan


def test_restore_steps_carry_their_covers_incidents():
    from nerrf_b200 import trace_sim
    from nerrf_b200.ai import train as T
    torch.manual_seed(0)
    model, scorer = GraphSAGE_T(G.F_IN, 128, 2), LSTMScorer()
    T.train(model, scorer, T.toy_set(range(100, 104)), epochs=25, lr=3e-3, device="cuda")
    ev = trace_sim.lockbit_trace(n_files=1000, benign_files=10, seed=5)               # a plan with a directory restore
    g = G.graph_from_events(ev, observable=True)
    seq, lengths, nodes = pipeline.file_sequences(ev, g, observable=True)
    kw = dict(top_a=1000, n_rollouts=1024, depth=40, iterations=8, commit_per_search=64, kill_candidates=True,
              restore_candidates=True)
    r0 = pipeline.run(g, seq, lengths, nodes, model, scorer, **kw)
    r1 = pipeline.run(g, seq, lengths, nodes, model, scorer, incidents=True, **kw)
    assert r0.plan.actions == r1.plan.actions and r1.restores
    plan = emit.from_pipeline(g, r1)
    restores = [s for s in plan["steps"] if s["op"] == "restore_snapshot_dir"]
    assert restores
    for s in restores:                                               # covers are not plan nodes, yet each has its incident
        assert s["incidents"] == ["pid:454"] and s["recovery_point"]["before"] is not None
    for r in r1.restores:
        assert all(r1.step_incident[c] == "pid:454" for c in r["covers"])


def test_col_ids_out_of_range_anywhere_are_refused():
    g = hub_graph()
    col = np.array(g.col)
    pos = int(g.rowptr[1])                                           # the first edge after the hub row: a row nobody flags
    assert pos < col.size
    col[pos] = g.num_nodes
    bad = G.TemporalGraph(g.rowptr, col, g.ew, g.x, g.meta)
    gd = dev_graph(bad)
    kind = torch.from_numpy(np.asarray(g.meta["node_kind"]).astype(np.int8)).cuda()
    sc = torch.zeros(g.num_nodes, device="cuda")
    with pytest.raises(ValueError, match="col holds node ids"):
        I.flag_files(gd.rowptr, gd.col, kind, sc, 0.5, [0])
    files, _, _ = I.flag_files(dev_graph(g).rowptr, dev_graph(g).col, kind, sc, 0.5, [0])   # the same call on valid ids
    assert files.cpu().tolist() == [0]
