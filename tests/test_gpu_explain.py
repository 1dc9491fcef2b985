"""Per-node GraphSAGE-T edge attributions on the GPU (nerrf_b200.explain) against the float64 autograd oracle
(oracle/explain_ref.py): attributions within the layer backward's gradient tolerance, top-k sets equal outside near-ties,
the receptive-field kernels edge for edge against the host restatement, and the plan carrying the evidence."""
import json
import os

import numpy as np
import pytest
import torch

from nerrf_b200 import explain as EX, graph as G, ingest, pipeline, stream
from nerrf_b200.ai.models import GraphSAGE_T
from oracle import explain_ref as XR

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M1 = os.path.join(ROOT, "tests", "golden", "m1_trace.jsonl")


def dev_graph(g):
    t = lambda a: (a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))).cuda()
    return G.TemporalGraph(t(g.rowptr), t(g.col), t(g.ew), t(g.x), g.meta)


def host(a):
    return a.cpu().numpy() if torch.is_tensor(a) else np.asarray(a)


def model_of(layers, seed=1):
    return GraphSAGE_T(32, 128, layers, seed=seed).cuda()


def full_attr(gd, model, nodes, max_edges=EX.DEFAULT_MAX_EDGES):
    """every kept edge's GPU attribution, per target: [(global CSR positions, a)] (subgraph scope only)"""
    sg = EX.subgraphs(gd.rowptr, gd.col, gd.ew, gd.x, nodes, model.num_layers, max_edges)
    hs = EX.forward_saved(model, sg["x"], sg["rowptr"], sg["col"], sg["ew"])
    d = EX.edge_weight_grad(model, hs, sg["rowptr"], sg["col"], sg["ew"], sg["target"].long())
    a = (sg["ew"] * d).cpu().numpy()
    seg, epos = host(sg["seg"]), host(sg["epos"])
    return sg, hs, [(epos[seg[i]:seg[i + 1]], a[seg[i]:seg[i + 1]]) for i in range(len(seg) - 1)]


def check_target(gd, model, v, pos, a_gpu, ex, k):
    rp, col, ew, x = host(gd.rowptr), host(gd.col), host(gd.ew), host(gd.x)
    p = model.oracle_params()
    z, a_ref = XR.attributions(p, x, rp, col, ew, v)
    want = a_ref[pos]
    rms = float(np.sqrt((want ** 2).mean())) if want.size else 0.0
    err = np.abs(a_gpu - want)
    assert (err <= 2e-4 * np.abs(want) + 2e-5 * rms + 1e-30).all(), (v, float(err.max()))
    outside = np.ones(col.size, bool); outside[pos] = False
    assert not a_ref[outside].any()                               # nothing outside the receptive field
    assert abs(ex["logit"] - z) <= 1e-4 * max(1.0, abs(z))
    # top-k: the GPU picks and the oracle's agree outside near-ties at the k-th value
    got = [e["pos"] for e in ex["edges"]]
    assert len(got) == min(k, pos.size)
    mag = np.abs(a_ref)
    tol = 2e-4 * mag.max() + 2e-5 * rms if pos.size else 0.0
    if got:
        kth = np.sort(mag[pos])[::-1][len(got) - 1]
        for q in got:
            assert mag[q] >= kth - tol
        for q in XR.top_edges(np.where(outside, 0.0, a_ref), len(got)):
            if mag[q] > kth + tol:
                assert q in got
        for e in ex["edges"]:
            assert e["src"] == col[e["pos"]] and rp[e["dst"]] <= e["pos"] < rp[e["dst"] + 1]


def run_case(g, layers, nodes, k=8, seed=1):
    gd = dev_graph(g)
    model = model_of(layers, seed)
    res = EX.explain_nodes(gd, model, nodes, k=k)
    _, _, fa = full_attr(gd, model, nodes)
    for v, ex, (pos, a) in zip(nodes, res, fa):
        assert ex["scope"] == "subgraph"
        check_target(gd, model, int(v), pos, a, ex, k)
    return gd, model, res


@pytest.mark.parametrize("layers", [2, 3])
def test_m1_golden_trace(layers):
    g = G.graph_from_events(G.read_trace_jsonl(M1), observable=True)
    kind = np.asarray(g.meta["node_kind"])
    nodes = np.concatenate([np.nonzero(kind == 0)[0][:12], np.nonzero(kind == 1)[0][:2]])
    gd, model, res = run_case(g, layers, nodes)
    ev = g.meta["edge_event"]
    for ex in res:
        for e in ex["edges"]:
            assert e["event"] == ev[e["pos"]]


def test_fleet_window_with_bystanders_overlapping_neighbourhoods():
    cols, _ = stream.fleet_columns(40, 3, seed=2, n_files=20, benign_files=10, bystanders=2)
    ds = stream.DeviceStream(cols, "cuda", observable=True)
    t0, t1 = ds.span()
    g = ds.window_graph(t1 - 60.0, t1, 60.0)
    kind = np.asarray(g.meta["node_kind"])
    lab = np.asarray(g.meta["label"])
    files = np.nonzero((kind == 0) & (lab == 1))[0][:16]          # encrypted files: several per attacking process
    nodes = np.concatenate([files, np.nonzero(kind == 1)[0][:4]])
    _, _, res = run_case(g, 2, nodes)
    ev = host(g.meta["edge_event"]())
    sel = host(ds.d_order)
    for ex in res:
        for e in ex["edges"]:
            assert e["event"] == ev[e["pos"]] and e["event"] in sel


@pytest.mark.parametrize("layers", [1, 2])
def test_hub_rows_and_zero_in_degree(layers):
    g = G.synthetic_graph(N=1500, E=12000, seed=3, hub="dst")
    rp = g.rowptr.astype(np.int64)
    deg = np.diff(rp)
    assert deg.max() > 128
    hubs = np.argsort(-deg, kind="stable")[:3]
    zero = np.nonzero(deg == 0)[0][:3]
    assert zero.size
    nodes = np.concatenate([hubs, zero, [7, 8]])
    max_e = EX.DEFAULT_MAX_EDGES
    run_case(g, layers, nodes)
    gd = dev_graph(g)
    res = EX.explain_nodes(gd, model_of(layers), zero, k=4, max_edges_per_target=max_e)
    if layers == 1:
        assert all(r["edges"] == [] for r in res)


def test_receptive_field_kernel_matches_host_restatement():
    g = G.synthetic_graph(N=800, E=4000, seed=5, hub="src")
    gd = dev_graph(g)
    rp, col = g.rowptr.astype(np.int64), g.col
    nodes = np.array([0, 1, 5, 5, 17, 400, 799])
    for hops in (1, 2, 3):
        sg = EX.subgraphs(gd.rowptr, gd.col, gd.ew, gd.x, nodes, hops, 1 << 20)
        assert sg["fit"].all()
        seg, node, epos, tgt = host(sg["seg"]), host(sg["node"]), host(sg["epos"]), host(sg["target"])
        b_rp, b_col = host(sg["rowptr"]), host(sg["col"])
        no = np.concatenate([[0], np.cumsum(sg["counts"][:, 0])])
        for i, v in enumerate(nodes):
            nn, dd, ee = XR.receptive_field(rp, col, v, hops)
            assert np.array_equal(node[no[i]:no[i + 1]], nn)
            assert np.array_equal(epos[seg[i]:seg[i + 1]], ee)
            assert node[tgt[i]] == v
            assert np.array_equal(node[b_col[seg[i]:seg[i + 1]]], col[ee])
            kept = np.where(dd < hops, np.diff(rp)[nn], 0)
            assert np.array_equal(np.diff(b_rp[no[i]:no[i + 1] + 1]), kept)
        assert np.array_equal(host(sg["x"]), g.x[node])


def test_subgraph_logits_equal_full_graph_bit_for_bit_and_runs_repeat():
    g = G.synthetic_graph(N=3000, E=24000, seed=9, hub="dst")
    gd = dev_graph(g)
    model = model_of(2)
    nodes = np.array([0, 3, 11, 2999, 1500])
    h_full, _ = model(gd.x, gd.rowptr, gd.col, gd.ew)
    sg, hs, _ = full_attr(gd, model, nodes)
    got = hs[-1][sg["target"].long()]
    assert torch.equal(got, h_full[torch.from_numpy(nodes).cuda()])
    a = EX.explain_nodes(gd, model, nodes, k=16)
    b = EX.explain_nodes(gd, model, nodes, k=16)
    assert json.dumps(a) == json.dumps(b)
    _, _, fa = full_attr(gd, model, nodes)
    _, _, fb = full_attr(gd, model, nodes)
    for (p1, a1), (p2, a2) in zip(fa, fb):
        assert np.array_equal(p1, p2) and np.array_equal(a1.view(np.uint32), a2.view(np.uint32))


def test_edge_budget_full_graph_scope_and_cap():
    g = G.synthetic_graph(N=600, E=3000, seed=4, hub="dst")
    gd = dev_graph(g)
    model = model_of(2)
    deg = np.diff(g.rowptr.astype(np.int64))
    big = np.argsort(-deg, kind="stable")[:3]                        # three targets over a tiny budget
    small = np.nonzero(deg == 1)[0][:1]
    nodes = np.concatenate([small, big])
    counts = EX.subgraphs(gd.rowptr, gd.col, gd.ew, gd.x, nodes, 2, 40)["counts"]
    assert counts[0, 0] > 0 and (counts[1:, 0] == -1).all()
    res = EX.explain_nodes(gd, model, nodes, k=8, max_edges_per_target=40, max_full_graph_targets=2)
    assert [r["scope"] for r in res] == ["subgraph", "full_graph", "full_graph", None]
    assert "reason" in res[3] and "edges" not in res[3]
    full = EX.explain_nodes(gd, model, nodes[:3], k=8)              # the same targets within the default budget
    for r, f in zip(res[:3], full):
        assert [e["pos"] for e in r["edges"]] == [e["pos"] for e in f["edges"]]
        assert np.allclose([e["attr"] for e in r["edges"]], [e["attr"] for e in f["edges"]], rtol=1e-5, atol=1e-7)
    _, _, fa = full_attr(gd, model, nodes[1:2], max_edges=1 << 20)
    check_target(gd, model, int(nodes[1]), fa[0][0], fa[0][1], res[1], 8)


def _toy_models():
    from nerrf_b200.ai import train as T
    from nerrf_b200.ai.models.lstm import LSTMScorer
    model, scorer = GraphSAGE_T(G.F_IN, 128, 2), LSTMScorer()
    torch.manual_seed(0)
    T.train(model, scorer, T.toy_set(range(100, 104)), epochs=25)
    return model.cuda(), scorer.cuda()


def test_pipeline_explain_keeps_the_plan_and_points_at_the_ransomware(tmp_path):
    events = G.read_trace_jsonl(M1)
    g = G.graph_from_events(events, observable=True)
    seq, lengths, nodes = pipeline.file_sequences(events, g, observable=True)
    model, scorer = _toy_models()
    kw = dict(top_a=64, n_rollouts=256, depth=20, iterations=8)
    r0 = pipeline.run(g, seq, lengths, nodes, model, scorer, kill_candidates=True, **kw)
    r1 = pipeline.run(g, seq, lengths, nodes, model, scorer, kill_candidates=True, explain=4, **kw)
    assert r0.plan.actions == r1.plan.actions and r0.plan_nodes == r1.plan_nodes and r0.evidence is None
    assert set(r1.evidence) == set(r1.plan_nodes)
    attackers = {int(e["pid"]) for e in events if e["event"] in G.ATTACK_EVENTS}
    lab = np.asarray(g.meta["label"])
    enc = [n for n in r1.plan_nodes if lab[n] == 1]
    assert enc
    hits = [r1.evidence[n]["edges"][0]["event"]["pid"] in attackers for n in enc]
    assert all(hits), "top evidence of %d of %d encrypted-file steps is not an event of the ransomware process" % (
        len(hits) - sum(hits), len(hits))
    from nerrf_b200.ai.planner import emit
    p0, p1 = emit.from_pipeline(g, r0), emit.from_pipeline(g, r1)
    strip = lambda p: [{k: v for k, v in s.items() if not k.startswith("evidence") and k != "hostile_name"} for s in p["steps"]]
    assert strip(p0) == strip(p1)
    assert emit.to_shell(p0) == emit.to_shell(p1)
    assert all(len(s["evidence"]) == 4 for s in p1["steps"] if "node" in s)


def test_undo_cli_writes_evidence(tmp_path):
    from nerrf_b200 import undo
    out = tmp_path / "plan.json"
    undo.main(["--trace", M1, "--train-epochs", "5", "--explain", "3", "--out", str(out), "--rollouts", "256"])
    plan = json.loads(out.read_text())
    steps = [s for s in plan["steps"] if "node" in s]
    assert steps and all("evidence" in s and "evidence_logit" in s for s in steps)
    e = steps[0]["evidence"][0]
    assert set(e["event"]) == {"time", "pid", "syscall", "path"}


def test_streaming_planner_evidence_for_new_steps():
    cols, _ = stream.fleet_columns(30, 2, seed=1, n_files=15, benign_files=10)
    model, scorer = model_of(2), None
    from nerrf_b200.ai.models.lstm import LSTMScorer
    scorer = LSTMScorer().cuda()
    sp = stream.StreamingPlanner(model, scorer, window_s=60.0, tick_s=30.0, top_a=64, n_rollouts=256, depth=16,
                                 iterations=4, kill_candidates=True, explain=2)
    ticks = sp.run(cols)
    assert any(t.planned for t in ticks)
    for t in ticks:
        assert set(t.planned) <= set(t.evidence)
        for key, ex in t.evidence.items():
            assert ex["scope"] == "subgraph" and len(ex["edges"]) <= 2
            for e in ex["edges"]:
                assert set(e["event"]) >= {"time", "pid", "syscall", "path"}
