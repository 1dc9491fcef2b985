"""The GraphSAGE-T edge head off the GPU: the hand-written float64 backward against torch.autograd over the forward spec,
per-pair edge labels, bystander processes in the simulated traces (and the planner's writer rule they defeat), and
training the edge head with edge_weight > 0."""
import numpy as np
import pytest
import torch

from edge_head_ref import edge_head_backward, model_backward_with_edges
from nerrf_b200 import graph as G, pipeline, trace_sim
from nerrf_b200.ai import train as T
from nerrf_b200.ai.models import GraphSAGE_T
from oracle import sage_ref


def _graph(kind):
    rng = np.random.default_rng(7)
    if kind == "isolated":                      # nodes 5..8 have no edges at all
        N, src, dst = 9, [0, 1, 2, 3, 4, 0, 2], [1, 2, 3, 4, 0, 3, 1]
    elif kind == "self_loops_multi_edges":
        N, src, dst = 6, [1, 1, 1, 2, 2, 3, 5, 5, 0], [1, 1, 2, 3, 3, 2, 5, 0, 5]
    elif kind == "no_out_edges":                # a star into node 0: nodes 0 and 7 have no out-edges
        N, src, dst = 8, [1, 2, 3, 4, 5, 6, 6], [0, 0, 0, 0, 0, 0, 1]
    elif kind == "no_edges":
        N, src, dst = 5, [], []
    else:
        N = 40
        src, dst = rng.integers(0, N, 300).tolist(), rng.integers(0, N, 300).tolist()
    src, dst = np.asarray(src, np.int64), np.asarray(dst, np.int64)
    t = rng.random(src.shape[0]).astype(np.float32) * 60
    rowptr, col, ew = G.csr_from_edges(src, dst, t, np.ones(src.shape[0], np.float32), N)
    return N, rowptr, col, ew


KINDS = ["isolated", "self_loops_multi_edges", "no_out_edges", "no_edges", "random"]


def _rel_close(got, want, rtol=1e-10):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = max(float(np.abs(want).max()) if want.size else 0.0, 1e-300)
    assert got.shape == want.shape and (want.size == 0 or float(np.abs(got - want).max()) <= rtol * scale)


@pytest.mark.parametrize("kind", KINDS)
def test_edge_head_backward_equals_autograd(kind):
    N, rowptr, col, ew = _graph(kind)
    E = col.shape[0]
    g = torch.Generator().manual_seed(3)
    h = torch.randn(N, 128, generator=g, dtype=torch.float64, requires_grad=True)
    We = torch.randn(256, 2, generator=g, dtype=torch.float64, requires_grad=True)
    be = torch.randn(2, generator=g, dtype=torch.float64, requires_grad=True)
    dL = torch.randn(E, 2, generator=g, dtype=torch.float64)
    params = {"layers": [], "node_w": torch.zeros(128, dtype=torch.float64), "node_b": torch.zeros(1, dtype=torch.float64),
              "edge_W": We, "edge_b": be}
    _, _, el = sage_ref.forward(params, h, torch.from_numpy(rowptr), torch.from_numpy(col), torch.from_numpy(ew),
                                edge_logits=True)
    (el * dL).sum().backward()
    dh, dWe, dbe = edge_head_backward(h, We, dL, rowptr, col)
    _rel_close(dh, h.grad); _rel_close(dWe, We.grad); _rel_close(dbe, be.grad)


@pytest.mark.parametrize("kind", KINDS)
def test_model_backward_with_both_heads_equals_autograd(kind):
    N, rowptr, col, ew = _graph(kind)
    E = col.shape[0]
    p = sage_ref.make_params(in_dim=32, hidden=128, num_layers=2, seed=5)
    p = {"layers": [(W.double().requires_grad_(), b.double().requires_grad_()) for W, b in p["layers"]],
         **{k: p[k].double().requires_grad_() for k in ("node_w", "node_b", "edge_W", "edge_b")}}
    g = torch.Generator().manual_seed(4)
    x = torch.randn(N, 32, generator=g, dtype=torch.float64, requires_grad=True)
    dscore = torch.randn(N, generator=g, dtype=torch.float64)
    dL = torch.randn(E, 2, generator=g, dtype=torch.float64)
    _, score, el = sage_ref.forward(p, x, torch.from_numpy(rowptr), torch.from_numpy(col), torch.from_numpy(ew),
                                    edge_logits=True)
    ((score * dscore).sum() + (el * dL).sum()).backward()
    dlogit = (dscore * score * (1 - score)).detach()            # d/d(node logit) of sum(dscore * sigmoid(logit))
    want = model_backward_with_edges(p, x, rowptr, col, ew, dlogit, dL)
    _rel_close(want["x"], x.grad)
    for k in ("node_w", "node_b", "edge_W", "edge_b"):
        _rel_close(want[k], p[k].grad)
    for (dW, db), (W, b) in zip(want["layers"], p["layers"]):
        _rel_close(dW, W.grad); _rel_close(db, b.grad)


# ------------------------------------------------------------------------------------------------ traces and labels
def _bystander_graph(seed=3):
    ev = trace_sim.lockbit_trace(n_files=20, seed=seed, benign_files=20, bystanders=2)
    return ev, G.graph_from_events(ev, observable=True)


@pytest.mark.parametrize("seed", [0, 3, 11])
def test_bystanders_zero_emits_the_same_trace(seed):
    assert trace_sim.lockbit_trace(seed=seed, bystanders=0) == trace_sim.lockbit_trace(seed=seed)
    assert trace_sim.lockbit_trace(n_files=7, seed=seed, benign_files=9, bystanders=0) == \
        trace_sim.lockbit_trace(n_files=7, seed=seed, benign_files=9)


def test_bystanders_touch_encrypted_files_after_their_encryption():
    ev, _ = _bystander_graph()
    ts = lambda e: G._parse_ts(e["timestamp"])
    done = {G._stem(e["path"]): ts(e) for e in ev if e["event"] == "file_encrypt_complete"}
    pids = {e["pid"] for e in ev}
    assert len(pids) == 3
    late = [e for e in ev if e["pid"] != 454 and e["path"].endswith(".lockbit3") and ts(e) > done[G._stem(e["path"])]]
    assert late and {e["phase"] for e in late} == {"benign"} and {e["event"] for e in late} <= {"openat", "write"}
    assert all(ts(a) <= ts(b) for a, b in zip(ev, ev[1:]))
    early = [e for e in ev if e["pid"] != 454 and ts(e) < min(done.values())]
    assert early


def test_edge_labels_are_per_pair_symmetric_and_in_csr_order():
    ev, g = _bystander_graph()
    lab = g.meta["edge_label"]
    assert lab.dtype == np.uint8 and lab.shape == (g.num_edges,)
    names, kind = g.meta["names"], g.meta["node_kind"]
    node_of_pid = {int(n[4:]): i for i, n in enumerate(names) if kind[i] == 1}
    attacked = {(node_of_pid[e["pid"]], g.meta["file_keys"][G._stem(e["path"])]) for e in ev if e["event"] in G.ATTACK_EVENTS}
    rp = g.rowptr.astype(np.int64)
    by_pair = {}
    for v in range(g.num_nodes):
        for i in range(rp[v], rp[v + 1]):
            u = int(g.col[i])
            want = int((u, v) in attacked or (v, u) in attacked)
            assert lab[i] == want, (u, v)
            by_pair.setdefault(frozenset((u, v)), set()).add(int(lab[i]))
    assert all(len(s) == 1 for s in by_pair.values())          # one label per pair, both directions
    enc = set(np.nonzero(g.meta["label"])[0].tolist())
    for v in range(g.num_nodes):
        for i in range(rp[v], rp[v + 1]):
            u = int(g.col[i])
            if v in enc and kind[u] == 1:
                assert lab[i] == (1 if names[u] == "pid:454" else 0)
    # file <-> file rename links are 0
    ren = [dict(e, event="rename", new_path=e["path"] + ".lockbit3") for e in ev if e["event"] == "file_encrypt_start"]
    g2 = G.graph_from_events(ev + ren, merge_renames=False)
    rp2 = g2.rowptr.astype(np.int64)
    dst2 = np.repeat(np.arange(g2.num_nodes), np.diff(rp2))
    ff = (g2.meta["node_kind"][g2.col] == 0) & (g2.meta["node_kind"][dst2] == 0)
    assert ff.any() and not g2.meta["edge_label"][ff].any() and g2.meta["edge_label"].any()


def test_writer_rule_takes_a_bystander_for_an_encrypted_file_and_edge_rule_does_not():
    """Documents the defect the edge head fixes: the last process to touch a file is taken for its writer."""
    _, g = _bystander_graph()
    enc = np.nonzero(g.meta["label"])[0]
    names = g.meta["names"]
    pids, guard = pipeline.process_kill_candidates(g, enc)
    owners = {names[int(pids[k])] for k in guard[guard >= 0]}
    assert owners - {"pid:454"}, owners                       # some encrypted file is "owned" by a bystander
    # with a perfect edge classifier (P(attack) = the label) every encrypted file is attributed to the attacker
    pids_e, guard_e = pipeline.process_kill_candidates(g, enc, edge_attack=g.meta["edge_label"].astype(np.float32))
    assert [names[int(p)] for p in pids_e] == ["pid:454"] and (guard_e == 0).all()
    conf = pipeline.edge_kill_confidence(g, enc, pids_e, g.meta["edge_label"].astype(np.float32))
    assert conf.tolist() == [1.0]


# ------------------------------------------------------------------------------------------------ training
@pytest.fixture(scope="module")
def edge_trained():
    torch.manual_seed(0)
    model = GraphSAGE_T(32, 128, 2)
    T.train(model, None, T.toy_set(range(100, 104), bystanders=2), epochs=25, lr=3e-3, edge_weight=1.0)
    return model


def test_edge_training_on_the_cpu_meets_the_gates(edge_trained):
    assert edge_trained.edge_head_trained is True
    assert "edge_head_trained" not in edge_trained.state_dict()
    auc = T.evaluate(edge_trained, None, T.toy_set(range(900, 903), bystanders=2), edges=True)
    assert auc["edge_auc"] >= 0.90 and auc["edge_auc_encrypted"] >= 0.90 and auc["gnn_auc"] >= 0.90, auc


def test_edge_weight_zero_trains_exactly_as_before():
    ex = T.toy_set(range(100, 102), windows=0)
    runs = []
    threads = torch.get_num_threads()
    torch.set_num_threads(1)                  # multi-threaded CPU reductions are not bit-reproducible run to run
    try:
        for kw in ({}, {"edge_weight": 0.0}):
            torch.manual_seed(0)
            m = GraphSAGE_T(32, 128, 2)
            We0 = m.edge_W.detach().clone()
            T.train(m, None, ex, epochs=3, lr=3e-3, **kw)
            assert not hasattr(m, "edge_head_trained") and torch.equal(m.edge_W.detach(), We0)
            runs.append([p.detach().clone() for p in m.parameters()])
    finally:
        torch.set_num_threads(threads)
    assert all(torch.equal(a, b) for a, b in zip(*runs))


def test_node_logits_are_the_node_head_over_the_shared_embeddings():
    ex = T.make_example(5, n_files=8, benign_files=8, bystanders=1)
    m = GraphSAGE_T(32, 128, 2)
    nl, el = T.sage_logits(m, ex["x"], ex["rowptr"], ex["col"], ex["ew"])
    assert torch.equal(nl, T.sage_node_logits(m, ex["x"], ex["rowptr"], ex["col"], ex["ew"]))
    with torch.no_grad():
        _, _, want = sage_ref.forward(m.oracle_params(), ex["x"], ex["rowptr"], ex["col"], ex["ew"], edge_logits=True)
    assert float((el.detach() - want).abs().max()) <= 1e-5


def test_edge_checkpoint_round_trip_into_the_undo_cli_loader(tmp_path):
    from nerrf_b200 import undo
    out = str(tmp_path / "w.pt")
    T.main(["--traces", "1", "--epochs", "1", "--no-lstm", "--edge-loss", "1.0", "--out", out])
    assert torch.load(out, map_location="cpu")["edge_head_trained"] is True
    model, _ = undo.load_models(out, 0)
    assert model.edge_head_trained is True
    T.main(["--traces", "1", "--epochs", "1", "--no-lstm", "--out", out])
    assert not getattr(undo.load_models(out, 0)[0], "edge_head_trained", False)
