"""The edge head backward kernel (csrc/sage_edge_bwd.cu) against the float64 statement, the full model gradient through
SageLayerFn + EdgeHeadFn, training the edge head on the GPU, and the planner attributing files by it (needs an H100)."""
import ctypes as C

import numpy as np
import pytest
import torch

from edge_head_ref import edge_head_backward, model_backward_with_edges
from gpu_util import assert_close_fp32
from nerrf_b200 import _lib as L, graph as G, pipeline
from nerrf_b200.ai import autograd as AG, train as T
from nerrf_b200.ai.models import GraphSAGE_T
from nerrf_b200.ai.models.lstm import LSTMScorer

pytestmark = pytest.mark.gpu


def _grad_close(got, want, what):
    """The bound of the layer backward tests: |got - want| <= 2e-4 |want| + 2e-5 rms(want)."""
    assert_close_fp32(got, torch.as_tensor(np.asarray(want, np.float64)), rtol=2e-4, atol_rms=2e-5, what=what)


def _edge_bwd(h, We, dL, rp, tg_rowptr, t_eid, dh=True, dw=True):
    n = h.shape[0]
    out_dh = torch.empty_like(h) if dh else None
    dW = torch.empty(256, 2, device=h.device) if dw else None
    db = torch.empty(2, device=h.device) if dw else None
    need = C.c_size_t()
    L.check(L.lib().nerrf_sage_edge_head_bwd_workspace_bytes(n, 128, C.byref(need)), "workspace_bytes")
    ws = torch.empty(need.value, dtype=torch.uint8, device=h.device)
    L.check(L.lib().nerrf_sage_edge_head_bwd(L.ptr(h), L.ptr(We), L.ptr(dL), L.ptr(rp), int(rp.dtype == torch.int64),
                                             L.ptr(tg_rowptr), L.ptr(t_eid), int(tg_rowptr.dtype == torch.int64),
                                             L.ptr(out_dh), L.ptr(dW), L.ptr(db), L.ptr(ws), need.value, n, 128,
                                             L.current_stream_ptr()), "nerrf_sage_edge_head_bwd")
    torch.cuda.synchronize()
    return out_dh, dW, db


@pytest.mark.parametrize("N,E,hub,rp64,t64", [(3001, 40000, "src", False, False), (3001, 40000, "dst", False, True),
                                              (70001, 300000, "src", True, True), (1000, 9999, "dst", True, False),
                                              (77, 0, "src", False, False), (1, 5, "src", False, False)])
def test_edge_head_backward_kernel_matches_the_float64_statement(N, E, hub, rp64, t64):
    g = G.synthetic_graph(N=N, E=E, seed=N + E, hub=hub, f_in=32)
    deg_in, deg_out = np.diff(g.rowptr.astype(np.int64)), np.bincount(g.col, minlength=N)
    if E >= 40000:
        assert deg_in.max() > 128 or deg_out.max() > 128
    dev = "cuda"
    rp = torch.from_numpy(g.rowptr.astype(np.int64 if rp64 else np.int32)).to(dev)
    tg = AG.TrainGraph(rp, torch.from_numpy(g.col).to(dev), torch.from_numpy(g.ew).to(dev))
    t_rowptr = tg.t_rowptr.to(torch.int64 if t64 else torch.int32)
    t_eid = tg.t_eid.to(torch.int64 if t64 else torch.int32)
    rng = np.random.default_rng(N)
    h = torch.from_numpy(np.maximum(rng.standard_normal((N, 128)), 0).astype(np.float32)).to(dev)
    We = GraphSAGE_T(32, 128, 1, seed=N).edge_W.detach().to(dev)
    dL = torch.from_numpy(rng.standard_normal((E, 2)).astype(np.float32)).to(dev)
    dh, dW, db = _edge_bwd(h, We, dL, rp, t_rowptr, t_eid)
    want = edge_head_backward(h.cpu(), We.cpu(), dL.cpu(), g.rowptr, g.col)
    _grad_close(dh, want[0], "dh"); _grad_close(dW, want[1], "d edge_W"); _grad_close(db, want[2], "d edge_b")
    # a second call gives the same bits; each half alone gives the same bits as both together
    dh2, dW2, db2 = _edge_bwd(h, We, dL, rp, t_rowptr, t_eid)
    assert torch.equal(dh, dh2) and torch.equal(dW, dW2) and torch.equal(db, db2)
    dh3, none_w, none_b = _edge_bwd(h, We, dL, rp, t_rowptr, t_eid, dw=False)
    none_h, dW3, db3 = _edge_bwd(h, We, dL, rp, t_rowptr, t_eid, dh=False)
    assert none_w is None and none_b is None and none_h is None
    assert torch.equal(dh, dh3) and torch.equal(dW, dW3) and torch.equal(db, db3)


def test_edge_head_backward_refuses_bad_arguments():
    h = torch.zeros(4, 128, device="cuda")
    rp = torch.zeros(5, dtype=torch.int32, device="cuda")
    We = torch.zeros(256, 2, device="cuda")
    lib = L.lib()
    assert lib.nerrf_sage_edge_head_bwd(L.ptr(h), L.ptr(We), None, L.ptr(rp), 0, L.ptr(rp), None, 0, L.ptr(h), None,
                                        None, None, 0, 4, 64, None) == -1
    assert b"128" in lib.nerrf_last_error()
    assert lib.nerrf_sage_edge_head_bwd(L.ptr(h), None, None, L.ptr(rp), 0, L.ptr(rp), None, 0, L.ptr(h), None,
                                        None, None, 0, 4, 128, None) == -1
    mis = C.c_void_p(h.data_ptr() + 4)
    assert lib.nerrf_sage_edge_head_bwd(L.ptr(h), L.ptr(We), None, L.ptr(rp), 0, L.ptr(rp), None, 0, mis, None,
                                        None, None, 0, 3, 128, None) == -1
    assert b"aligned" in lib.nerrf_last_error()


@pytest.mark.parametrize("N,E,layers,rp64,seed", [(3000, 30000, 2, False, 1), (700, 9000, 1, True, 2)])
def test_node_and_edge_loss_gradients_match_the_oracle(N, E, layers, rp64, seed):
    g = G.synthetic_graph(N=N, E=E, seed=seed, f_in=32)
    model = GraphSAGE_T(32, 128, layers, seed=seed).cuda()
    rng = np.random.default_rng(seed)
    dlogit = rng.standard_normal(N).astype(np.float32)
    dedge = rng.standard_normal((E, 2)).astype(np.float32)
    x = torch.from_numpy(g.x).cuda().requires_grad_()
    rp = torch.from_numpy(g.rowptr.astype(np.int64 if rp64 else np.int32)).cuda()
    tg = AG.TrainGraph(rp, torch.from_numpy(g.col).cuda(), torch.from_numpy(g.ew).cuda())

    def grads():
        model.zero_grad(); x.grad = None
        nl, el = AG.sage_logits(model, x, tg)
        ((nl * torch.from_numpy(dlogit).cuda()).sum() + (el * torch.from_numpy(dedge).cuda()).sum()).backward()
        return [x.grad.clone()] + [p.grad.clone() for p in model.parameters()]

    got = grads()
    want = model_backward_with_edges(model.oracle_params(), g.x, g.rowptr, g.col, g.ew, dlogit, dedge)
    _grad_close(x.grad, want["x"], "dx")
    for k in ("node_w", "node_b", "edge_W", "edge_b"):
        _grad_close(getattr(model, k).grad, want[k], f"d {k}")
    for l, (dW, db) in enumerate(want["layers"]):
        _grad_close(model.weights[l].grad, dW, f"dW[{l}]"); _grad_close(model.biases[l].grad, db, f"db[{l}]")
    assert all(torch.equal(a, b) for a, b in zip(got, grads()))


@pytest.fixture(scope="module")
def gpu_edge_model():
    torch.manual_seed(0)
    model, scorer = GraphSAGE_T(32, 128, 2), LSTMScorer()
    T.train(model, scorer, T.toy_set(range(100, 104), bystanders=2), epochs=25, lr=3e-3, device="cuda", edge_weight=1.0)
    return model, scorer


def test_edge_training_on_the_gpu_meets_the_gates(gpu_edge_model):
    model, _ = gpu_edge_model
    assert model.edge_head_trained is True
    auc = T.evaluate(model, None, T.toy_set(range(900, 903), bystanders=2), device="cuda", edges=True)
    assert auc["edge_auc"] >= 0.90 and auc["edge_auc_encrypted"] >= 0.90 and auc["gnn_auc"] >= 0.90, auc
    ex = T._to(T.make_example(901, n_files=30, benign_files=40, bystanders=2), "cuda")
    _, _, el = model(ex["x"], ex["rowptr"], ex["col"], ex["ew"], return_edge_logits=True)
    with torch.no_grad():
        _, want = T.sage_logits(model, ex["x"], ex["rowptr"], ex["col"], ex["ew"])
    assert float((el - want).abs().max()) <= 1e-4


def test_pipeline_attributes_encrypted_files_to_the_attacker(gpu_edge_model):
    model, scorer = gpu_edge_model
    ex = T.make_example(907, n_files=25, benign_files=30, bystanders=2)
    g = ex["graph"]
    names = g.meta["names"]
    kw = dict(top_a=4096, n_rollouts=1024, depth=40, iterations=8, kill_candidates=True)
    res = pipeline.run(g, ex["seq"].numpy(), ex["lengths"].numpy(), ex["seq_nodes"], model, scorer, **kw)
    assert res.kill_attribution == "edges"
    killed = [names[int(v)] for v in res.plan_nodes if g.meta["node_kind"][int(v)] == 1]
    reverted = sorted(int(v) for v in res.plan_nodes if g.meta["node_kind"][int(v)] == 0)
    assert killed == ["pid:454"], killed
    assert reverted == sorted(np.nonzero(g.meta["label"])[0].tolist())
    assert names[int(res.candidates[0])] == "pid:454"            # the attacker owns the most candidate files
    # the same weights without the mark: the writer rule, exactly as before
    model.edge_head_trained = False
    try:
        res_w = pipeline.run(g, ex["seq"].numpy(), ex["lengths"].numpy(), ex["seq_nodes"], model, scorer, **kw)
    finally:
        model.edge_head_trained = True
    assert res_w.kill_attribution == "writer"
    a_cand = res_w.candidates[res_w.n_kill:]
    pids, _ = pipeline.process_kill_candidates(g, a_cand)
    assert np.array_equal(res_w.candidates[:res_w.n_kill], pids)
    assert set(names[int(v)] for v in pids) - {"pid:454"}        # a bystander is taken for some file's writer
