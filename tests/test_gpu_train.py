"""Weights trained by ai.train (autograd, CPU) drive the CUDA inference path: same scores, same AUC, and the
pipeline plans from MODEL confidence alone (needs an H100)."""
import numpy as np
import pytest
import torch

from nerrf_b200 import pipeline
from nerrf_b200.ai import train as T
from nerrf_b200.ai.models import GraphSAGE_T
from nerrf_b200.ai.models.lstm import LSTMScorer

pytestmark = pytest.mark.gpu


def test_trained_weights_through_the_cuda_kernels():
    torch.manual_seed(0)
    model, scorer = GraphSAGE_T(32, 128, 2), LSTMScorer()
    T.train(model, scorer, T.toy_set(range(100, 104)), epochs=25, lr=3e-3)
    ex = T.make_example(901, n_files=30, benign_files=40)
    with torch.no_grad():
        want_node = torch.sigmoid(T.sage_node_logits(model, ex["x"], ex["rowptr"], ex["col"], ex["ew"]))
        want_seq = torch.sigmoid(T.lstm_logits(scorer, ex["seq"], ex["lengths"]))
    model.cuda(); scorer.cuda()
    c = lambda k: ex[k].cuda()
    _, score = model(c("x"), c("rowptr"), c("col"), c("ew"))
    probs = scorer(c("seq"), c("lengths"))
    assert float((score.cpu() - want_node).abs().max()) <= 1e-4          # fp32 spec tolerance (north star: 1e-4 rel)
    assert float((probs.cpu() - want_seq).abs().max()) <= 1e-4
    files = ex["is_file"].numpy()
    assert T.roc_auc(score.cpu().numpy()[files], ex["label"].numpy()[files]) >= 0.90
    assert T.roc_auc(probs[:, 0].cpu().numpy(), ex["seq_label"].numpy()) >= 0.90
    # plan from model confidence alone (no labels): exactly the encrypted files are reverted
    g = ex["graph"]
    res = pipeline.run(g, ex["seq"].numpy(), ex["lengths"].numpy(), ex["seq_nodes"], model, scorer, top_a=4096,
                       n_rollouts=1024, depth=40, iterations=8)
    assert sorted(res.plan_nodes) == sorted(np.nonzero(g.meta["label"])[0].tolist())


# ---------------------------------------------------------------- backward kernels (csrc/sage_bwd.cu) vs the oracle
def _grad_close(got, want, what, rtol=2e-4, atol_rms=2e-5):
    """Gradients are sums over up to N rows of fp32 products: same form of bound as the forward tolerance
    (|got-want| <= rtol*|want| + atol_rms*rms(want)), with a factor 2 for the two chained fp32 GEMMs."""
    got = got.detach().double().cpu().numpy(); want = np.asarray(want, np.float64)
    rms = float(np.sqrt((want ** 2).mean())) if want.size else 0.0
    bad = np.abs(got - want) > rtol * np.abs(want) + atol_rms * max(rms, 1e-30)
    assert not bad.any(), f"{what}: {int(bad.sum())}/{bad.size} out of tolerance, max err {np.abs(got - want).max():.3e} (rms {rms:.3e})"


@pytest.mark.parametrize("N,E,L,F,seed", [(3000, 30000, 3, 32, 1), (257, 1500, 2, 64, 2), (1000, 20000, 2, 128, 3),
                                          (33, 20, 1, 32, 4), (5000, 400000, 2, 32, 5)])
def test_backward_kernels_match_the_oracle(N, E, L, F, seed):
    """d(loss)/d(every parameter) and d(loss)/dx from the CUDA path (fused wgmma forward + sage_bwd.cu backward) against
    the hand-written fp64 backward oracle (itself pinned to autograd, tests/test_oracle_sage_bwd.py)."""
    from nerrf_b200 import graph as G
    from nerrf_b200.ai import autograd as AG
    from oracle import sage_bwd_ref as B
    g = G.synthetic_graph(N=N, E=E, seed=seed, f_in=F)
    model = GraphSAGE_T(F, 128, L, seed=seed).cuda()
    rng = np.random.default_rng(seed)
    dlogit = rng.standard_normal(N).astype(np.float32)
    x = torch.from_numpy(g.x).cuda().requires_grad_()
    tg = AG.TrainGraph(torch.from_numpy(g.rowptr).cuda(), torch.from_numpy(g.col).cuda(), torch.from_numpy(g.ew).cuda())
    logit = AG.sage_node_logits(model, x, tg)
    (logit * torch.from_numpy(dlogit).cuda()).sum().backward()
    want = B.model_backward(model.oracle_params(), g.x, g.rowptr, g.col, g.ew, dlogit)
    _grad_close(x.grad, want["x"], "dx")
    _grad_close(model.node_w.grad, want["node_w"], "d node_w"); _grad_close(model.node_b.grad, want["node_b"], "d node_b")
    for l, (dW, db) in enumerate(want["layers"]):
        _grad_close(model.weights[l].grad, dW, f"dW[{l}]"); _grad_close(model.biases[l].grad, db, f"db[{l}]")
    # deterministic: a second backward gives the same bits
    g1 = [p.grad.clone() for p in model.parameters() if p.grad is not None]
    model.zero_grad(); x.grad = None
    (AG.sage_node_logits(model, x, tg) * torch.from_numpy(dlogit).cuda()).sum().backward()
    assert all(torch.equal(a, p.grad) for a, p in zip(g1, [p for p in model.parameters() if p.grad is not None]))


def test_backward_int64_rowptr_and_frozen_input():
    """int64 row pointers; x without requires_grad (first layer: no dZ / dh launches)."""
    from nerrf_b200 import graph as G
    from nerrf_b200.ai import autograd as AG
    from oracle import sage_bwd_ref as B
    g = G.synthetic_graph(N=700, E=9000, seed=8)
    model = GraphSAGE_T(32, 128, 2, seed=8).cuda()
    dlogit = np.random.default_rng(8).standard_normal(700).astype(np.float32)
    tg = AG.TrainGraph(torch.from_numpy(g.rowptr.astype(np.int64)).cuda(), torch.from_numpy(g.col).cuda(), torch.from_numpy(g.ew).cuda())
    (AG.sage_node_logits(model, torch.from_numpy(g.x).cuda(), tg) * torch.from_numpy(dlogit).cuda()).sum().backward()
    want = B.model_backward(model.oracle_params(), g.x, g.rowptr, g.col, g.ew, dlogit)
    for l, (dW, db) in enumerate(want["layers"]):
        _grad_close(model.weights[l].grad, dW, f"dW[{l}]"); _grad_close(model.biases[l].grad, db, f"db[{l}]")


def test_training_on_the_gpu_through_the_library_kernels():
    """ai.train with device='cuda': GraphSAGE-T forward/backward through the C-ABI kernels; the ROADMAP gate (ROC-AUC >=
    0.90 on a held-out toy trace) holds and the trained weights give the same scores through GraphSAGE_T.forward."""
    torch.manual_seed(0)
    model, scorer = GraphSAGE_T(32, 128, 2), LSTMScorer()
    T.train(model, scorer, T.toy_set(range(100, 104)), epochs=25, lr=3e-3, device="cuda")
    ex = T._to(T.make_example(901, n_files=30, benign_files=40), "cuda")
    with torch.no_grad():
        logit_train_path = T.node_logits(model, ex)
    _, score = model(ex["x"], ex["rowptr"], ex["col"], ex["ew"])
    assert float((score - torch.sigmoid(logit_train_path)).abs().max()) <= 1e-5
    files = ex["is_file"].cpu().numpy()
    assert T.roc_auc(score.cpu().numpy()[files], ex["label"].cpu().numpy()[files]) >= 0.90
