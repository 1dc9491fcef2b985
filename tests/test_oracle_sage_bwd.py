"""The hand-written GraphSAGE-T backward oracle (oracle/sage_bwd_ref.py) against torch.autograd over the forward oracle
(oracle/sage_ref.py): two independent witnesses of the gradients the CUDA backward kernels are checked against."""
import numpy as np
import torch

from nerrf_b200.graph import synthetic_graph
from oracle import sage_bwd_ref as B, sage_ref as S


def _autograd(P, g, dlogit):
    t = torch.from_numpy
    leaves = {"x": t(g.x).double().requires_grad_()}
    params = {"layers": [(W.double().requires_grad_(), b.double().requires_grad_()) for W, b in P["layers"]],
              "node_w": P["node_w"].double().requires_grad_(), "node_b": P["node_b"].double().requires_grad_()}
    h, _ = S.forward(params, leaves["x"], t(g.rowptr), t(g.col), t(g.ew), dtype=torch.float64)
    logit = h @ params["node_w"] + params["node_b"]
    (logit * t(dlogit)).sum().backward()
    return params, leaves


def test_backward_oracle_equals_autograd():
    for (N, E, L, seed) in [(300, 2500, 3, 3), (64, 40, 2, 4), (500, 9000, 1, 5)]:
        g = synthetic_graph(N=N, E=E, seed=seed)
        P = S.make_params(32, 128, L, seed=seed)
        dlogit = np.random.default_rng(seed).standard_normal(N)
        got = B.model_backward(P, g.x, g.rowptr, g.col, g.ew, dlogit)
        params, leaves = _autograd(P, g, dlogit)
        close = lambda a, b: np.allclose(a, b.numpy(), rtol=1e-9, atol=1e-11 * max(1.0, float(np.abs(b.numpy()).max())))
        assert close(got["x"], leaves["x"].grad)
        assert close(got["node_w"], params["node_w"].grad) and close(got["node_b"], params["node_b"].grad)
        for (dW, db), (W, b) in zip(got["layers"], params["layers"]):
            assert close(dW, W.grad) and close(db, b.grad)


def test_transposed_graph_is_the_same_operator():
    """A^T as a gather over transpose_graph == A^T as a scatter over the original edges; isolated nodes, hub rows."""
    g = synthetic_graph(N=400, E=6000, seed=11)
    t_rowptr, t_col, t_w = B.transpose_graph(g.rowptr, g.col, g.ew)
    assert t_rowptr[-1] == g.col.size and np.all(np.diff(t_rowptr) >= 0)
    v = np.random.default_rng(0).standard_normal((400, 8))
    scatter = np.zeros_like(v)
    np.add.at(scatter, g.col.astype(np.int64), B.norm_weights(g.rowptr, g.ew)[:, None] * v[B.edge_dst(g.rowptr)])
    gather = np.zeros_like(v)
    for u in range(400):
        e = slice(t_rowptr[u], t_rowptr[u + 1])
        gather[u] = (t_w[e, None] * v[t_col[e]]).sum(0)
    assert np.allclose(gather, scatter, rtol=1e-12, atol=1e-12)
    # forward operator: rows of A sum to 1 where a node has in-edges
    a = B.norm_weights(g.rowptr, g.ew)
    rs = np.zeros(400); np.add.at(rs, B.edge_dst(g.rowptr), a)
    deg = np.diff(g.rowptr)
    assert np.allclose(rs[deg > 0], 1.0) and np.all(rs[deg == 0] == 0)


def test_hand_computed_layer_backward():
    # 3 nodes, edges 0->1 (w 1), 2->1 (w 3), 1->2 (w 2); F=1, H=1, W = [[2],[4]], b = 0.5, all pre-activations positive
    rowptr = np.array([0, 0, 2, 3]); col = np.array([0, 2, 1]); ew = np.array([1.0, 3.0, 2.0])
    h = np.array([[1.0], [2.0], [3.0]]); W = np.array([[2.0], [4.0]]); b = np.array([0.5])
    y, m = B.layer_forward(h, rowptr, col, ew, W, b)
    assert np.allclose(m[:, 0], [0.0, (1 * 1 + 3 * 3) / 4, 2.0]) and np.allclose(y[:, 0], [2.5, 14.5, 14.5])
    dy = np.array([[1.0], [10.0], [100.0]])
    dh, dW, db = B.layer_backward(h, m, y, dy, W, rowptr, col, ew)
    # dZ = dy * [2, 4]; dh_u = 2 dy_u + sum over out-edges a_e * 4 dy_dst
    assert np.allclose(dh[:, 0], [2 * 1 + 0.25 * 40, 2 * 10 + 1.0 * 400, 2 * 100 + 0.75 * 40])
    assert np.allclose(dW[:, 0], [1 * 1 + 2 * 10 + 3 * 100, 0 + 2.5 * 10 + 2 * 100]) and np.allclose(db, [111.0])


def _pin_graphs():
    """(name, rowptr, col, ew, x): the small graphs above, a hub-destination graph, and degenerate_graph with and without
    edges (isolated nodes, self-loops, multi-edges, a row of weights summing below 1e-12, a row of zero weights)."""
    for (N, E, seed, hub) in [(300, 2500, 3, "src"), (64, 40, 4, "src"), (500, 9000, 5, "src"), (400, 6000, 6, "dst")]:
        g = synthetic_graph(N=N, E=E, seed=seed, hub=hub)
        yield f"synthetic-{N}-{hub}", g.rowptr, g.col, g.ew, g.x
    for (N, E, seed) in [(200, 1500, 7), (50, 0, 8)]:
        rowptr, col, ew = B.degenerate_graph(N, E, seed)
        yield f"degenerate-{N}-{E}", rowptr, col, ew, np.random.default_rng(seed).standard_normal((N, 32)).astype(np.float32)


def _rel(got, want, what, rtol=1e-12):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = float(np.abs(want).max()) if want.size else 0.0
    assert got.shape == want.shape, what
    assert want.size == 0 or float(np.abs(got - want).max()) <= rtol * max(scale, 1e-300), what


def test_degenerate_graph_has_the_rows_it_promises():
    rowptr, col, ew = B.degenerate_graph(200, 1500, 7)
    dst = B.edge_dst(rowptr)
    deg_in, deg_out = np.diff(rowptr), np.bincount(col, minlength=200)
    iso = np.arange(200) % 7 == 3
    assert np.all(deg_in[iso] == 0) and np.all(deg_out[iso] == 0)
    assert np.any(col == dst)                                                     # self-loops
    pairs = col.astype(np.int64) * 200 + dst
    assert np.unique(pairs).size < pairs.size                                     # multi-edges
    assert 0 < ew[dst == 1].sum(dtype=np.float64) < 1e-12 and np.all(ew[dst == 2] == 0) and deg_in[2] > 0


def test_sparse_oracle_equals_the_edge_by_edge_oracle():
    """sparse=True (scipy CSR products) and the np.add.at path compute the same statements: 1e-12 relative."""
    from edge_head_ref import edge_head_backward, model_backward_with_edges
    P = S.make_params(32, 128, 2, seed=9)
    for name, rowptr, col, ew, x in _pin_graphs():
        N, E = rowptr.size - 1, col.size
        rng = np.random.default_rng(N + E)
        h = np.maximum(rng.standard_normal((N, 32)), 0)
        _rel(B.aggregate(h, rowptr, col, ew, sparse=True), B.aggregate(h, rowptr, col, ew), f"{name} m")
        dlogit, dedge = rng.standard_normal(N), rng.standard_normal((E, 2))
        want = B.model_backward(P, x, rowptr, col, ew, dlogit)
        got = B.model_backward(P, x, rowptr, col, ew, dlogit, sparse=True)
        for k in ("x", "node_w", "node_b"):
            _rel(got[k], want[k], f"{name} {k}")
        for l, ((dW, db), (wW, wb)) in enumerate(zip(got["layers"], want["layers"])):
            _rel(dW, wW, f"{name} dW[{l}]"); _rel(db, wb, f"{name} db[{l}]")
        hh = rng.standard_normal((N, 128))
        for a, b, k in zip(edge_head_backward(hh, P["edge_W"], dedge, rowptr, col, sparse=True),
                           edge_head_backward(hh, P["edge_W"], dedge, rowptr, col), ("dh", "dWe", "dbe")):
            _rel(a, b, f"{name} edge head {k}")
        want = model_backward_with_edges(P, x, rowptr, col, ew, dlogit, dedge)
        got = model_backward_with_edges(P, x, rowptr, col, ew, dlogit, dedge, sparse=True)
        for k in ("x", "node_w", "node_b", "edge_W", "edge_b"):
            _rel(got[k], want[k], f"{name} both heads {k}")
        for l, ((dW, db), (wW, wb)) in enumerate(zip(got["layers"], want["layers"])):
            _rel(dW, wW, f"{name} both heads dW[{l}]"); _rel(db, wb, f"{name} both heads db[{l}]")
        if E == 0:                                   # no edges: the aggregate is zero and dh is the self half of dZ
            assert np.all(B.aggregate(h, rowptr, col, ew, sparse=True) == 0)
