"""Per-node edge attributions without a GPU: the float64 oracle (oracle/explain_ref.py) against two independent
witnesses -- central finite differences and a hand-computed one-layer case -- the receptive-field rule, and the plan
emitter's evidence fields."""
import json

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.csgraph as csg
import torch

from nerrf_b200.ai.planner import emit
from oracle import explain_ref as X, sage_ref


def random_graph(N, E, seed, zero_in=()):
    rng = np.random.default_rng(seed)
    src, dst = rng.integers(0, N, E), rng.integers(0, N, E)
    keep = ~np.isin(dst, list(zero_in))
    src, dst = src[keep], dst[keep]
    w = (0.2 + rng.random(src.size)).astype(np.float64)
    order = np.argsort(dst, kind="stable")
    rowptr = np.zeros(N + 1, np.int64)
    np.cumsum(np.bincount(dst, minlength=N), out=rowptr[1:])
    x = rng.standard_normal((N, 32))
    return rowptr, src[order], w[order], x


def params_f64(layers, seed=3):
    p = sage_ref.make_params(32, 128, layers, seed=seed, edge_head=False)
    return {"layers": [(W.double(), b.double()) for W, b in p["layers"]], "node_w": p["node_w"].double(),
            "node_b": p["node_b"].double()}


@pytest.mark.parametrize("layers", [1, 2, 3])
def test_oracle_matches_central_differences(layers):
    rowptr, col, ew, x = random_graph(24, 90, seed=layers)
    p = params_f64(layers)
    for target in (0, 5, 17):
        z, a = X.attributions(p, x, rowptr, col, ew, target)
        _, g = X.logit_and_grad(p, x, rowptr, col, ew, target)
        g = g.numpy()
        step = 1e-6
        for e in range(0, col.size, 7):
            wp, wm = ew.copy(), ew.copy()
            wp[e] += step; wm[e] -= step
            fd = (X.logit_and_grad(p, x, rowptr, col, wp, target)[0] - X.logit_and_grad(p, x, rowptr, col, wm, target)[0]) / (2 * step)
            assert abs(fd - g[e]) <= 1e-6 * max(1.0, abs(fd)), (layers, target, e, fd, g[e])
        assert np.allclose(a, ew * g, rtol=0, atol=0)


def _hand_one_layer(x, rowptr, col, ew, W, b, w_n, target, eps=1e-12):
    """a_e = ew_e dZ[dst, F:] . (h_src - [S >= eps] m_dst) / max(S, eps), dZ = (w_n * [y > 0]) W^T, written out per edge"""
    N, F = x.shape
    S = np.zeros(N); m = np.zeros((N, F))
    dst = np.repeat(np.arange(N), np.diff(rowptr))
    for e in range(col.size):
        S[dst[e]] += ew[e]; m[dst[e]] += ew[e] * x[col[e]]
    D = np.maximum(S, eps)
    m /= D[:, None]
    y = np.concatenate([x, m], 1) @ W + b
    dP = np.where(y[target] > 0, w_n, 0.0)
    dZ = dP @ W.T
    a = np.zeros(col.size)
    for e in range(col.size):
        if dst[e] == target:
            ind = 1.0 if S[target] >= eps else 0.0
            a[e] = ew[e] * dZ[F:] @ (x[col[e]] - ind * m[target]) / D[target]
    return a


def test_hand_computed_one_layer_three_nodes():
    """node 0: two in-edges (from 1 and 2); node 1: one in-edge whose weight sums to below 1e-12; node 2: no in-edges"""
    rowptr = np.array([0, 2, 3, 3])
    col = np.array([1, 2, 2])
    ew = np.array([0.75, 0.25, 1e-13])
    rng = np.random.default_rng(7)
    x = rng.standard_normal((3, 32))
    p = params_f64(1, seed=11)
    W, b = p["layers"][0][0].numpy(), p["layers"][0][1].numpy()
    w_n = p["node_w"].numpy()
    for target in (0, 1, 2):
        _, a = X.attributions(p, x, rowptr, col, ew, target)
        want = _hand_one_layer(x, rowptr, col, ew, W, b, w_n, target)
        assert np.allclose(a, want, rtol=1e-10, atol=1e-300), (target, a, want)
    # node 2 has no in-edges and nothing of its row exists: every attribution is zero
    assert not X.attributions(p, x, rowptr, col, ew, 2)[1].any()
    # below 1e-12 the normaliser is the constant 1e-12: a_e = ew dZ . h_src / 1e-12, no mean term
    assert X.attributions(p, x, rowptr, col, ew, 1)[1][2] != 0.0


def test_boundary_weight_sum_equal_to_eps_passes_the_gradient():
    """torch's clamp_min(1e-12) has gradient [S >= 1e-12]: at S == 1e-12 exactly the mean term is present"""
    rowptr = np.array([0, 2, 2, 2])
    col = np.array([1, 2])
    ew = np.array([0.5e-12, 0.5e-12])
    assert ew.sum() == 1e-12
    x = np.random.default_rng(2).standard_normal((3, 32))
    p = params_f64(1, seed=5)
    W, b = p["layers"][0][0].numpy(), p["layers"][0][1].numpy()
    _, a = X.attributions(p, x, rowptr, col, ew, 0)
    with_mean = _hand_one_layer(x, rowptr, col, ew, W, b, p["node_w"].numpy(), 0)
    assert np.allclose(a, with_mean, rtol=1e-9, atol=0)
    # (with the indicator taken as [S > 1e-12] the two attributions would be ew dZ.h_src / 1e-12 instead)
    s = torch.tensor([1e-12], dtype=torch.float64, requires_grad=True)
    s.clamp_min(1e-12).sum().backward()
    assert float(s.grad) == 1.0


def _spec_field(rowptr, col, target, hops):
    """the rule stated through graph distances: scipy's unweighted shortest paths from the target along in-edges"""
    N = rowptr.size - 1
    dst = np.repeat(np.arange(N), np.diff(rowptr))
    A = sp.csr_matrix((np.ones(col.size), (dst, col)), shape=(N, N))     # u -> its in-neighbours
    d = csg.shortest_path(A, unweighted=True, indices=[target])[0]
    nodes = np.nonzero(d <= hops)[0]
    edges = np.concatenate([np.arange(rowptr[u], rowptr[u + 1]) for u in nodes if d[u] <= hops - 1] + [np.zeros(0, np.int64)])
    return nodes, d[nodes].astype(np.int64), edges


@pytest.mark.parametrize("hops", [1, 2, 3])
def test_receptive_field_restatement_matches_distances(hops):
    rowptr, col, ew, x = random_graph(60, 150, seed=10 + hops, zero_in=(4, 9))
    for target in (0, 4, 9, 33):
        n1, d1, e1 = X.receptive_field(rowptr, col, target, hops)
        n2, d2, e2 = _spec_field(rowptr, col, target, hops)
        assert np.array_equal(n1, n2) and np.array_equal(d1, d2) and np.array_equal(e1, e2)


@pytest.mark.parametrize("hops", [1, 2])
def test_edges_outside_the_receptive_field_get_exactly_zero(hops):
    rowptr, col, ew, x = random_graph(40, 80, seed=20 + hops)
    p = params_f64(hops)
    for target in range(0, 40, 6):
        _, a = X.attributions(p, x, rowptr, col, ew, target)
        _, _, kept = X.receptive_field(rowptr, col, target, hops)
        outside = np.ones(col.size, bool); outside[kept] = False
        assert not a[outside].any()


def test_top_edges_ties_go_to_the_lower_position():
    a = np.array([0.5, -2.0, 2.0, 0.0, -0.5, 2.0])
    assert X.top_edges(a, 4).tolist() == [1, 2, 5, 0]


# ------------------------------------------------------------------------------------------------ plan emitter
NAMES = ["/data/a.lockbit3", "pid:42", "/data/b.dat", "/data/evil\nrm -rf x.lockbit3", "/data/c.lockbit3"]


def _plan(**kw):
    return emit.undo_plan(NAMES, [1, 0, 4], scores=[0.0, 1.0, 2.0, 3.0], attack_id="t", size_mb=np.ones(5),
                          node_score=np.linspace(0, 1, 5), **kw)


def _ex(node, path="/data/a.dat", other=2):
    return {"node": node, "scope": "subgraph", "logit": 3.5,
            "edges": [{"pos": 7, "src": 1, "dst": node, "attr": 0.25, "event": {"time": 12.5, "pid": 42, "syscall": "write",
                                                                                  "path": path},
                       "src_name": NAMES[1], "dst_name": NAMES[node]},
                      {"pos": 3, "src": other, "dst": 1, "attr": -0.125, "event": None, "src_name": NAMES[other],
                       "dst_name": NAMES[1]}]}


def test_plan_without_evidence_is_unchanged():
    base = emit.to_json(_plan())
    assert emit.to_json(_plan(evidence=None)) == base
    assert emit.to_json(_plan(evidence={})) == base
    assert not any(k.startswith("evidence") for s in json.loads(base)["steps"] for k in s)


def test_evidence_schema():
    ev = {1: _ex(1), 0: _ex(0), 4: {"node": 4, "scope": None, "reason": "over budget"}}
    plan = json.loads(emit.to_json(_plan(evidence=ev)))
    s0, s1, s2 = plan["steps"]
    assert s0["evidence_logit"] == 3.5 and len(s0["evidence"]) == 2
    e = s0["evidence"][0]
    assert set(e) == {"event", "src", "dst", "attribution"}
    assert e["event"] == {"time": 12.5, "pid": 42, "syscall": "write", "path": "/data/a.dat"}
    assert e["src"] == "pid:42" and e["dst"] == "pid:42" and e["attribution"] == 0.25
    assert s0["evidence"][1]["event"] is None
    assert s2["evidence"] is None and s2["evidence_reason"] == "over budget" and "evidence_logit" not in s2
    for s in plan["steps"]:
        assert "hostile_name" not in s


def test_evidence_hosts_and_hostile_paths():
    ex = _ex(0, path="/data/x\n; reboot", other=3)
    ex["edges"][0]["event"]["source"] = 1
    plan = _plan(evidence={0: ex}, host_names=["alpha", "beta"])
    s = plan["steps"][1]
    assert s["hostile_name"] is True
    assert s["evidence"][0]["event"]["host"] == "beta"
    assert s["evidence"][0]["event"]["path"] == "/data/x\n; reboot"          # exact bytes kept, JSON escapes them
    with pytest.raises(ValueError):
        emit.evidence_fields(dict(ex), host_names=["alpha", "../etc"])


def test_to_shell_never_reads_evidence():
    ev = {1: _ex(1, path="/data/$(reboot)\n"), 0: _ex(0), 4: _ex(4, other=3)}
    assert emit.to_shell(_plan(evidence=ev)) == emit.to_shell(_plan())
