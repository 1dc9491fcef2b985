"""GraphSAGE-T BACKWARD oracle (numpy, float64 by default; test infra -- see oracle/__init__.py).

Reference surface: the GraphSAGE-T half of ``ai/train.py`` "joint GNN+LSTM training script" (README.md:75;
ROADMAP.md:62-69 -- named, never written).  The forward spec is oracle/sage_ref.py (frozen, SURVEY.md 8a rows a1-a3):

    m = A h,  A[v,u] = sum_{e: u->v} w_e / max(sum_{e: ->v} w_e, 1e-12)        (CSR by destination)
    y = relu([h || m] W + b)

The backward written out by hand (the chain rule, one statement per kernel of nerrf_b200/csrc/sage_bwd.cu):

    dP = dy * [y > 0]
    db = sum_v dP[v]            dW = [h || m]^T dP
    dZ = dP W^T                 dh = dZ[:, :F] + A^T dZ[:, F:]

tests/test_oracle_sage_bwd.py pins every function here against torch.autograd over oracle/sage_ref.py (a second,
independent witness: autograd differentiates the index_add_ / addmm graph, this file never builds one).

sparse=True computes the same statements with A as a scipy.sparse CSR matrix (m = A @ h, A^T dZ = A.T @ dZ) instead of
np.add.at over [E, F] arrays: what makes 10^5-10^6-node graphs checkable.  The test file pins the two paths together.
"""
import numpy as np
import scipy.sparse as sp


def edge_dst(rowptr):
    rowptr = np.asarray(rowptr, np.int64)
    return np.repeat(np.arange(rowptr.size - 1, dtype=np.int64), np.diff(rowptr))


def degenerate_graph(N, E, seed=0):
    """A CSR-by-destination graph with the rows the kernels must survive: isolated nodes (every id = 3 mod 7), self-loops,
    multi-edges, a row whose weights sum to below 1e-12 but not to zero (node 1) and a row whose weights are all zero
    (node 2); E = 0 gives an edgeless graph.  N >= 8.  -> (rowptr int32 [N+1], col int32, ew float32)."""
    if E == 0:
        return np.zeros(N + 1, np.int32), np.zeros(0, np.int32), np.zeros(0, np.float32)
    rng = np.random.default_rng(seed)
    ids = np.arange(N, dtype=np.int64)
    live = ids[ids % 7 != 3]
    src, dst = rng.choice(live, E), rng.choice(live, E)
    loop = rng.random(E) < 0.05
    src[loop] = dst[loop]
    dup = rng.integers(0, E, E // 10)
    src, dst = np.concatenate([src, src[dup]]), np.concatenate([dst, dst[dup]])
    w = (0.5 + 0.5 * rng.random(src.size)).astype(np.float32)
    keep = (dst != 1) & (dst != 2)
    src = np.concatenate([src[keep], rng.choice(live, 5), [1], rng.choice(live, 4)])
    dst = np.concatenate([dst[keep], np.full(6, 1), np.full(4, 2)])
    w = np.concatenate([w[keep], np.full(6, 1e-14, np.float32), np.zeros(4, np.float32)])
    order = np.argsort(dst, kind="stable")
    rowptr = np.zeros(N + 1, np.int32)
    np.cumsum(np.bincount(dst, minlength=N), out=rowptr[1:])
    return rowptr, src[order].astype(np.int32), w[order]


def norm_weights(rowptr, ew, dtype=np.float64):
    """a_e = w_e / max(weight sum of the edge's destination, 1e-12)  -- the entries of A, edge by edge."""
    dst = edge_dst(rowptr)
    w = np.asarray(ew, dtype)
    wsum = np.zeros(np.asarray(rowptr).size - 1, dtype)
    np.add.at(wsum, dst, w)
    return w / np.maximum(wsum, 1e-12)[dst]


def transpose_graph(rowptr, col, ew, dtype=np.float64):
    """CSR by SOURCE of the same edges: (t_rowptr [N+1], t_col [E] = destinations, t_w [E] = normalised weights a_e).
    Stable in the original edge order, i.e. the out-edges of a source keep (destination, time) order."""
    n = np.asarray(rowptr).size - 1
    src = np.asarray(col, np.int64)
    order = np.argsort(src, kind="stable")
    t_rowptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(src, minlength=n), out=t_rowptr[1:])
    return t_rowptr, edge_dst(rowptr)[order].astype(np.int32), norm_weights(rowptr, ew, dtype)[order]


def adjacency(rowptr, col, ew, dtype=np.float64):
    """A as an [N, N] scipy.sparse CSR matrix (row = destination, column = source; multi-edges are summed by products)."""
    n = np.asarray(rowptr).size - 1
    return sp.csr_matrix((norm_weights(rowptr, ew, dtype), np.asarray(col, np.int64), np.asarray(rowptr, np.int64)),
                         shape=(n, n))


def aggregate(h, rowptr, col, ew, dtype=np.float64, sparse=False):
    if sparse:
        return np.asarray(adjacency(rowptr, col, ew, dtype) @ np.asarray(h, dtype))
    a = norm_weights(rowptr, ew, dtype)
    m = np.zeros((np.asarray(rowptr).size - 1, h.shape[1]), dtype)
    np.add.at(m, edge_dst(rowptr), a[:, None] * np.asarray(h, dtype)[np.asarray(col, np.int64)])
    return m


def layer_forward(h, rowptr, col, ew, W, b, relu=True, dtype=np.float64, sparse=False):
    h = np.asarray(h, dtype)
    m = aggregate(h, rowptr, col, ew, dtype, sparse)
    y = np.concatenate([h, m], 1) @ np.asarray(W, dtype) + np.asarray(b, dtype)
    return (np.maximum(y, 0) if relu else y), m


def layer_backward(h, m, y, dy, W, rowptr, col, ew, relu=True, dtype=np.float64, sparse=False):
    """-> (dh, dW, db) of one layer."""
    h, m, y, dy, W = (np.asarray(a, dtype) for a in (h, m, y, dy, W))
    F = h.shape[1]
    dP = dy * (y > 0) if relu else dy
    db = dP.sum(0)
    dW = np.concatenate([h, m], 1).T @ dP
    dZ = dP @ W.T
    if sparse:
        return dZ[:, :F] + adjacency(rowptr, col, ew, dtype).T @ dZ[:, F:], dW, db
    dh = dZ[:, :F].copy()
    a = norm_weights(rowptr, ew, dtype)
    np.add.at(dh, np.asarray(col, np.int64), a[:, None] * dZ[edge_dst(rowptr), F:])     # A^T applied edge by edge
    return dh, dW, db


def model_backward(params, x, rowptr, col, ew, dlogit, dtype=np.float64, sparse=False):
    """Gradients of  sum_v dlogit[v] * (h_L[v] . node_w + node_b)  w.r.t. every parameter and x.
    params as oracle/sage_ref.py (numpy arrays or torch tensors).  -> dict(layers=[(dW, db)...], node_w, node_b, x)."""
    A = lambda t: np.asarray(t.detach().numpy() if hasattr(t, "detach") else t, dtype)
    layers = [(A(W), A(b)) for W, b in params["layers"]]
    hs, ms = [A(x)], []
    for W, b in layers:
        y, m = layer_forward(hs[-1], rowptr, col, ew, W, b, True, dtype, sparse)
        hs.append(y); ms.append(m)
    dlogit = A(dlogit)
    out = {"node_w": hs[-1].T @ dlogit, "node_b": dlogit.sum(keepdims=True), "layers": [None] * len(layers)}
    dy = dlogit[:, None] * A(params["node_w"])[None, :]
    for l in reversed(range(len(layers))):
        dy, dW, db = layer_backward(hs[l], ms[l], hs[l + 1], dy, layers[l][0], rowptr, col, ew, True, dtype, sparse)
        out["layers"][l] = (dW, db)
    out["x"] = dy
    return out
