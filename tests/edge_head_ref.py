"""Edge head backward written out by hand (numpy, float64): the statement nerrf_sage_edge_head_bwd
(csrc/sage_edge_bwd.cu) is checked against, itself pinned to torch.autograd over oracle/sage_ref.py in
tests/test_edge_head_cpu.py.

    forward   logit[e] = [h_src(e) || h_dst(e)] We + be          (edges in CSR-by-destination order)
    backward  g_src[v] = sum_{e: src(e)=v} dL[e],   g_dst[v] = sum_{e: dst(e)=v} dL[e]
              dh = g_src We[:H]^T + g_dst We[H:]^T,   dWe = [h^T g_src ; h^T g_dst],   dbe = sum_e dL[e]
sparse=True: g_src / g_dst as products of [N, E] incidence matrices with dL, and the layers through the sparse path of
oracle/sage_bwd_ref.py (10^5-10^6-node graphs).
"""
import numpy as np
import scipy.sparse as sp

from oracle import sage_bwd_ref as B


def _np(t, dtype=np.float64):
    return np.asarray(t.detach().cpu().numpy() if hasattr(t, "detach") else t, dtype)


def edge_head_backward(h, We, dL, rowptr, col, dtype=np.float64, sparse=False):
    """-> (dh [N,H], dWe [2H,2], dbe [2]) of sum(dL * edge_logit)."""
    h, We, dL = _np(h, dtype), _np(We, dtype), _np(dL, dtype).reshape(-1, 2)
    n, H = h.shape
    src = np.asarray(col, np.int64)
    if sparse:
        E = src.size
        ones, eid = np.ones(E, dtype), np.arange(E, dtype=np.int64)
        g_src = sp.csr_matrix((ones, (src, eid)), shape=(n, E)) @ dL
        g_dst = sp.csr_matrix((ones, eid, np.asarray(rowptr, np.int64)), shape=(n, E)) @ dL
    else:
        dst = B.edge_dst(rowptr)
        g_src = np.zeros((n, 2), dtype); np.add.at(g_src, src, dL)
        g_dst = np.zeros((n, 2), dtype); np.add.at(g_dst, dst, dL)
    dh = g_src @ We[:H].T + g_dst @ We[H:].T
    dWe = np.concatenate([h.T @ g_src, h.T @ g_dst], 0)
    return dh, dWe, g_dst.sum(0)


def model_backward_with_edges(params, x, rowptr, col, ew, dlogit, dedge, dtype=np.float64, sparse=False, acts=None):
    """Gradients of  sum_v dlogit[v] (h_L[v] . node_w + node_b) + sum_e dedge[e] . edge_logit[e]  w.r.t. every parameter
    and x (both heads read h_L: their input gradients add).  acts: the L layer outputs to evaluate the backward at (e.g.
    a device forward's, so the ReLU masks are that forward's); default the forward in `dtype`.
    -> dict(layers=[(dW, db)...], node_w, node_b, edge_W, edge_b, x)."""
    layers = [(_np(W, dtype), _np(b, dtype)) for W, b in params["layers"]]
    hs, ms = [_np(x, dtype)], []
    for l, (W, b) in enumerate(layers):
        y, m = B.layer_forward(hs[-1], rowptr, col, ew, W, b, True, dtype, sparse)
        hs.append(y if acts is None else _np(acts[l], dtype)); ms.append(m)
    dlogit = _np(dlogit, dtype)
    dh_e, dWe, dbe = edge_head_backward(hs[-1], params["edge_W"], dedge, rowptr, col, dtype, sparse)
    out = {"node_w": hs[-1].T @ dlogit, "node_b": dlogit.sum(keepdims=True), "edge_W": dWe, "edge_b": dbe,
           "layers": [None] * len(layers)}
    dy = dlogit[:, None] * _np(params["node_w"], dtype)[None, :] + dh_e
    for l in reversed(range(len(layers))):
        dy, dW, db = B.layer_backward(hs[l], ms[l], hs[l + 1], dy, layers[l][0], rowptr, col, ew, True, dtype, sparse)
        out["layers"][l] = (dW, db)
    out["x"] = dy
    return out
