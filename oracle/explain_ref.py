"""Per-node edge attributions oracle (float64 torch autograd; test infra -- see oracle/__init__.py).

Statement (DESIGN.md 1.1.1): for target v with logit z_v = h_v^L . w_n + b_n over the plain-torch GraphSAGE-T of
oracle/sage_ref.py, the attribution of CSR edge e is a_e(v) = ew_e * dz_v / dew_e, the derivative taken by autograd with
ew.requires_grad through every layer (one backward per target, on the full graph).  sage_ref normalises by
wsum.clamp_min(1e-12), whose gradient torch defines as [wsum >= 1e-12]: a row whose weights sum to exactly 1e-12 passes
the gradient of its weight sum.  Evidence = the k edges of largest |a_e|, ties to the lower CSR position.

receptive_field restates the extraction rule on the host: every node within distance <= L - 1 of the target (along
in-edges) keeps all its in-edges, in CSR order; distance-L nodes keep none.
"""
import numpy as np
import torch

from . import sage_ref


def logit_and_grad(params, x, rowptr, col, ew, target, dtype=torch.float64):
    """-> (z_v, dz_v / dew [E]) in `dtype`"""
    w = torch.as_tensor(np.asarray(ew)).to(dtype).clone().requires_grad_(True)
    rp = torch.as_tensor(np.asarray(rowptr)).to(torch.int64)
    cl = torch.as_tensor(np.asarray(col)).to(torch.int64)
    h = torch.as_tensor(np.asarray(x)).to(dtype)
    dst = sage_ref.edge_dst(rp)
    for W, b in params["layers"]:
        h = sage_ref.layer(h, rp, cl, w, torch.as_tensor(W), torch.as_tensor(b), relu=True, dst=dst, dtype=dtype)
    z = h[int(target)] @ torch.as_tensor(params["node_w"]).to(dtype) + torch.as_tensor(params["node_b"]).to(dtype)[0]
    (g,) = torch.autograd.grad(z, w, allow_unused=True)
    if g is None:
        g = torch.zeros_like(w)
    return float(z.detach()), g.detach()


def attributions(params, x, rowptr, col, ew, target, dtype=torch.float64):
    """-> (z_v, a [E] = ew * dz_v / dew) as (float, float64 numpy)"""
    z, g = logit_and_grad(params, x, rowptr, col, ew, target, dtype)
    return z, (torch.as_tensor(np.asarray(ew)).to(dtype) * g).numpy()


def top_edges(a, k):
    """the k CSR positions of largest |a|, ties to the lower position"""
    a = np.abs(np.asarray(a, np.float64))
    return np.lexsort((np.arange(a.size), -a))[:k]


def receptive_field(rowptr, col, target, hops):
    """-> (nodes: sorted global ids of the receptive field, dist: their distances, edges: CSR positions of the kept edges in
    the batched order -- rows by ascending node id, each row's edges in CSR order)"""
    rowptr = np.asarray(rowptr, np.int64)
    col = np.asarray(col, np.int64)
    dist = {int(target): 0}
    frontier = [int(target)]
    for d in range(hops):
        nxt = []
        for u in frontier:
            for e in range(rowptr[u], rowptr[u + 1]):
                s = int(col[e])
                if s not in dist:
                    dist[s] = d + 1
                    nxt.append(s)
        frontier = nxt
    nodes = np.array(sorted(dist), np.int64)
    dd = np.array([dist[int(u)] for u in nodes], np.int64)
    edges = [np.arange(rowptr[u], rowptr[u + 1]) for u, du in zip(nodes, dd) if du < hops]
    return nodes, dd, (np.concatenate(edges) if edges else np.zeros(0, np.int64))
