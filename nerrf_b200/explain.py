"""Per-node explanations of GraphSAGE-T scores: which events of the window drove a node's logit (DESIGN.md 1.1.1).

For a target node v with logit z_v = h_v^L . w_n + b_n (sigmoid(z_v) is node_score), the attribution of CSR edge e is

    a_e(v) = ew_e * dz_v / dew_e          (gradient x input; ew is shared by the L layers, so the derivative sums over them)

and v's evidence is the k edges of largest |a_e(v)|, ties to the lower CSR position, each mapped to the event that made it.
Every target is explained on its own: its L-hop in-neighbourhood is extracted (nerrf_explain_subgraph_count / _fill),
the batch of neighbourhoods runs the fused layer forward (GraphSAGE_T.layer_forward) and one backward seeded with
dh^L = w_n on the target rows (nerrf_sage_layer_bwd_ex, which accumulates d_ew), and nerrf_explain_topk picks the edges.
Neighbourhoods are disjoint blocks of one batched graph, so one target's gradient never reaches another's edges.
A target whose neighbourhood holds more than max_edges_per_target edges is explained the same way on the whole graph
(at most max_full_graph_targets of them per call); past that cap it gets no evidence and a reason.  CUDA tensors only.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib as L
from .ai.autograd import TrainGraph

DEFAULT_MAX_EDGES = 1 << 15
DEFAULT_MAX_FULL_GRAPH = 4


def _edge_event(g, dev):
    ev = g.meta.get("edge_event")
    if callable(ev):
        ev = ev()
    if ev is None:
        return None
    return torch.as_tensor(ev).to(device=dev, dtype=torch.int64).contiguous()


def subgraphs(rowptr, col, ew, x, targets, hops: int, max_edges: int = DEFAULT_MAX_EDGES):
    """The batched receptive fields of `targets` (int64 node ids) -> dict with "fit" (bool [B]: the target's block is in
    the batch), "counts" ([B, 2] int64 nodes / edges, -1 over budget), and for the fitting targets, in order: rowptr (int64),
    col, ew, epos (CSR position in the input graph), node (global id of each batched node), x, target (batched node id),
    seg (int64 [fit + 1] edge offsets of the blocks)."""
    dev = rowptr.device
    t = torch.as_tensor(np.asarray(targets, np.int64)).to(dev).to(torch.int32).contiguous()
    B = int(t.numel())
    is64 = int(rowptr.dtype == torch.int64)
    need = C.c_size_t()
    L.check(L.lib().nerrf_explain_subgraph_workspace_bytes(B, int(max_edges), C.byref(need)), "nerrf_explain_subgraph_workspace_bytes")
    ws = torch.empty(max(need.value, 16), dtype=torch.uint8, device=dev)
    counts = torch.empty(2 * max(B, 1), dtype=torch.int64, device=dev)
    n = rowptr.numel() - 1
    with torch.cuda.device(dev):
        L.check(L.lib().nerrf_explain_subgraph_count(L.ptr(rowptr), is64, L.ptr(col), n, L.ptr(t), B, hops, int(max_edges),
                                                     L.ptr(counts), L.ptr(ws), ws.numel(), L.current_stream_ptr()),
                "nerrf_explain_subgraph_count")
    cnt = counts[:2 * B].view(B, 2).cpu().numpy()
    fit = cnt[:, 0] >= 0
    out = {"fit": fit, "counts": cnt}
    tf = t[torch.from_numpy(np.nonzero(fit)[0]).to(dev)].contiguous()
    nf = int(tf.numel())
    nodes_c, edges_c = cnt[fit, 0], cnt[fit, 1]
    node_off = np.concatenate([[0], np.cumsum(nodes_c)]).astype(np.int64)
    edge_off = np.concatenate([[0], np.cumsum(edges_c)]).astype(np.int64)
    NB, EB = int(node_off[-1]), int(edge_off[-1])
    if NB >= 2 ** 31:
        raise L.NerrfError("explain: the batched receptive fields hold %d nodes (at most 2^31 - 1)" % NB)
    F_in = x.shape[1]
    b_rowptr = torch.zeros(NB + 1, dtype=torch.int64, device=dev)
    b_col = torch.empty(EB, dtype=torch.int32, device=dev)
    b_ew = torch.empty(EB, dtype=torch.float32, device=dev)
    b_epos = torch.empty(EB, dtype=torch.int64, device=dev)
    b_node = torch.empty(NB, dtype=torch.int32, device=dev)
    b_x = torch.empty(NB, F_in, dtype=torch.float32, device=dev)
    b_t = torch.empty(nf, dtype=torch.int32, device=dev)
    if nf:
        d_no = torch.from_numpy(node_off[:-1].copy()).to(dev)
        d_eo = torch.from_numpy(edge_off[:-1].copy()).to(dev)
        with torch.cuda.device(dev):
            L.check(L.lib().nerrf_explain_subgraph_fill(L.ptr(rowptr), is64, L.ptr(col), L.ptr(ew), L.ptr(x), F_in, n, L.ptr(tf), nf,
                                                        hops, int(max_edges), L.ptr(d_no), L.ptr(d_eo), L.ptr(b_rowptr),
                                                        L.ptr(b_col), L.ptr(b_ew), L.ptr(b_epos), L.ptr(b_node), L.ptr(b_x),
                                                        L.ptr(b_t), L.ptr(ws), ws.numel(), L.current_stream_ptr()),
                    "nerrf_explain_subgraph_fill")
    out.update(rowptr=b_rowptr, col=b_col, ew=b_ew, epos=b_epos, node=b_node, x=b_x, target=b_t,
               seg=torch.from_numpy(edge_off).to(dev))
    return out


def forward_saved(model, x, rowptr, col, ew):
    """The fused layers of `model` over one graph, keeping every layer's input: -> [x, h^1, ..., h^L]"""
    hs = [x]
    for l in range(model.num_layers):
        hs.append(model.layer_forward(l, hs[-1], rowptr, col, ew))
    return hs


def edge_weight_grad(model, hs, rowptr, col, ew, seeds):
    """d_ew [E] = sum over the seeds of dz / dew (the layer backwards of nerrf_sage_layer_bwd_ex), seeded with
    dh^L = w_n on the rows `seeds` (int64 CUDA tensor) and 0 elsewhere."""
    dev = rowptr.device
    tg = TrainGraph(rowptr, col, ew)
    n = tg.n
    dy = torch.zeros(n, model.hidden, dtype=torch.float32, device=dev)
    dy[seeds] = model.node_w.detach().to(torch.float32)
    d_ew = torch.zeros(col.numel(), dtype=torch.float32, device=dev)
    is64 = int(rowptr.dtype == torch.int64)
    for l in reversed(range(model.num_layers)):
        h, y = hs[l], hs[l + 1]
        F = h.shape[1]
        dh = torch.empty_like(h) if l > 0 else None
        ws = tg.workspace(F)
        W = model.weights[l].detach().contiguous()
        with torch.cuda.device(dev):
            L.check(L.lib().nerrf_sage_layer_bwd_ex(L.ptr(h), None, L.ptr(y), L.ptr(dy), L.ptr(W), L.ptr(tg.t_rowptr),
                                                    int(tg.t_rowptr.dtype == torch.int64), L.ptr(tg.t_col), L.ptr(tg.t_w),
                                                    L.ptr(dh), None, None, L.ptr(ws), ws.numel() * 4, n, F, model.hidden, 1,
                                                    L.ptr(rowptr), is64, L.ptr(col), L.ptr(ew), L.ptr(d_ew),
                                                    L.current_stream_ptr()), "nerrf_sage_layer_bwd_ex")
        dy = dh
    return d_ew


def topk(seg, ew, d_ew, epos, edge_event, k: int):
    """-> (edge [S, k], attr [S, k], pos [S, k], event [S, k]) CUDA tensors (nerrf_explain_topk)"""
    dev = seg.device
    S = int(seg.numel()) - 1
    oe = torch.empty(S, k, dtype=torch.int64, device=dev)
    oa = torch.empty(S, k, dtype=torch.float32, device=dev)
    op = torch.empty(S, k, dtype=torch.int64, device=dev)
    ov = torch.empty(S, k, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        L.check(L.lib().nerrf_explain_topk(L.ptr(seg), S, L.ptr(ew), L.ptr(d_ew), L.ptr(epos), L.ptr(edge_event), k, L.ptr(oe),
                                           L.ptr(oa), L.ptr(op), L.ptr(ov), L.current_stream_ptr()), "nerrf_explain_topk")
    return oe, oa, op, ov


def _results(targets, scope, logits, attr, pos, event, rowptr, col):
    """host records of one batch: per target {node, scope, logit, edges: [{pos, src, dst, attr, event}]}"""
    p = pos.clamp_min(0)
    src = col.long()[p]
    dst = torch.searchsorted(rowptr.long(), p, right=True) - 1
    logits, attr, pos, event = (a.cpu().numpy() for a in (logits, attr, pos, event))
    src, dst = src.cpu().numpy(), dst.cpu().numpy()
    out = []
    for i, v in enumerate(targets):
        keep = pos[i] >= 0
        edges = [{"pos": int(pos[i, j]), "src": int(src[i, j]), "dst": int(dst[i, j]), "attr": float(attr[i, j]),
                  "event": int(event[i, j])} for j in np.nonzero(keep)[0]]
        out.append({"node": int(v), "scope": scope, "logit": float(logits[i]), "edges": edges})
    return out


def explain_nodes(g, model, nodes, k: int = 8, max_edges_per_target: int = DEFAULT_MAX_EDGES,
                  max_full_graph_targets: int = DEFAULT_MAX_FULL_GRAPH) -> list:
    """Evidence for each node of `nodes` (ids into g): a list, in the order of `nodes`, of
        {"node", "scope": "subgraph" | "full_graph", "logit": z_v, "edges": [{"pos": CSR position, "src", "dst",
         "attr": a_e, "event": event index (g.meta["edge_event"]), -1 without a map}]}   (at most k edges, |attr| descending)
    or {"node", "scope": None, "reason": ...} for a target past the full-graph cap.  g.x, g.rowptr, g.col, g.ew must be
    CUDA tensors (no CPU fallback)."""
    x, rowptr, col, ew = g.x, g.rowptr, g.col, g.ew
    if not all(torch.is_tensor(a) for a in (x, rowptr, col, ew)):
        raise L.NerrfError("explain_nodes takes a graph of CUDA tensors (no CPU fallback)")
    model._check_graph(x, rowptr, col, ew)
    if x.shape[1] != model.in_dim:
        raise ValueError(f"x has {x.shape[1]} features, model expects {model.in_dim}")
    if not 1 <= int(k) <= 1024:
        raise ValueError("k must lie in 1..1024")
    nodes = np.asarray(nodes, np.int64).reshape(-1)
    n = rowptr.numel() - 1
    if nodes.size and (nodes.min() < 0 or nodes.max() >= n):
        raise ValueError("explain_nodes: node ids must lie in [0, %d)" % n)
    dev = x.device
    ev = _edge_event(g, dev)
    res = [None] * nodes.size
    if nodes.size == 0:
        return res
    sg = subgraphs(rowptr, col, ew, x, nodes, model.num_layers, max_edges_per_target)
    fit = np.nonzero(sg["fit"])[0]
    if fit.size:
        hs = forward_saved(model, sg["x"], sg["rowptr"], sg["col"], sg["ew"])
        tl = sg["target"].long()
        logits = hs[-1][tl] @ model.node_w.detach() + model.node_b.detach()
        d_ew = edge_weight_grad(model, hs, sg["rowptr"], sg["col"], sg["ew"], tl)
        _, oa, op, ov = topk(sg["seg"], sg["ew"], d_ew, sg["epos"], ev, int(k))
        for i, r in zip(fit, _results(nodes[fit], "subgraph", logits, oa, op, ov, rowptr, col)):
            res[i] = r
    over = np.nonzero(~sg["fit"])[0]
    for j, i in enumerate(over):
        if j >= max_full_graph_targets:
            res[i] = {"node": int(nodes[i]), "scope": None,
                      "reason": "receptive field over %d edges and %d full-graph explanations already in this call"
                                % (max_edges_per_target, max_full_graph_targets)}
            continue
        hs = forward_saved(model, x, rowptr, col, ew)
        seed = torch.tensor([int(nodes[i])], dtype=torch.int64, device=dev)
        logits = hs[-1][seed] @ model.node_w.detach() + model.node_b.detach()
        d_ew = edge_weight_grad(model, hs, rowptr, col, ew, seed)
        seg = torch.tensor([0, col.numel()], dtype=torch.int64, device=dev)
        _, oa, op, ov = topk(seg, ew, d_ew, None, ev, int(k))
        res[i] = _results(nodes[i:i + 1], "full_graph", logits, oa, op, ov, rowptr, col)[0]
    return res


def attach_events(g, explained: list) -> list:
    """Resolve each evidence edge's event through g.meta["event_info"] (event index -> {time, pid, syscall, path[, source]})
    and its two endpoints through g.meta["names"]: -> the same list with "event" replaced by the record (None without one)
    and "src_name" / "dst_name" added."""
    info = g.meta.get("event_info")
    names = g.meta.get("names")
    ids = sorted({e["event"] for r in explained if r and r.get("edges") for e in r["edges"] if e["event"] >= 0})
    rec = dict(zip(ids, info(np.asarray(ids, np.int64)))) if (info is not None and ids) else {}
    nid = sorted({v for r in explained if r and r.get("edges") for e in r["edges"] for v in (e["src"], e["dst"])})
    nm = dict(zip(nid, names.take(nid) if hasattr(names, "take") else [names[i] for i in nid])) if names is not None else {}
    out = []
    for r in explained:
        if r is None or not r.get("edges"):
            out.append(r)
            continue
        r = dict(r)
        r["edges"] = [dict(e, event=rec.get(e["event"]), src_name=nm.get(e["src"]), dst_name=nm.get(e["dst"])) for e in r["edges"]]
        out.append(r)
    return out
