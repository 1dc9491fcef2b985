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

The BiLSTM half of a file reversion's confidence is explained the same way over the file's event sequence (DESIGN.md
1.2.1, explain_sequences): a_t = x_t . dz/dx_t for the encrypt logit z, through nerrf_lstm_forward_train,
nerrf_lstm_input_grad and nerrf_lstm_explain_steps, each step mapped to the event that made it.
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


def lstm_forward_tape(seq_model, weights, seq, ln):
    """nerrf_lstm_forward_train (the fp32 CUDA-core forward) over one batch: -> (hfin fp32 [B, 2H], tape) CUDA tensors.
    weights = _seq_weights(seq_model, device)."""
    wih_t, whh_t, bias = weights[:3]
    B, T, D = seq.shape
    H, nl = seq_model.hidden, seq_model.num_layers
    tb, wb = C.c_size_t(), C.c_size_t()
    L.check(L.lib().nerrf_lstm_train_workspace_bytes(B, T, D, H, nl, C.byref(tb), C.byref(wb)), "nerrf_lstm_train_workspace_bytes")
    tape = torch.empty(max(tb.value, 16), dtype=torch.uint8, device=seq.device)
    hfin = torch.empty(B, 2 * H, dtype=torch.float32, device=seq.device)
    with torch.cuda.device(seq.device):
        L.check(L.lib().nerrf_lstm_forward_train(L.ptr(seq), L.ptr(ln), B, T, D, H, nl, L.ptr_array(wih_t), L.ptr_array(whh_t),
                                                 L.ptr_array(bias), L.ptr(hfin), L.ptr(tape), tape.numel(),
                                                 L.current_stream_ptr()), "nerrf_lstm_forward_train")
    return hfin, tape


def lstm_input_grad(seq_model, weights, seq, ln, tape):
    """dseq fp32 [B, T, D] = dz/dseq of the encrypt logit z = head_W[0] . hfin + head_b[0]: nerrf_lstm_input_grad over
    the tape of lstm_forward_tape (which it consumes), seeded with dhfin = head_W[0] on every row."""
    W_ih, W_hh, hw = weights[3:]
    B, T, D = seq.shape
    H, nl = seq_model.hidden, seq_model.num_layers
    gb = C.c_size_t()
    L.check(L.lib().nerrf_lstm_input_grad_workspace_bytes(B, T, D, H, nl, C.byref(gb)), "nerrf_lstm_input_grad_workspace_bytes")
    ws = torch.empty(max(gb.value, 16), dtype=torch.uint8, device=seq.device)
    dseq = torch.empty_like(seq)
    dhfin = hw[0].expand(B, 2 * H).contiguous()
    with torch.cuda.device(seq.device):
        L.check(L.lib().nerrf_lstm_input_grad(L.ptr(seq), L.ptr(ln), B, T, D, H, nl, L.ptr_array(W_ih), L.ptr_array(W_hh),
                                              L.ptr(tape), tape.numel(), L.ptr(dhfin), L.ptr(dseq), L.ptr(ws), ws.numel(),
                                              L.current_stream_ptr()), "nerrf_lstm_input_grad")
    return dseq


def lstm_input_grad_chunk(seq_model, weights, seq, ln):
    """One batch of the encrypt-logit gradient: -> (hfin fp32 [B, 2H], dseq fp32 [B, T, D]) CUDA tensors."""
    hfin, tape = lstm_forward_tape(seq_model, weights, seq, ln)
    return hfin, lstm_input_grad(seq_model, weights, seq, ln, tape)


def explain_steps(seq, dseq, ln, step_event, k: int):
    """-> (step int32 [B, k], attr fp32, feature int32, event int64) CUDA tensors (nerrf_lstm_explain_steps)"""
    B, T, D = seq.shape
    dev = seq.device
    os_ = torch.empty(B, k, dtype=torch.int32, device=dev)
    oa = torch.empty(B, k, dtype=torch.float32, device=dev)
    of = torch.empty(B, k, dtype=torch.int32, device=dev)
    ov = torch.empty(B, k, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        L.check(L.lib().nerrf_lstm_explain_steps(L.ptr(seq), L.ptr(dseq), L.ptr(ln), B, T, D, L.ptr(step_event), k, L.ptr(os_),
                                                 L.ptr(oa), L.ptr(of), L.ptr(ov), L.current_stream_ptr()), "nerrf_lstm_explain_steps")
    return os_, oa, of, ov


def _seq_weights(seq_model, dev):
    """the forward's pre-transposed weights and the backward's torch-layout ones, and head_W, on `dev`"""
    from .ai.autograd import lstm_params
    wih_t, whh_t, bias, hw, _ = seq_model._pack(dev)
    params = lstm_params(seq_model)
    nl2 = 2 * seq_model.num_layers
    W_ih = [params[4 * i].detach().to(device=dev, dtype=torch.float32).contiguous() for i in range(nl2)]
    W_hh = [params[4 * i + 1].detach().to(device=dev, dtype=torch.float32).contiguous() for i in range(nl2)]
    return wih_t, whh_t, bias, W_ih, W_hh, hw


def explain_sequences(seq_model, seq, lengths, k: int = 8, step_event=None, max_batch: int = 512) -> list:
    """Evidence for the encrypt logit z = head_W[0] . hfin + head_b[0] of each sequence (DESIGN.md 1.2.1):
        a_t = sum_d x[t,d] * dz/dx[t,d]   over the valid steps t < len
    -> a list, in sequence order, of {"logit": z, "steps": [{"t", "attr": a_t, "feature": dominant feature index (-1 when
    every term is 0), "event": step_event[b, t] (-1 without a map)}]} (at most k steps, |attr| descending, ties to the
    lower t).  seq fp32 [B, T, D_in] and lengths [B] (numpy or torch; moved to the model's device, which must be CUDA);
    step_event int64 [B, T] or None.  z is evaluated in float64 over the fp32 CUDA-core forward's hfin.  The sequences
    run max_batch at a time; every kernel on this path treats sequences independently, so the result does not depend on
    max_batch."""
    dev = seq_model.head.weight.device
    if dev.type != "cuda":
        raise L.NerrfError("explain_sequences needs a CUDA model (no CPU fallback)")
    if not 1 <= int(k) <= 1024:
        raise ValueError("k must lie in 1..1024")
    if int(max_batch) < 1:
        raise ValueError("max_batch must be >= 1")
    seq = torch.as_tensor(seq).to(device=dev)
    if seq.dtype != torch.float32 or seq.dim() != 3 or seq.shape[2] != seq_model.in_dim:
        raise ValueError(f"seq must be float32 [B,T,{seq_model.in_dim}]")
    seq = seq.contiguous()
    B, T, _ = seq.shape
    ln = torch.as_tensor(lengths).to(device=dev, dtype=torch.int32).contiguous()
    if ln.numel() != B:
        raise ValueError("lengths must have B entries")
    ev = None
    if step_event is not None:
        ev = torch.as_tensor(step_event).to(device=dev, dtype=torch.int64).contiguous()
        if tuple(ev.shape) != (B, T):
            raise ValueError("step_event must be int64 [B, T]")
    out = []
    if B == 0:
        return out
    weights = _seq_weights(seq_model, dev)
    w0 = seq_model.head.weight.detach()[0].double().cpu().numpy()
    b0 = float(seq_model.head.bias.detach()[0].double())
    for s in range(0, B, int(max_batch)):
        e = min(s + int(max_batch), B)
        sq, lc = seq[s:e], ln[s:e]
        hfin, dseq = lstm_input_grad_chunk(seq_model, weights, sq, lc)
        st, at, ft, vt = explain_steps(sq, dseq, lc, None if ev is None else ev[s:e], int(k))
        z = (hfin.double().cpu().numpy() * w0).sum(1) + b0          # per row, a fixed order: independent of the chunking
        st, at, ft, vt = (a.cpu().numpy() for a in (st, at, ft, vt))
        for i in range(e - s):
            keep = np.nonzero(st[i] >= 0)[0]
            out.append({"logit": float(z[i]),
                        "steps": [{"t": int(st[i, j]), "attr": float(at[i, j]), "feature": int(ft[i, j]), "event": int(vt[i, j])}
                                  for j in keep]})
    return out


def attach_events(g, explained: list, sequences: list | None = None):
    """Resolve each evidence edge's event through g.meta["event_info"] (event index -> {time, pid, syscall, path[, source]})
    and its two endpoints through g.meta["names"]: -> the same list with "event" replaced by the record (None without one)
    and "src_name" / "dst_name" added.  sequences: explain_sequences results, resolved in the same single event_info call
    (over the union of the ids of both kinds of evidence); then -> (explained, sequences), each step's "event" replaced by
    its record."""
    info = g.meta.get("event_info")
    names = g.meta.get("names")
    ids = {e["event"] for r in explained if r and r.get("edges") for e in r["edges"] if e["event"] >= 0}
    ids |= {s["event"] for r in (sequences or []) if r and r.get("steps") for s in r["steps"] if s["event"] >= 0}
    ids = sorted(ids)
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
    if sequences is None:
        return out
    seq_out = []
    for r in sequences:
        if r is not None and r.get("steps"):
            r = dict(r, steps=[dict(s, event=rec.get(s["event"])) for s in r["steps"]])
        seq_out.append(r)
    return out, seq_out
