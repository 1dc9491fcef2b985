"""GraphSAGE-T layers as torch.autograd Functions over the C-ABI kernels (SURVEY.md 8f rank 3: training on the GPU).

Reference surface: the GraphSAGE-T half of ai/train.py "joint GNN+LSTM training script" (README.md:75; ROADMAP.md:62-69 --
named, never written).  Forward = the fused tensor-core (wgmma) layer kernel the inference path uses (`nerrf_sage_layer_fwd_ex`),
backward = `nerrf_sage_layer_bwd` (csrc/sage_bwd.cu): dP = dy*[y>0], dW = [h||m]^T dP, db, dZ = dP W^T,
dh = dZ[:, :F] + A^T dZ[:, F:], the last as a gather over the transposed graph.  CUDA tensors only; no CPU fallback
(ai/train.py keeps its plain-torch restatement for CPU runs and as the thing the gradients are checked against).
"""
from __future__ import annotations

import ctypes as C

import torch

from .. import _lib as L


class TrainGraph:
    """A graph prepared for training: CSR by destination (what the forward reads) + its transpose, CSR by source with the
    edge weights pre-normalised by the destination's weight sum (what the backward of the aggregate gathers over).
    Built once per graph with device-wide torch primitives (sort / bincount / cumsum): preparation, not the hot path."""

    def __init__(self, rowptr, col, edge_w):
        L.require_cuda(rowptr, col, edge_w)
        self.rowptr, self.col, self.edge_w = rowptr.contiguous(), col.contiguous(), edge_w.contiguous()
        n = rowptr.numel() - 1
        self.n = n
        deg = (rowptr[1:] - rowptr[:-1]).long()
        dst = torch.repeat_interleave(torch.arange(n, device=rowptr.device), deg)
        wsum = torch.zeros(n, device=rowptr.device, dtype=torch.float32).index_add_(0, dst, edge_w)
        a = edge_w / wsum.clamp_min(1e-12)[dst]
        src = col.long()
        order = torch.sort(src, stable=True).indices
        t_rowptr = torch.zeros(n + 1, device=rowptr.device, dtype=torch.int64)
        t_rowptr[1:] = torch.cumsum(torch.bincount(src, minlength=n), 0)
        self.t_rowptr = t_rowptr.to(rowptr.dtype).contiguous()
        self.t_col = dst[order].to(torch.int32).contiguous()
        self.t_w = a[order].contiguous()
        self._ws = None

    def workspace(self, F: int):
        need = C.c_size_t()
        L.check(L.lib().nerrf_sage_layer_bwd_workspace_bytes(self.n, F, C.byref(need)), "bwd_workspace_bytes")
        if self._ws is None or self._ws.numel() * 4 < need.value:
            self._ws = torch.empty((need.value + 3) // 4, dtype=torch.float32, device=self.rowptr.device)
        return self._ws


def aggregate(h, tg: TrainGraph):
    """m = A h through the standalone K1 kernel (`nerrf_sage_aggregate`)."""
    m = torch.empty_like(h)
    L.check(L.lib().nerrf_sage_aggregate(L.ptr(h), L.ptr(tg.rowptr), int(tg.rowptr.dtype == torch.int64), L.ptr(tg.col),
                                         L.ptr(tg.edge_w), L.ptr(m), tg.n, 0, tg.n, h.shape[1], L.current_stream_ptr()),
            "nerrf_sage_aggregate")
    return m


class SageLayerFn(torch.autograd.Function):
    """y = relu([h || A h] W + b) -- forward on wgmma (fused gather + aggregate + GEMM), backward in csrc/sage_bwd.cu."""

    @staticmethod
    def forward(ctx, h, W, b, tg: TrainGraph, model, l: int):
        h = h.contiguous()
        with torch.no_grad():
            y = model.layer_forward(l, h, tg.rowptr, tg.col, tg.edge_w)
        ctx.save_for_backward(h, W, y)
        ctx.tg = tg
        return y

    @staticmethod
    def backward(ctx, dy):
        h, W, y = ctx.saved_tensors
        tg = ctx.tg
        F = h.shape[1]
        dy = dy.contiguous()
        need_h, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1] or ctx.needs_input_grad[2]
        dh = torch.empty_like(h) if need_h else None
        dW = torch.empty_like(W) if need_w else None
        db = torch.empty(W.shape[1], device=W.device, dtype=torch.float32) if need_w else None
        m = aggregate(h, tg) if need_w else None
        ws = tg.workspace(F)
        with torch.cuda.device(h.device):
            L.check(L.lib().nerrf_sage_layer_bwd(L.ptr(h), L.ptr(m), L.ptr(y), L.ptr(dy), L.ptr(W.detach().contiguous()),
                                                 L.ptr(tg.t_rowptr), int(tg.t_rowptr.dtype == torch.int64), L.ptr(tg.t_col),
                                                 L.ptr(tg.t_w), L.ptr(dh), L.ptr(dW), L.ptr(db), L.ptr(ws), ws.numel() * 4,
                                                 tg.n, F, W.shape[1], 1, L.current_stream_ptr()), "nerrf_sage_layer_bwd")
        return dh, dW, db, None, None, None


def sage_node_logits(model, x, tg: TrainGraph):
    """Node-head logits with gradients: the L fused layers through SageLayerFn, then h . w_n + b_n (a matvec, left to torch).
    sigmoid(logit) is what GraphSAGE_T.forward returns as node_score."""
    model._check_graph(x, tg.rowptr, tg.col, tg.edge_w)
    h = x
    for l, (W, b) in enumerate(zip(model.weights, model.biases)):
        h = SageLayerFn.apply(h, W, b, tg, model, l)
    return h @ model.node_w + model.node_b
