"""GraphSAGE-T layers and the BiLSTM scorer as torch.autograd Functions over the C-ABI kernels (SURVEY.md 8f rank 3:
training on the GPU).

Reference surface: the GraphSAGE-T half of ai/train.py "joint GNN+LSTM training script" (README.md:75; ROADMAP.md:62-69 --
named, never written).  Forward = the fused tensor-core (wgmma) layer kernel the inference path uses (`nerrf_sage_layer_fwd_ex`),
backward = `nerrf_sage_layer_bwd` (csrc/sage_bwd.cu): dP = dy*[y>0], dW = [h||m]^T dP, db, dZ = dP W^T,
dh = dZ[:, :F] + A^T dZ[:, F:], the last as a gather over the transposed graph.  The BiLSTM: forward =
`nerrf_lstm_forward_train` (the fp32 CUDA-core recurrence, saving its activations to a tape), backward =
`nerrf_lstm_backward` (csrc/lstm_bwd.cu, backward-through-time).  The attack / normal edge head: forward =
`nerrf_sage_node_head` (proj) + `nerrf_sage_edge_head`, backward = `nerrf_sage_edge_head_bwd` (csrc/sage_edge_bwd.cu: row
sums of dL over the CSR and its transpose, then dh, dWe, dbe).  CUDA tensors only; no CPU fallback (ai/train.py keeps
its plain-torch restatements for CPU runs and as the thing the gradients are checked against).
"""
from __future__ import annotations

import ctypes as C

import torch

from .. import _lib as L


class TrainGraph:
    """A graph prepared for training: CSR by destination (what the forward reads) + its transpose, CSR by source with the
    edge weights pre-normalised by the destination's weight sum (what the backward of the aggregate gathers over).
    Built once per graph with device-wide torch primitives (sort / bincount / cumsum) and `nerrf_sage_norm_weights` for
    the normalised weights (no float atomics, so two constructions of one graph give the same bits): preparation, not
    the hot path."""

    def __init__(self, rowptr, col, edge_w):
        L.require_cuda(rowptr, col, edge_w)
        self.rowptr, self.col, self.edge_w = rowptr.contiguous(), col.contiguous(), edge_w.contiguous()
        n = rowptr.numel() - 1
        self.n = n
        deg = (rowptr[1:] - rowptr[:-1]).long()
        dst = torch.repeat_interleave(torch.arange(n, device=rowptr.device), deg)
        a = torch.empty_like(self.edge_w)
        with torch.cuda.device(rowptr.device):
            L.check(L.lib().nerrf_sage_norm_weights(L.ptr(self.rowptr), int(rowptr.dtype == torch.int64), L.ptr(self.edge_w),
                                                    L.ptr(a), n, L.current_stream_ptr()), "nerrf_sage_norm_weights")
        src = col.long()
        order = torch.sort(src, stable=True).indices
        t_rowptr = torch.zeros(n + 1, device=rowptr.device, dtype=torch.int64)
        t_rowptr[1:] = torch.cumsum(torch.bincount(src, minlength=n), 0)
        self.t_rowptr = t_rowptr.to(rowptr.dtype).contiguous()
        self.t_col = dst[order].to(torch.int32).contiguous()
        self.t_w = a[order].contiguous()
        self.t_eid = order.to(rowptr.dtype).contiguous()         # CSR position of each out-edge (edge head backward)
        self._ws = self._edge_ws = None

    def workspace(self, F: int):
        need = C.c_size_t()
        L.check(L.lib().nerrf_sage_layer_bwd_workspace_bytes(self.n, F, C.byref(need)), "bwd_workspace_bytes")
        if self._ws is None or self._ws.numel() * 4 < need.value:
            self._ws = torch.empty((need.value + 3) // 4, dtype=torch.float32, device=self.rowptr.device)
        return self._ws

    def edge_workspace(self, H: int):
        need = C.c_size_t()
        L.check(L.lib().nerrf_sage_edge_head_bwd_workspace_bytes(self.n, H, C.byref(need)), "edge_head_bwd_workspace_bytes")
        if self._edge_ws is None or self._edge_ws.numel() * 4 < need.value:
            self._edge_ws = torch.empty((need.value + 3) // 4, dtype=torch.float32, device=self.rowptr.device)
        return self._edge_ws


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


class EdgeHeadFn(torch.autograd.Function):
    """edge_logit [E, 2] = [h_src || h_dst] We + be (CSR order) -- forward = `nerrf_sage_node_head` (its proj output) +
    `nerrf_sage_edge_head`, backward = `nerrf_sage_edge_head_bwd` (csrc/sage_edge_bwd.cu)."""

    @staticmethod
    def forward(ctx, h, edge_W, edge_b, tg: TrainGraph, model):
        h = h.contiguous()
        We = edge_W.detach().contiguous()
        n = h.shape[0]
        score = torch.empty(n, device=h.device, dtype=torch.float32)       # the node head's output, not used here
        proj = torch.empty(n, 4, device=h.device, dtype=torch.float32)
        el = torch.empty(tg.col.numel(), 2, device=h.device, dtype=torch.float32)
        with torch.cuda.device(h.device):
            L.check(L.lib().nerrf_sage_node_head(L.ptr(h), L.ptr(model.node_w), 0.0, L.ptr(score), L.ptr(We), L.ptr(proj), 0,
                                                 n, h.shape[1], L.current_stream_ptr()), "nerrf_sage_node_head")
            L.check(L.lib().nerrf_sage_edge_head(L.ptr(proj), L.ptr(tg.rowptr), int(tg.rowptr.dtype == torch.int64),
                                                 L.ptr(tg.col), L.ptr(edge_b.detach().contiguous()), L.ptr(el), 0, n,
                                                 L.current_stream_ptr()), "nerrf_sage_edge_head")
        ctx.save_for_backward(h, We)
        ctx.tg = tg
        return el

    @staticmethod
    def backward(ctx, dlogit):
        h, We = ctx.saved_tensors
        tg = ctx.tg
        dlogit = dlogit.contiguous()
        need_w = ctx.needs_input_grad[1] or ctx.needs_input_grad[2]
        dh = torch.empty_like(h) if ctx.needs_input_grad[0] else None
        dW = torch.empty_like(We) if need_w else None
        db = torch.empty(2, device=h.device, dtype=torch.float32) if need_w else None
        ws = tg.edge_workspace(h.shape[1]) if need_w else None
        with torch.cuda.device(h.device):
            L.check(L.lib().nerrf_sage_edge_head_bwd(L.ptr(h), L.ptr(We), L.ptr(dlogit), L.ptr(tg.rowptr),
                                                     int(tg.rowptr.dtype == torch.int64), L.ptr(tg.t_rowptr), L.ptr(tg.t_eid),
                                                     int(tg.t_rowptr.dtype == torch.int64), L.ptr(dh), L.ptr(dW), L.ptr(db),
                                                     L.ptr(ws), 0 if ws is None else ws.numel() * 4, tg.n, h.shape[1],
                                                     L.current_stream_ptr()), "nerrf_sage_edge_head_bwd")
        return dh, dW, db, None, None


def sage_logits(model, x, tg: TrainGraph):
    """(node logits [N], edge logits [E, 2]) with gradients: the fused layers through SageLayerFn, the node head as in
    sage_node_logits, the edge head through EdgeHeadFn.  Both heads read the final h, so autograd adds their
    contributions to dh before the last layer's backward."""
    if model.edge_W is None:
        raise ValueError("the model has no edge head (GraphSAGE_T(edge_head=False))")
    model._check_graph(x, tg.rowptr, tg.col, tg.edge_w)
    h = x
    for l, (W, b) in enumerate(zip(model.weights, model.biases)):
        h = SageLayerFn.apply(h, W, b, tg, model, l)
    return h @ model.node_w + model.node_b, EdgeHeadFn.apply(h, model.edge_W, model.edge_b, tg, model)


# ---------------------------------------------------------------------------------------------------- BiLSTM scorer
_LSTM_PARAM_NAMES = ("weight_ih", "weight_hh", "bias_ih", "bias_hh")


def lstm_params(scorer):
    """The flat parameter list LSTMFn takes: per layer l, per direction (forward, reverse), w_ih, w_hh, b_ih, b_hh."""
    return [getattr(scorer.lstm, f"{n}_l{l}{sfx}") for l in range(scorer.num_layers) for sfx in ("", "_reverse")
            for n in _LSTM_PARAM_NAMES]


class LSTMTape:
    """The activation tape and backward workspace of one scorer, grown when a larger shape arrives (like
    TrainGraph.workspace).  A tape holds one forward until its backward has run: the backward overwrites the saved gates
    with their gradients, and a second forward before that backward gets a tape of its own."""

    def __init__(self):
        self._tape = self._ws = None
        self._busy = False

    def buffers(self, B, T, D_in, H, num_layers, device, hold):
        tb, wb = C.c_size_t(), C.c_size_t()
        L.check(L.lib().nerrf_lstm_train_workspace_bytes(B, T, D_in, H, num_layers, C.byref(tb), C.byref(wb)),
                "nerrf_lstm_train_workspace_bytes")
        if self._busy:
            tape = torch.empty(tb.value, dtype=torch.uint8, device=device)
            return tape, None
        if self._tape is None or self._tape.numel() < tb.value or self._tape.device != device:
            self._tape = torch.empty(tb.value, dtype=torch.uint8, device=device)
        self._busy = hold
        return self._tape, (self if hold else None)

    def workspace(self, bytes_, device):
        if self._ws is None or self._ws.numel() < bytes_ or self._ws.device != device:
            self._ws = torch.empty(bytes_, dtype=torch.uint8, device=device)
        return self._ws

    def release(self):
        self._busy = False


class LSTMFn(torch.autograd.Function):
    """hfin [B, 2H] = [h_fwd_final || h_bwd_final] of the top layer of a BiLSTM (torch.nn.LSTM semantics on packed
    sequences).  Forward on `nerrf_lstm_forward_train`, backward on `nerrf_lstm_backward`; the gradient of b_ih and of
    b_hh is the same db.  Differentiable once per forward (the backward consumes the tape)."""

    @staticmethod
    def forward(ctx, seq, lengths, cache: LSTMTape, num_layers: int, will_backward: bool, *params):
        seq = seq.contiguous()
        B, T, D_in = seq.shape
        H = params[1].shape[1]
        ln = lengths.to(device=seq.device, dtype=torch.int32).contiguous()
        W_ih = [params[4 * i].detach().contiguous() for i in range(2 * num_layers)]
        W_hh = [params[4 * i + 1].detach().contiguous() for i in range(2 * num_layers)]
        wih_t = [w.t().contiguous() for w in W_ih]
        whh_t = [w.t().contiguous() for w in W_hh]
        bias = [(params[4 * i + 2].detach() + params[4 * i + 3].detach()).contiguous() for i in range(2 * num_layers)]
        hfin = torch.empty(B, 2 * H, device=seq.device, dtype=torch.float32)
        tape, owner = cache.buffers(B, T, D_in, H, num_layers, seq.device, will_backward)
        L.check(L.lib().nerrf_lstm_forward_train(L.ptr(seq), L.ptr(ln), B, T, D_in, H, num_layers, L.ptr_array(wih_t),
                                                 L.ptr_array(whh_t), L.ptr_array(bias), L.ptr(hfin), L.ptr(tape),
                                                 tape.numel(), L.current_stream_ptr()), "nerrf_lstm_forward_train")
        ctx.save_for_backward(seq, ln, tape, *W_ih, *W_hh)
        ctx.cache, ctx.owner, ctx.num_layers, ctx.done = cache, owner, num_layers, False
        return hfin

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dhfin):
        if ctx.done:
            raise RuntimeError("LSTMFn: the tape of this forward was already differentiated (it is consumed by backward)")
        ctx.done = True
        nl = ctx.num_layers
        saved = ctx.saved_tensors
        seq, ln, tape = saved[0], saved[1], saved[2]
        W_ih, W_hh = saved[3:3 + 2 * nl], saved[3 + 2 * nl:]
        B, T, D_in = seq.shape
        H = W_hh[0].shape[1]
        dhfin = dhfin.contiguous()
        dseq = torch.empty_like(seq) if ctx.needs_input_grad[0] else None
        dW_ih = [torch.empty_like(w) for w in W_ih]
        dW_hh = [torch.empty_like(w) for w in W_hh]
        db = [torch.empty(4 * H, device=seq.device, dtype=torch.float32) for _ in range(2 * nl)]
        tb, wb = C.c_size_t(), C.c_size_t()
        L.check(L.lib().nerrf_lstm_train_workspace_bytes(B, T, D_in, H, nl, C.byref(tb), C.byref(wb)),
                "nerrf_lstm_train_workspace_bytes")
        ws = ctx.cache.workspace(wb.value, seq.device)
        try:
            with torch.cuda.device(seq.device):
                L.check(L.lib().nerrf_lstm_backward(L.ptr(seq), L.ptr(ln), B, T, D_in, H, nl, L.ptr_array(W_ih),
                                                    L.ptr_array(W_hh), L.ptr(tape), tape.numel(), L.ptr(dhfin),
                                                    L.ptr(dseq), L.ptr_array(dW_ih), L.ptr_array(dW_hh), L.ptr_array(db),
                                                    L.ptr(ws), ws.numel(), L.current_stream_ptr()), "nerrf_lstm_backward")
        finally:
            if ctx.owner is not None:
                ctx.owner.release()
        grads = []
        for i in range(2 * nl):
            grads += [dW_ih[i], dW_hh[i], db[i], db[i]]
        return (dseq, None, None, None, None, *grads)


def lstm_logits(scorer, seq, lengths):
    """Head logits [B, 2] of the BiLSTM scorer with gradients for every LSTMScorer parameter (and seq, if it requires
    grad): the recurrence through LSTMFn, then the head (a [2H] -> 2 linear map, left to torch).  sigmoid(logits) is what
    LSTMScorer.forward returns.  CUDA tensors only."""
    L.require_cuda(seq, lengths)
    if seq.dtype != torch.float32 or seq.dim() != 3 or seq.shape[2] != scorer.in_dim:
        raise ValueError(f"seq must be float32 [B,T,{scorer.in_dim}]")
    if lengths.numel() != seq.shape[0]:
        raise ValueError("lengths must have B entries")
    cache = getattr(scorer, "_train_tape", None)
    if cache is None:
        cache = scorer._train_tape = LSTMTape()
    params = lstm_params(scorer)
    will_backward = torch.is_grad_enabled() and (seq.requires_grad or any(p.requires_grad for p in params))
    hfin = LSTMFn.apply(seq, lengths, cache, scorer.num_layers, will_backward, *params)
    return scorer.head(hfin)
