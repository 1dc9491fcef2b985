"""ai.models.GraphSAGE_T -- temporal GraphSAGE anomaly scorer (CUDA, sm_90a).

Reference surface: ai/models/GraphSAGE-T.py `GraphSAGE_T.forward` (README.md:73; ROADMAP.md:67,127
-- named, never written).  Behaviour: docs/content/docs/architecture.mdx:49-53,157 (edge
normal/attack classes, node anomaly_score in [0,1]); threat-model.mdx:176-189.  Frozen spec:
SURVEY.md 8a rows a1-a3 / DESIGN.md.

    h'_v = ReLU([h_v || m_v] @ W_l + b_l),  m_v = sum_e w_e h_src(e) / max(sum_e w_e, 1e-12)
    node_score = sigmoid(h . w_n + b_n);  edge_logit = [h_src || h_dst] @ W_e + b_e

Parameters are ordinary torch tensors (state_dict works); compute goes through the C-ABI
library (include/nerrf_b200.h).  CUDA tensors only -- there is no CPU fallback.
"""
from __future__ import annotations

import math

import torch
from torch import nn

from ... import _lib as L

ALGOS = {"auto": 0, "ffma": 1, "umma": 2, "umma2": 3}


class GraphSAGE_T(nn.Module):
    def __init__(self, in_dim: int = 32, hidden: int = 128, num_layers: int = 3, edge_head: bool = True,
                 algo: str = "auto", seed: int | None = 1):
        super().__init__()
        if hidden != 128:
            raise ValueError("hidden must be 128 (kernel tile width)")
        if in_dim not in (32, 64, 128):
            raise ValueError("in_dim must be 32, 64 or 128 (pad the node features)")
        self.in_dim, self.hidden, self.num_layers, self.algo = in_dim, hidden, num_layers, algo
        # L2 eviction-priority hints of the tensor-core layer (NERRF_SAGE_FLAG_NO_L2_POLICY when off); no result bit
        # depends on it
        self.l2_policy = True
        g = torch.Generator().manual_seed(seed) if seed is not None else None

        def xavier(fi, fo):
            a = math.sqrt(6.0 / (fi + fo))
            return (torch.rand(fi, fo, generator=g) * 2 - 1) * a

        self.weights = nn.ParameterList()
        self.biases = nn.ParameterList()
        F = in_dim
        for _ in range(num_layers):
            self.weights.append(nn.Parameter(xavier(2 * F, hidden)))
            self.biases.append(nn.Parameter((torch.rand(hidden, generator=g) * 2 - 1) * 0.1))
            F = hidden
        self.node_w = nn.Parameter(xavier(hidden, 1)[:, 0].contiguous())
        self.node_b = nn.Parameter((torch.rand(1, generator=g) * 2 - 1) * 0.1)
        if edge_head:
            self.edge_W = nn.Parameter(xavier(2 * hidden, 2))
            self.edge_b = nn.Parameter((torch.rand(2, generator=g) * 2 - 1) * 0.1)
        else:
            self.edge_W = self.edge_b = None
        self._node_b_cache = (None, 0.0)

    # -- helpers ------------------------------------------------------------------------
    def _algo_flags(self) -> int:
        return ALGOS[self.algo] | (0 if self.l2_policy else 0x200)

    def oracle_params(self):
        """The same weights in the dict layout oracle/sage_ref.py takes (tests only use this)."""
        p = {"layers": [(w.detach().cpu(), b.detach().cpu()) for w, b in zip(self.weights, self.biases)],
             "node_w": self.node_w.detach().cpu(), "node_b": self.node_b.detach().cpu()}
        if self.edge_W is not None:
            p["edge_W"] = self.edge_W.detach().cpu(); p["edge_b"] = self.edge_b.detach().cpu()
        return p

    def load_oracle_params(self, p):
        with torch.no_grad():
            for i, (w, b) in enumerate(p["layers"]):
                self.weights[i].copy_(w); self.biases[i].copy_(b)
            self.node_w.copy_(p["node_w"]); self.node_b.copy_(p["node_b"])
            if self.edge_W is not None and "edge_W" in p:
                self.edge_W.copy_(p["edge_W"]); self.edge_b.copy_(p["edge_b"])
        return self

    def _node_b_host(self) -> float:
        ver = self.node_b._version
        if self._node_b_cache[0] != (ver, self.node_b.data_ptr()):
            self._node_b_cache = ((ver, self.node_b.data_ptr()), float(self.node_b.detach().cpu()))
        return self._node_b_cache[1]

    def _check_graph(self, x, rowptr, col, edge_w):
        L.require_cuda(x, rowptr, col, edge_w)
        # raw pointers cross the C-ABI: a model left on the CPU or on another GPU would be a sticky illegal-address fault
        if self.weights[0].device != x.device:
            raise L.NerrfError(f"model parameters are on {self.weights[0].device}, inputs on {x.device}: call model.to(x.device)")
        for t in (rowptr, col, edge_w):
            if t.device != x.device:
                raise L.NerrfError(f"graph tensors must share one device (got {t.device} and {x.device})")
        if x.dtype != torch.float32 or edge_w.dtype != torch.float32:
            raise TypeError("x and edge_w must be float32")
        if col.dtype != torch.int32:
            raise TypeError("col must be int32")
        if rowptr.dtype not in (torch.int32, torch.int64):
            raise TypeError("rowptr must be int32 or int64")
        if rowptr.numel() != x.shape[0] + 1:
            raise ValueError("rowptr must have N+1 entries")
        for t in (x, rowptr, col, edge_w):
            if not t.is_contiguous():
                raise ValueError("graph tensors must be contiguous")

    # -- single layer (used by the sharded forward) ---------------------------------------
    def layer_forward(self, l: int, h, rowptr, col, edge_w, out=None, row_begin=0, row_end=None, relu=True, score_out=None,
                      edge_base: int = 0, reuse_long_scan: bool = False, peer_outs=None, multicast_ptr: int = 0,
                      peer_need=None):
        """One fused layer.  score_out (fp32 [N]) fuses the node head into the layer's epilogue.
        edge_base: `col` / `edge_w` hold only the edge block [edge_base, edge_base + len) of the graph (a
        1-D shard); rowptr keeps absolute edge offsets, so the pointers are shifted instead of the data.
        reuse_long_scan: the previous layer_forward call on this model used the SAME graph and row range, so
        the hub-row scan held in the scratch is still valid (layers 2..L of one forward).
        peer_outs: list of peer-mapped [N, H] tensors (other ranks' `out` buffers): the epilogue also stores
        the produced rows there (fused per-layer exchange of the sharded forward, nerrf_b200.dist).
        peer_need: uint8 [N], bit i set <=> peer_outs[i]'s rank reads that row as a source (send only those)."""
        self._check_graph(h, rowptr, col, edge_w)
        N = h.shape[0]
        row_end = N if row_end is None else row_end
        if out is None:
            out = torch.empty(N, self.hidden, device=h.device, dtype=torch.float32)
        W, b = self.weights[l], self.biases[l]
        if edge_base:
            import ctypes as C
            colp = C.c_void_p(col.data_ptr() - 4 * edge_base); ewp = C.c_void_p(edge_w.data_ptr() - 4 * edge_base)
        else:
            colp, ewp = L.ptr(col), L.ptr(edge_w)
        lws, lws_bytes = self._long_rows_ws(col.numel(), h.device) if self._has_hub_rows(rowptr) else (None, 0)
        algo_flags = self._algo_flags() | (0x100 if reuse_long_scan else 0)
        if multicast_ptr:                       # NVSwitch multicast address of `out` on every rank (nerrf_b200.dist)
            import ctypes as C
            pp = (C.c_void_p * 1)(multicast_ptr); npeers = -1
        elif peer_outs:
            pp, npeers = L.ptr_array(peer_outs), len(peer_outs)
        else:
            pp, npeers = None, 0
        with torch.cuda.device(h.device):
            L.check(L.lib().nerrf_sage_layer_fwd_ex(
                L.ptr(h), L.ptr(rowptr), int(rowptr.dtype == torch.int64), colp, ewp, L.ptr(W), L.ptr(b), L.ptr(out), N,
                row_begin, row_end, h.shape[1], self.hidden, int(relu), algo_flags,
                L.ptr(self.node_w) if score_out is not None else None, self._node_b_host() if score_out is not None else 0.0,
                L.ptr(score_out), L.ptr(lws), lws_bytes, pp, npeers, L.ptr(peer_need), L.current_stream_ptr()),
                "nerrf_sage_layer_fwd_ex")
        return out

    def _has_hub_rows(self, rowptr) -> bool:
        """Graph metadata (max in-degree > 128: the kernel's long-row threshold), computed once per rowptr tensor (one device sync) and cached.
        A stale cache entry can only cost speed, never correctness: without the scratch hub rows are
        processed inline, with it the pre-pass simply finds nothing."""
        key = (rowptr.data_ptr(), rowptr.numel(), rowptr._version)
        if getattr(self, "_hub_key", None) != key:
            self._hub_key = key
            self._hub_val = bool((rowptr[1:] - rowptr[:-1]).max() > 128) if rowptr.numel() > 1 else False
        return self._hub_val

    def _long_rows_ws(self, n_edges, device):
        """Device scratch for the hub-row pre-aggregation (include/nerrf_b200.h); cached, grows with E."""
        import ctypes as C
        need = C.c_size_t()
        L.check(L.lib().nerrf_sage_long_rows_workspace_bytes(int(n_edges), C.byref(need)), "long_rows_workspace_bytes")
        ws = getattr(self, "_lws", None)
        if ws is None or ws.numel() < need.value or ws.device != device:
            ws = torch.empty(need.value, dtype=torch.uint8, device=device)
            self._lws = ws
        return ws, need.value

    def heads(self, h, rowptr, col, return_edge_logits=False, row_begin=0, row_end=None):
        N = h.shape[0]
        row_end = N if row_end is None else row_end
        score = torch.empty(N, device=h.device, dtype=torch.float32)
        want_edges = return_edge_logits and self.edge_W is not None
        proj = torch.empty(N, 4, device=h.device, dtype=torch.float32) if want_edges else None
        L.check(L.lib().nerrf_sage_node_head(L.ptr(h), L.ptr(self.node_w), self._node_b_host(), L.ptr(score),
                                             L.ptr(self.edge_W) if want_edges else None, L.ptr(proj), row_begin, row_end,
                                             self.hidden, L.current_stream_ptr()), "nerrf_sage_node_head")
        if not want_edges:
            return score, None
        el = torch.empty(col.numel(), 2, device=h.device, dtype=torch.float32)
        L.check(L.lib().nerrf_sage_edge_head(L.ptr(proj), L.ptr(rowptr), int(rowptr.dtype == torch.int64), L.ptr(col),
                                             L.ptr(self.edge_b), L.ptr(el), row_begin, row_end,
                                             L.current_stream_ptr()), "nerrf_sage_edge_head")
        return score, el

    # -- the reference-named entry point ------------------------------------------------------
    @torch.no_grad()
    def forward(self, x, rowptr, col, edge_w, return_edge_logits: bool = False):
        """x fp32 [N,F_in]; CSR-by-destination rowptr [N+1], col int32 [E], edge_w fp32 [E].
        Returns (h [N,H], node_score [N]) or (h, node_score, edge_logit [E,2])."""
        self._check_graph(x, rowptr, col, edge_w)
        if x.shape[1] != self.in_dim:
            raise ValueError(f"x has {x.shape[1]} features, model expects {self.in_dim}")
        N = x.shape[0]
        dev = x.device
        h = torch.empty(N, self.hidden, device=dev, dtype=torch.float32)
        score = torch.empty(N, device=dev, dtype=torch.float32)
        lbytes = self._long_rows_ws(col.numel(), dev)[1] if self._has_hub_rows(rowptr) else 0
        pp = ((N * self.hidden * 4 + 255) // 256) * 256 if self.num_layers > 1 else 0
        ws = torch.empty(pp + lbytes, device=dev, dtype=torch.uint8)
        Wp = L.ptr_array(list(self.weights)); bp = L.ptr_array(list(self.biases))
        with torch.cuda.device(dev):
            L.check(L.lib().nerrf_sage_forward(L.ptr(x), L.ptr(rowptr), int(rowptr.dtype == torch.int64), L.ptr(col),
                                               L.ptr(edge_w), N, self.in_dim, self.hidden, self.num_layers, Wp, bp,
                                               L.ptr(self.node_w), self._node_b_host(), L.ptr(h), L.ptr(score), L.ptr(ws),
                                               ws.numel(), self._algo_flags(),
                                               L.current_stream_ptr()), "nerrf_sage_forward")
        if return_edge_logits and self.edge_W is not None:
            _, el = self.heads(h, rowptr, col, return_edge_logits=True)
            return h, score, el
        return h, score


class HostSession:
    """HOST-buffer path (the e2e call of bench.py): pinned host arrays in, node scores out, all
    copies inside the C-ABI call `nerrf_sage_session_forward_host`."""

    def __init__(self, model: GraphSAGE_T, max_nodes: int, max_edges: int):
        import ctypes as C
        self.model = model
        self._h = C.c_void_p()
        self._inflight = {}
        L.check(L.lib().nerrf_sage_session_create(max_nodes, max_edges, model.in_dim, model.hidden, model.num_layers,
                                                  C.byref(self._h)), "nerrf_sage_session_create")
        Ws = [w.detach().cpu().contiguous() for w in model.weights]
        bs = [b.detach().cpu().contiguous() for b in model.biases]
        nw = model.node_w.detach().cpu().contiguous()
        L.check(L.lib().nerrf_sage_session_set_weights(self._h, L.ptr_array(Ws), L.ptr_array(bs), L.ptr(nw),
                                                       float(model.node_b.detach().cpu())), "set_weights")

    def forward(self, x, rowptr, col, edge_w, score_out, h_out=None):
        """All arguments are CPU (ideally pinned) torch tensors; score_out/h_out are written in place."""
        for t in (x, rowptr, col, edge_w, score_out):
            if t.is_cuda:
                raise L.NerrfError("HostSession takes host tensors")
        if rowptr.dtype != torch.int32:
            raise TypeError("host session uses int32 rowptr")
        algo = self.model._algo_flags()
        L.check(L.lib().nerrf_sage_session_forward_host(self._h, L.ptr(x), L.ptr(rowptr), L.ptr(col), L.ptr(edge_w),
                                                        x.shape[0], col.numel(), L.ptr(score_out), L.ptr(h_out), algo),
                "nerrf_sage_session_forward_host")
        return score_out

    def submit(self, x, rowptr, col, edge_w, score_out, h_out=None) -> int:
        """Pipelined form (`nerrf_sage_session_submit_host`): queue the step and return a ticket at once; up to two
        steps are in flight, the upload of one overlapping the layers of the other.  The host tensors must stay alive and
        unmodified until `wait(ticket)` returns -- the session keeps references to them until then."""
        import ctypes as C
        for t in (x, rowptr, col, edge_w, score_out):
            if t.is_cuda:
                raise L.NerrfError("HostSession takes host tensors")
        if rowptr.dtype != torch.int32:
            raise TypeError("host session uses int32 rowptr")
        ticket = C.c_uint64(0)
        L.check(L.lib().nerrf_sage_session_submit_host(self._h, L.ptr(x), L.ptr(rowptr), L.ptr(col), L.ptr(edge_w),
                                                       x.shape[0], col.numel(), L.ptr(score_out), L.ptr(h_out),
                                                       self.model._algo_flags(), C.byref(ticket)),
                "nerrf_sage_session_submit_host")
        self._inflight[ticket.value] = (x, rowptr, col, edge_w, score_out, h_out)
        return ticket.value

    def wait(self, ticket: int):
        """Block until the outputs of `ticket` are in its host tensors; returns its score tensor."""
        L.check(L.lib().nerrf_sage_session_wait(self._h, int(ticket)), "nerrf_sage_session_wait")
        held = self._inflight.pop(int(ticket), None)
        for t in [k for k in self._inflight if k < int(ticket) - 1]:      # older tickets completed when their slot was reused
            self._inflight.pop(t, None)
        return held[4] if held else None

    def close(self):
        if self._h:
            L.lib().nerrf_sage_session_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
