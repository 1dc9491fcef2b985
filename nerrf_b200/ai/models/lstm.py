"""ai.models.lstm -- BiLSTM per-file event-sequence scorer (CUDA, sm_90a).

Reference surface: ai/models/lstm.py `forward` (README.md:73 -- named, never written).
Behaviour: "Bidirectional LSTM (256 hidden, 2 layers)", "last 100 events per file"
(docs/content/docs/architecture.mdx:55-59); outputs encrypt_probability, ransomware_score
(threat-model.mdx:191-203).  Frozen spec: SURVEY.md 8a row a4 (torch.nn.LSTM semantics).

The parameters live in a real torch.nn.LSTM + nn.Linear (so state_dicts interchange with
PyTorch), but forward() never calls them: compute goes through `nerrf_lstm_forward`.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from ... import _lib as L

D_IN = 16      # event feature width (SURVEY.md 8a a4: syscall one-hot, log1p(bytes), dt, flags, ext pattern ...)
T_MAX = 100
# name of each of the D_IN event features, in the layout of pipeline.file_sequences (event kind one-hot x 8, size, dt,
# time, .lockbit name, /tmp|/proc path, 3 spare); sequence explanations name a step's dominant feature by it
FEATURE_NAMES = ("kind:file_created", "kind:file_encrypt_start", "kind:file_encrypt_complete", "kind:ransom_note_created",
                 "kind:openat", "kind:write", "kind:rename", "kind:other", "size", "dt", "time", "lockbit_name",
                 "tmp_or_proc_path", "spare_13", "spare_14", "spare_15")


class LSTMScorer(nn.Module):
    def __init__(self, in_dim: int = D_IN, hidden: int = 256, num_layers: int = 2, seed: int | None = 3):
        super().__init__()
        if hidden != 256:
            raise ValueError("hidden must be 256 (kernel block width)")
        if seed is not None:
            with torch.random.fork_rng(devices=[]):
                torch.manual_seed(seed)
                self.lstm = nn.LSTM(in_dim, hidden, num_layers=num_layers, bidirectional=True, batch_first=True)
                self.head = nn.Linear(2 * hidden, 2)
        else:
            self.lstm = nn.LSTM(in_dim, hidden, num_layers=num_layers, bidirectional=True, batch_first=True)
            self.head = nn.Linear(2 * hidden, 2)
        self.in_dim, self.hidden, self.num_layers = in_dim, hidden, num_layers
        self._packed = None
        self._packed_key = None

    def oracle_params(self):
        layers = []
        for l in range(self.num_layers):
            dirs = []
            for sfx in ("", "_reverse"):
                dirs.append(tuple(getattr(self.lstm, f"{n}_l{l}{sfx}").detach().cpu()
                                  for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")))
            layers.append(dirs)
        return {"lstm": layers, "head_W": self.head.weight.detach().cpu(), "head_b": self.head.bias.detach().cpu()}

    def _pack(self, device):
        params = [p for p in self.parameters()]
        key = (str(device),) + tuple((p._version, p.data_ptr()) for p in params)
        if self._packed_key == key:
            return self._packed
        wih, whh, bias = [], [], []
        for l in range(self.num_layers):
            for sfx in ("", "_reverse"):
                g = lambda n: getattr(self.lstm, f"{n}_l{l}{sfx}").detach().to(device=device, dtype=torch.float32)
                wih.append(g("weight_ih").t().contiguous())        # [D_l, 4H]
                whh.append(g("weight_hh").t().contiguous())        # [H, 4H]
                bias.append((g("bias_ih") + g("bias_hh")).contiguous())
        hw = self.head.weight.detach().to(device=device, dtype=torch.float32).contiguous()
        hb = self.head.bias.detach().to(device=device, dtype=torch.float32).contiguous()
        self._packed = (wih, whh, bias, hw, hb)
        self._packed_key = key
        return self._packed

    @torch.no_grad()
    def forward(self, seq, lengths):
        """seq fp32 [B,T,D_in] (CUDA), lengths int [B] (valid steps t < len) -> probs fp32 [B,2]
        = (encrypt_probability, ransomware_score)."""
        L.require_cuda(seq, lengths)
        if seq.dtype != torch.float32 or seq.dim() != 3 or seq.shape[2] != self.in_dim:
            raise ValueError(f"seq must be float32 [B,T,{self.in_dim}]")
        seq = seq.contiguous()
        B, T, _ = seq.shape
        ln = lengths.to(torch.int32).contiguous()
        if ln.numel() != B:
            raise ValueError("lengths must have B entries")
        wih, whh, bias, hw, hb = self._pack(seq.device)
        out = torch.empty(B, 2, device=seq.device, dtype=torch.float32)
        need = C.c_size_t()
        L.check(L.lib().nerrf_lstm_workspace_bytes(B, T, self.hidden, C.byref(need)), "nerrf_lstm_workspace_bytes")
        ws = torch.empty(need.value, device=seq.device, dtype=torch.uint8)
        L.check(L.lib().nerrf_lstm_forward(L.ptr(seq), L.ptr(ln), B, T, self.in_dim, self.hidden, self.num_layers,
                                           L.ptr_array(wih), L.ptr_array(whh), L.ptr_array(bias), L.ptr(hw), L.ptr(hb),
                                           L.ptr(out), L.ptr(ws), need.value, L.current_stream_ptr()),
                "nerrf_lstm_forward")
        return out


Model = LSTMScorer


def default_algo() -> str:
    """Which kernel family nerrf_lstm_forward runs: the wgmma path unless NERRF_LSTM_ALGO=ffma selects the fp32
    CUDA-core kernel (kept as an independent cross-check)."""
    import os
    return "ffma" if os.environ.get("NERRF_LSTM_ALGO", "").lower().startswith("f") else "umma (wgmma)"

_default = None


def forward(seq, lengths, model: LSTMScorer | None = None):
    """Module-level `lstm.forward` named by the north star; uses a process-wide default model."""
    global _default
    if model is None:
        if _default is None:
            _default = LSTMScorer().to(seq.device)
        model = _default
    return model(seq, lengths)
