"""BiLSTM training step timing at the benchmark's LSTM shape (B=4096, T=100, D_in=16, H=256, 2 layers, lengths in
[T/2, T]): the library's saved-activation forward (`nerrf_lstm_forward_train`) and backward-through-time
(`nerrf_lstm_backward`) against torch.nn.LSTM (cuDNN) forward + backward with TF32 off and on.  CUDA events, after
warm-up, median of several repetitions.  Also: the algorithmic FLOPs, the activation bytes each path keeps for its
backward, and a full-batch cross-check of the library's gradients against cuDNN with TF32 off.

    python scripts/lstm_train_timing.py [--out DIR] [--reps 5]      # one JSON line -> stdout and DIR/lstm_train_timing.json
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from torch.nn.utils.rnn import pack_padded_sequence

from nerrf_b200 import _lib as L
from nerrf_b200.ai import autograd as AG
from nerrf_b200.ai.models.lstm import LSTMScorer


def card():
    """Name and power limit, by read-only queries."""
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["nvidia_smi"] = q
    except Exception as e:                   # the timing stands without it; say why it is missing
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def timed(fn, reps, pre=None):
    """Median ms of fn() over reps runs, each bracketed by CUDA events (pre() runs outside the bracket)."""
    out = []
    for _ in range(reps):
        if pre:
            pre()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out)), [round(x, 3) for x in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="lstm_train_timing_out"); ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--B", type=int, default=4096); ap.add_argument("--T", type=int, default=100)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda")
    B, T, D, H, NL = a.B, a.T, 16, 256, 2
    torch.manual_seed(0)
    scorer = LSTMScorer(D, H, NL).to(dev)
    seq = torch.randn(B, T, D, device=dev)
    lengths = torch.randint(T // 2, T + 1, (B,), device=dev)
    ln = lengths.to(torch.int32).contiguous()
    dlogit = torch.randn(B, 2, device=dev)
    lib = L.lib()

    # ---- raw library calls on preallocated buffers
    params = AG.lstm_params(scorer)
    W_ih = [params[4 * i].detach().contiguous() for i in range(2 * NL)]
    W_hh = [params[4 * i + 1].detach().contiguous() for i in range(2 * NL)]
    wih_t = [w.t().contiguous() for w in W_ih]; whh_t = [w.t().contiguous() for w in W_hh]
    bias = [(params[4 * i + 2] + params[4 * i + 3]).detach().contiguous() for i in range(2 * NL)]
    tb, wb = C.c_size_t(), C.c_size_t()
    L.check(lib.nerrf_lstm_train_workspace_bytes(B, T, D, H, NL, C.byref(tb), C.byref(wb)), "workspace bytes")
    tape = torch.empty(tb.value, dtype=torch.uint8, device=dev)
    ws = torch.empty(wb.value, dtype=torch.uint8, device=dev)
    hfin = torch.empty(B, 2 * H, device=dev)
    dhfin = (dlogit @ scorer.head.weight).detach().contiguous()
    dseq = torch.empty_like(seq)
    dW_ih = [torch.empty_like(w) for w in W_ih]; dW_hh = [torch.empty_like(w) for w in W_hh]
    db = [torch.empty(4 * H, device=dev) for _ in range(2 * NL)]
    s = L.current_stream_ptr()
    fwd = lambda: L.check(lib.nerrf_lstm_forward_train(L.ptr(seq), L.ptr(ln), B, T, D, H, NL, L.ptr_array(wih_t),
                                                       L.ptr_array(whh_t), L.ptr_array(bias), L.ptr(hfin), L.ptr(tape),
                                                       tape.numel(), s), "forward_train")
    bwd = lambda: L.check(lib.nerrf_lstm_backward(L.ptr(seq), L.ptr(ln), B, T, D, H, NL, L.ptr_array(W_ih),
                                                  L.ptr_array(W_hh), L.ptr(tape), tape.numel(), L.ptr(dhfin), L.ptr(dseq),
                                                  L.ptr_array(dW_ih), L.ptr_array(dW_hh), L.ptr_array(db), L.ptr(ws),
                                                  ws.numel(), s), "backward")
    fwd(); bwd(); torch.cuda.synchronize()                                        # warm-up
    fwd_ms, fwd_all = timed(fwd, a.reps)
    bwd_ms, bwd_all = timed(bwd, a.reps, pre=fwd)                                 # each backward consumes a fresh tape

    # ---- torch.nn.LSTM (cuDNN) forward + backward
    lens_cpu = lengths.cpu()

    def torch_step():
        scorer.zero_grad(set_to_none=True)
        packed = pack_padded_sequence(seq, lens_cpu, batch_first=True, enforce_sorted=False)
        _, (hn, _) = scorer.lstm(packed)
        (scorer.head(torch.cat([hn[-2], hn[-1]], 1)) * dlogit).sum().backward()

    cudnn = {}
    for tf32 in (False, True):
        torch.backends.cudnn.allow_tf32 = tf32
        torch.backends.cuda.matmul.allow_tf32 = tf32
        torch_step(); torch_step(); torch.cuda.synchronize()
        cudnn["tf32_on" if tf32 else "tf32_off"] = timed(torch_step, a.reps)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    # activation memory cuDNN keeps for its backward (saved tensors + reserve space), at TF32 off
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    packed = pack_padded_sequence(seq, lens_cpu, batch_first=True, enforce_sorted=False)
    _, (hn, _) = scorer.lstm(packed)
    loss = (scorer.head(torch.cat([hn[-2], hn[-1]], 1)) * dlogit).sum()
    torch.cuda.synchronize()
    cudnn_saved = torch.cuda.memory_allocated() - base
    scorer.zero_grad(set_to_none=True)
    loss.backward()
    want = {n: p.grad.detach().clone() for n, p in scorer.named_parameters() if n.startswith("lstm.")}
    del loss, hn, packed

    # ---- cross-check: library gradients (through LSTMFn, the training path) vs cuDNN at TF32 off, full batch
    scorer.zero_grad(set_to_none=True)
    (AG.lstm_logits(scorer, seq, lengths) * dlogit).sum().backward()
    cross = {}
    for n, p in scorer.named_parameters():
        if n in want:
            g, w = p.grad.double(), want[n].double()
            cross[n] = {"max_abs_diff": float((g - w).abs().max()), "max_abs": float(w.abs().max()),
                        "rel_l2": float((g - w).norm() / w.norm().clamp_min(1e-30))}

    # ---- counts
    valid = int(lengths.sum())
    Ds = [D] + [2 * H] * (NL - 1)
    fwd_flops = sum(2 * 2 * valid * 4 * H * (d + H) for d in Ds)                            # 2 directions, 4 gates
    bwd_flops = sum(2 * 2 * valid * 4 * H * (2 * d + 2 * H) for d in Ds)   # dW_ih + d in, dW_hh + dh recurrence
    lib_tape = tb.value
    # the backward reads every layer's gates, cells and outputs once and writes the gates back (dg) once
    lib_bwd_tape_traffic = lib_tape + NL * 2 * B * T * 4 * H * 4
    res = {"script": "lstm_train_timing", "card": card(), "B": B, "T": T, "D_in": D, "H": H, "layers": NL,
           "lengths": f"uniform [{T // 2}, {T}]", "valid_steps": valid, "reps": a.reps,
           "library_forward_train_ms": round(fwd_ms, 3), "library_backward_ms": round(bwd_ms, 3),
           "library_step_ms": round(fwd_ms + bwd_ms, 3),
           "cudnn_fwd_bwd_ms_tf32_off": round(cudnn["tf32_off"][0], 3), "cudnn_fwd_bwd_ms_tf32_on": round(cudnn["tf32_on"][0], 3),
           "samples_ms": {"forward_train": fwd_all, "backward": bwd_all, "cudnn_tf32_off": cudnn["tf32_off"][1],
                          "cudnn_tf32_on": cudnn["tf32_on"][1]},
           "flops_forward": fwd_flops, "flops_backward": bwd_flops,
           "library_forward_tflops": round(fwd_flops / fwd_ms * 1e-9, 2),
           "library_backward_tflops": round(bwd_flops / bwd_ms * 1e-9, 2),
           "library_tape_bytes": lib_tape, "library_backward_tape_traffic_bytes": lib_bwd_tape_traffic,
           "library_backward_workspace_bytes": wb.value, "cudnn_saved_activation_bytes": int(cudnn_saved),
           "grad_vs_cudnn_tf32_off": cross}
    line = json.dumps(res)
    print(line)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "lstm_train_timing.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
